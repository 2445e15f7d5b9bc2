"""Thin-film coatings on the device: the stack and field engine of prysm.x.coatings (stack.py), its analytic
gradients (diff.py), and the design layer on top of them: the merit terms (merit.py) and the needle function
(needle.py).

Every evaluation is one launch of `pb_stack_eval` (csrc/thinfilm.cu), one thread per (wavelength, angle) sample with
the transfer-matrix chain in fp64 registers; gradients are one `pb_stack_grad` pass plus a fixed-order reduction.
Results are device arrays in `config.precision`.  The functions take the reference's own `Stack` as well as this
module's (they read `indices`, `thicknesses`, `substrate_index`, `ambient_index` and `len`).  Layer indices are
resolved on the host as the reference's `_resolve` does (a constant, a callable of the wavelength, or an object with
`.nk`) and uploaded as one (layers, *wavelength shape) table.  Angles are radians, thicknesses and wavelengths
microns.
"""
import types

import numpy as np
import torch

from . import _capi as capi
from . import _ops
from .conf import config
from .thinfilm import _cplx, _real


def _resolve(index, wvl):
    """Resolve a constant, callable, or material index at wavelength wvl."""
    nk = getattr(index, 'nk', None)
    if callable(nk):
        return nk(wvl)
    if callable(index):
        return index(wvl)
    return index


def _rdtype():
    return _ops.torch_dtype(config.precision)


def _pol(pol):
    pol = pol.lower()
    if pol not in ('p', 's'):
        raise ValueError("unknown polarization, use 'p' or 's'")
    return capi.TF_POL_P if pol == 'p' else capi.TF_POL_S


class Stack:
    """A multilayer thin-film stack.

    Parameters
    ----------
    indices : sequence
        per-layer refractive index, ambient side first.
    thicknesses : sequence or ndarray
        per-layer physical thicknesses, microns.
    substrate_index : float, complex, or callable
        index of the medium after the last layer.
    ambient_index : float, complex, or callable, optional
        index of the incidence medium.

    """

    __slots__ = ('indices', 'thicknesses', 'substrate_index', 'ambient_index')

    def __init__(self, indices, thicknesses, substrate_index, ambient_index=1.0):
        indices = list(indices)
        thicknesses = np.asarray(thicknesses, dtype=config.precision)
        if thicknesses.ndim == 0:
            thicknesses = np.full(len(indices), thicknesses, dtype=config.precision)
        if len(indices) != thicknesses.shape[0]:
            raise ValueError('indices and thicknesses must describe the same number of layers')
        self.indices = indices
        self.thicknesses = thicknesses
        self.substrate_index = substrate_index
        self.ambient_index = ambient_index

    def __len__(self):
        return self.thicknesses.shape[0]

    def resolved_indices(self, wvl):
        """List of per-layer indices evaluated at wavelength wvl."""
        return [_resolve(n, wvl) for n in self.indices]

    def __repr__(self):
        return f'Stack({len(self)} layers, substrate={self.substrate_index!r})'


def _operands(stack, wvl, theta0):
    """The six device operands of pb_stack_eval and the host-resolved ambient index."""
    hw = _ops.asnumpy(wvl) if isinstance(wvl, torch.Tensor) else wvl
    n0 = _resolve(stack.ambient_index, hw)
    nsub = _resolve(stack.substrate_index, hw)
    ns = [_resolve(n, hw) for n in stack.indices]
    shape = np.broadcast_shapes(*[np.shape(n) for n in ns]) if ns else ()
    table = np.empty((len(ns),) + shape, dtype=np.complex128)
    for j, n in enumerate(ns):
        table[j] = n
    d = np.asarray(stack.thicknesses, dtype=np.float64)
    # the wavelength enters only through the layers: without any, the reference's results take no shape from it
    w = _real(wvl) if ns else _real(np.ones(()))
    return [w, _real(theta0), _cplx(n0), _cplx(nsub), _cplx(table), _real(d)], n0


def _evaluate(stack, wvl, theta0, pol, outputs):
    ipol = _pol(pol)
    ops, _ = _operands(stack, wvl, theta0)
    return _ops.stack_eval(capi.TF_COATINGS, ipol, ops, outputs, _rdtype())


def stack_rt(stack, wvl, theta0, pol):
    """Amplitude reflection and transmission coefficients r, t for a unit-amplitude incident wave."""
    res = _evaluate(stack, wvl, theta0, pol, (capi.TF_OUT_R, capi.TF_OUT_T))
    return res[capi.TF_OUT_R], res[capi.TF_OUT_T]


def internal_fields(stack, wvl, theta0, pol):
    """Tangential electric and magnetic field at every boundary; the leading axis indexes boundaries from the ambient
    side."""
    res = _evaluate(stack, wvl, theta0, pol, (capi.TF_OUT_E, capi.TF_OUT_H))
    return res[capi.TF_OUT_E], res[capi.TF_OUT_H]


def RTA(stack, wvl, theta0, pol):
    """Reflectance, transmittance, and per-layer absorptance (one leading entry per layer)."""
    res = _evaluate(stack, wvl, theta0, pol, (capi.TF_OUT_REFL, capi.TF_OUT_TRANS, capi.TF_OUT_ABS))
    return res[capi.TF_OUT_REFL], res[capi.TF_OUT_TRANS], res[capi.TF_OUT_ABS]


def field_at_depth(stack, z, wvl, theta0, pol):
    """Tangential field E, H at depth(s) z (microns from the ambient side) inside the stack: shaped like z at one
    wavelength and angle of incidence, or shaped like the samples for one depth and arrays of wavelength, angle or
    index."""
    N = len(stack)
    if N == 0:
        raise ValueError('field_at_depth requires at least one layer')
    ipol = _pol(pol)
    zb = np.concatenate([np.zeros(1), np.cumsum(np.asarray(stack.thicknesses, dtype=np.float64))])
    if isinstance(z, torch.Tensor):
        bad = bool(((z < 0) | (z > zb[-1])).any())
    else:
        zh = np.asarray(z, dtype=np.float64)
        bad = bool(np.any((zh < 0) | (zh > zb[-1])))
    if bad:
        raise ValueError('z must lie within the coating stack')
    ops, n0 = _operands(stack, wvl, theta0)
    if ops[0].numel() == 1 and ops[1].numel() == 1 and ops[2].numel() == 1 and ops[4][0].numel() == 1:
        # one sample, any depths: the boundary fields, then one thread per depth
        ops = [o.reshape(()) if q not in (capi.TF_IN_N, capi.TF_IN_D) else o.reshape(o.shape[0])
               for q, o in enumerate(ops)]
        res = _ops.stack_eval(capi.TF_COATINGS, ipol, ops, (capi.TF_OUT_E, capi.TF_OUT_H), torch.float64)
        return _ops.field_at_depth(ipol, _real(z), _real(zb), ops[capi.TF_IN_N], complex(np.asarray(n0).reshape(())),
                                   float(np.asarray(_ops.asnumpy(wvl)).reshape(())),
                                   float(np.asarray(_ops.asnumpy(theta0)).reshape(())),
                                   res[capi.TF_OUT_E], res[capi.TF_OUT_H], _ops.torch_dtype(config.precision_complex))
    if np.ndim(_ops.asnumpy(z)) != 0:
        raise ValueError('field_at_depth takes one depth when the wavelength, angle or indices are arrays')
    # one depth, many samples: z splits its layer in two, and the field at z is the field at the boundary between
    # the parts (the characteristic matrix of a layer is the product of those of its parts)
    zs = float(np.asarray(_ops.asnumpy(z)))
    li = min(max(int(np.searchsorted(zb, zs, side='right')) - 1, 0), N - 1)
    d = np.asarray(stack.thicknesses, dtype=np.float64)
    split = types.SimpleNamespace(
        indices=list(stack.indices[:li + 1]) + list(stack.indices[li:]),
        thicknesses=np.concatenate([d[:li], [zs - zb[li], zb[li + 1] - zs], d[li + 1:]]),
        substrate_index=stack.substrate_index, ambient_index=stack.ambient_index)
    res = _evaluate(split, wvl, theta0, pol, (capi.TF_OUT_E, capi.TF_OUT_H))
    return res[capi.TF_OUT_E][li + 1], res[capi.TF_OUT_H][li + 1]


_FWD_OUT = (capi.TF_OUT_R, capi.TF_OUT_T, capi.TF_OUT_E, capi.TF_OUT_H, capi.TF_OUT_REFL, capi.TF_OUT_TRANS,
            capi.TF_OUT_ABS, capi.TF_OUT_ESQ, capi.TF_OUT_ETA0, capi.TF_OUT_ETASUB)


class ForwardEval:
    """Cached forward evaluation of a stack, on the device.

    The boundary fields are kept in fp64 for the gradients whatever `config.precision` is; the attributes `r`, `t`,
    `E`, `H`, `v_sub`, `eta0`, `eta_sub` and the `*_value` results are device arrays in `config.precision`.  The
    reference's per-layer lists (`matrices`, `L`, `R`, `betas`, `etas`, `dbeta_dd`, `ns`, `costs`) are not kept.
    """

    __slots__ = ('stack', 'wvl', 'theta0', 'pol', 'n0', 'eta0', 'eta_sub', 'r', 't', 'v_sub', 'E', 'H',
                 'R_value', 'T_value', 'A_value', 'Esq_value', '_ops', '_ipol', '_E64', '_H64')

    def __init__(self, stack, wvl, theta0, pol):
        """Evaluate and cache stack state.

        Parameters
        ----------
        stack : Stack
        wvl : float or ndarray
            wavelength(s), microns.
        theta0 : float or ndarray
            angle(s) of incidence in the ambient medium, radians.
        pol : str
            polarization, 'p' or 's'.

        """
        self._ipol = _pol(pol)
        self.stack = stack
        self.wvl = wvl
        self.theta0 = theta0
        self.pol = pol.lower()
        self._ops, n0 = _operands(stack, wvl, theta0)
        self.n0 = self._ops[capi.TF_IN_N0]
        res = _ops.stack_eval(capi.TF_COATINGS, self._ipol, self._ops, _FWD_OUT, torch.float64)
        self._E64, self._H64 = res[capi.TF_OUT_E], res[capi.TF_OUT_H]
        if _rdtype() != torch.float64:
            res = {k: v.to(torch.complex64 if v.is_complex() else torch.float32) for k, v in res.items()}
        self.r, self.t = res[capi.TF_OUT_R], res[capi.TF_OUT_T]
        self.E, self.H = res[capi.TF_OUT_E], res[capi.TF_OUT_H]
        self.eta0, self.eta_sub = res[capi.TF_OUT_ETA0], res[capi.TF_OUT_ETASUB]
        self.v_sub = torch.stack([self.E[-1], self.H[-1]], dim=-1)     # f_N = t [1, eta_sub]
        self.R_value, self.T_value = res[capi.TF_OUT_REFL], res[capi.TF_OUT_TRANS]
        self.A_value, self.Esq_value = res[capi.TF_OUT_ABS], res[capi.TF_OUT_ESQ]


def forward_eval(stack, wvl, theta0, pol):
    """Build a ForwardEval for one sample set."""
    return ForwardEval(stack, wvl, theta0, pol)


def _seed(v, shape):
    """A cotangent (numpy, scalar or device array) as a contiguous fp64 device array of the full shape."""
    if v is None:
        return None
    if isinstance(v, torch.Tensor):
        t = v if v.is_cuda else v.to(_ops.device())
        return t.to(torch.float64).expand(shape).contiguous()
    return torch.as_tensor(np.broadcast_to(np.asarray(v, dtype=np.float64), shape).copy()).to(_ops.device())


def _gradient(fwd, kinds, dR, dT, dA, dEsq):
    shape = tuple(fwd._E64.shape[1:])
    N = fwd._E64.shape[0] - 1
    seeds = [_seed(dR, shape), _seed(dT, shape), _seed(dA, (N,) + shape), _seed(dEsq, (N + 1,) + shape)]
    return _ops.stack_grad(fwd._ipol, kinds, fwd._ops, fwd._E64, fwd._H64, seeds, _rdtype())


def thickness_gradient(fwd, dR=None, dT=None, dA=None, dEsq=None):
    """Gradient of a scalar merit w.r.t. every layer thickness: real, one value per layer.  The seeds are the
    cotangents of R, T (sample shape), A (layers, *sample shape) and |E|^2 (boundaries, *sample shape)."""
    return _gradient(fwd, capi.TF_GRAD_THICKNESS, dR, dT, dA, dEsq)


def index_gradient(fwd, dR=None, dT=None, dA=None, dEsq=None):
    """Gradient of a scalar merit w.r.t. every layer index: real, one value per layer (seeds as thickness_gradient)."""
    return _gradient(fwd, capi.TF_GRAD_INDEX, dR, dT, dA, dEsq)


# ---- coating design: merit terms and the needle function (prysm/x/coatings merit.py, needle.py) -----------------
# Each term is one pb_coating_merit launch over its sample grid plus one fixed-order reduce launch; the seed of the
# reverse sweep is formed in registers, so no forward-eval fields or seed arrays are materialised.  Values are Python
# floats (one device-to-host copy per call), residuals, gradients and P(z) device arrays in config.precision.

def _as_grid(x):
    return np.asarray(x, dtype=config.precision)


def _validate_term_shapes(wvl, theta, target, weight):
    if wvl.ndim == 1 and theta.ndim == 1 and wvl.size > 1 and theta.size > 1:
        raise ValueError(
            'wvl and theta are both 1-D; pass meshgridded arrays for a '
            'spectral/angular grid')
    try:
        np.broadcast_arrays(wvl, theta, target, weight)
    except ValueError as exc:
        raise ValueError(
            'wvl, theta, target, and weight must be broadcast-compatible'
        ) from exc


def _index(i, size):
    """i as a non-negative index into an axis of `size`, numpy's rules (IndexError with numpy's message)."""
    i = int(i)
    if not -size <= i < size:
        raise IndexError(f'index {i} is out of bounds for axis 0 with size {size}')
    return i % size


_GRAD_FNS = {'thickness_gradient': capi.CM_OUT_GRAD_THICKNESS, 'index_gradient': capi.CM_OUT_GRAD_INDEX}


def _grad_flag(grad_fn):
    """The gradient kind of grad_fn: this module's or the reference's thickness_gradient / index_gradient."""
    name = getattr(grad_fn, '__name__', None)
    if name in _GRAD_FNS and getattr(grad_fn, '__module__', None) in (__name__, 'prysm.x.coatings.diff'):
        return _GRAD_FNS[name]
    raise TypeError(f'grad_fn must be thickness_gradient or index_gradient, got {grad_fn!r}')


class _Term:
    """Base spectral/angular merit term; the sample grid is uploaded once, here."""

    quantity = None
    _code = None

    def __init__(self, wvl, theta=0.0, pol='avg', target=0.0, weight=1.0):
        """Define a merit term over a (wvl, theta, pol) sample grid.

        Parameters
        ----------
        wvl : float or ndarray
            wavelength sample(s), microns.
        theta : float or ndarray, optional
            angle(s) of incidence in the ambient medium, radians.
        pol : str, optional
            's', 'p', or 'avg' (the unpolarized mean of s and p).
        target : float or ndarray, optional
            desired value of the quantity at each sample.
        weight : float or ndarray, optional
            relative weight of each sample in the sum-of-squares merit.

        """
        self.wvl = _as_grid(wvl)
        self.theta = _as_grid(theta)
        pol = pol.lower()
        if pol not in ('s', 'p', 'avg'):
            raise ValueError("pol must be 's', 'p', or 'avg'")
        self.pol = pol
        self.target = _as_grid(target)
        self.weight = _as_grid(weight)
        _validate_term_shapes(self.wvl, self.theta, self.target, self.weight)
        self._dev = [_real(self.wvl), _real(self.theta), _real(self.target), _real(self.weight)]

    def _ipol(self):
        return {'s': capi.TF_POL_S, 'p': capi.TF_POL_P, 'avg': capi.CM_POL_AVG}[self.pol]

    def _indices(self, N):
        """(b0, b1, device boundary list) of the term for a stack of N layers."""
        return 0, 0, None

    def _operands(self, stack):
        ops, _ = _operands(stack, self.wvl, self.theta)
        if len(stack):
            ops[capi.TF_IN_WVL] = self._dev[0]
        ops[capi.TF_IN_THETA] = self._dev[1]
        return ops + self._dev[2:]

    def _launch(self, stack, flags, value=None, residuals=None, grad=None, ops=None):
        b0, b1, blist = self._indices(len(stack))
        ops = self._operands(stack) if ops is None else ops
        if flags & (capi.CM_OUT_GRAD_THICKNESS | capi.CM_OUT_GRAD_INDEX):
            # the reference broadcasts dF/dq = 2 w (q - target) to the shape of q: a target or weight that extends it
            # is refused as numpy refuses it
            calc = [tuple(t.shape[1:]) if q in (capi.TF_IN_N, capi.TF_IN_D) else tuple(t.shape)
                    for q, t in enumerate(ops[:capi.TF_NOPS])]
            qshape = np.broadcast_shapes(*calc)
            np.broadcast_to(np.broadcast_to(False, np.broadcast_shapes(qshape, *[t.shape for t in ops[6:]])), qshape)
        _ops.coating_merit(self._code, self._ipol(), flags, ops, b0, b1, blist, value, residuals, grad, _rdtype())

    def _count(self, stack):
        ops = self._operands(stack)
        calc = [tuple(t.shape[1:]) if q in (capi.TF_IN_N, capi.TF_IN_D) else tuple(t.shape) for q, t in enumerate(ops)]
        return int(np.prod(np.broadcast_shapes(*calc), dtype=np.int64)), ops

    def residuals(self, stack):
        """Weighted residual vector sqrt(w) (q - target), flattened over samples (a device array)."""
        return MeritFunction([self]).residuals(stack)

    def value(self, stack):
        """Weighted sum of squared deviations from target (a scalar)."""
        return MeritFunction([self]).value(stack)

    def value_and_grad(self, stack, grad_fn=thickness_gradient):
        """Scalar value and gradient (a device array) via grad_fn."""
        return MeritFunction([self]).value_and_grad(stack, grad_fn=grad_fn)


class Reflectance(_Term):
    """Target the intensity reflectance R = abs(r)^2 over a sample grid."""

    quantity = 'R'
    _code = capi.CM_Q_R


class Transmittance(_Term):
    """Target the intensity transmittance T over a sample grid."""

    quantity = 'T'
    _code = capi.CM_Q_T


class LayerAbsorptance(_Term):
    """Target the absorptance A of one layer over a sample grid."""

    quantity = 'A'
    _code = capi.CM_Q_ABS

    def __init__(self, layer, wvl, theta=0.0, pol='avg', target=0.0, weight=1.0):
        super().__init__(wvl, theta=theta, pol=pol, target=target, weight=weight)
        self.layer = int(layer)

    def _indices(self, N):
        return _index(self.layer, N), 0, None


class FieldIntensityAtBoundary(_Term):
    """Target the standing-wave intensity abs(E)^2 at one boundary."""

    quantity = 'Esq'
    _code = capi.CM_Q_ESQ

    def __init__(self, boundary, wvl, theta=0.0, pol='avg', target=0.0, weight=1.0):
        super().__init__(wvl, theta=theta, pol=pol, target=target, weight=weight)
        self.boundary = int(boundary)

    def _indices(self, N):
        return _index(self.boundary, N + 1), 0, None


class PeakFieldAtInterfaces(_Term):
    """Target the peak standing-wave intensity over a set of boundaries (default every boundary); ties go to the first
    maximum, and a boundary listed twice keeps the seed of its last listing only, as numpy's fancy assignment does."""

    quantity = 'Esq'
    _code = capi.CM_Q_PEAK

    def __init__(self, wvl, theta=0.0, pol='avg', boundaries=None, target=0.0, weight=1.0):
        super().__init__(wvl, theta=theta, pol=pol, target=target, weight=weight)
        self.boundaries = None if boundaries is None else list(boundaries)
        self._blist = {}

    def _indices(self, N):
        if N not in self._blist:
            b = list(range(N + 1)) if self.boundaries is None else [_index(i, N + 1) for i in self.boundaries]
            if not b:
                raise ValueError('zero-size array to reduction operation maximum which has no identity')
            last = [int(all(b[j] != b[i] for j in range(i + 1, len(b)))) for i in range(len(b))]
            self._blist[N] = torch.as_tensor(np.asarray(b + last, dtype=np.int32)).to(_ops.device())
        return 0, 0, self._blist[N]


class FieldInLayer(_Term):
    """Target the mean standing-wave intensity at a layer's two boundaries (layer and layer + 1, numpy's indexing:
    layer -1 averages boundaries N and 0)."""

    quantity = 'Esq'
    _code = capi.CM_Q_LAYER

    def __init__(self, layer, wvl, theta=0.0, pol='avg', target=0.0, weight=1.0):
        super().__init__(wvl, theta=theta, pol=pol, target=target, weight=weight)
        self.layer = int(layer)

    def _indices(self, N):
        return _index(self.layer, N + 1), _index(self.layer + 1, N + 1), None


_TERM_CLASSES = {c.__name__: c for c in (Reflectance, Transmittance, LayerAbsorptance, FieldIntensityAtBoundary,
                                         PeakFieldAtInterfaces, FieldInLayer)}


def _as_term(t):
    """One of this module's terms, or a reference term rebuilt from its public attributes."""
    if isinstance(t, _Term):
        return t
    cls = _TERM_CLASSES.get(type(t).__name__)
    if cls is None:
        raise TypeError(f'not a merit term: {t!r}')
    kw = dict(theta=t.theta, pol=t.pol, target=t.target, weight=t.weight)
    if cls is PeakFieldAtInterfaces:
        return cls(t.wvl, boundaries=t.boundaries, **kw)
    if cls in (LayerAbsorptance, FieldInLayer):
        return cls(t.layer, t.wvl, **kw)
    if cls is FieldIntensityAtBoundary:
        return cls(t.boundary, t.wvl, **kw)
    return cls(t.wvl, **kw)


class MeritFunction:
    """A weighted collection of merit terms; each call takes two launches per term and, for value and
    value_and_grad, one device-to-host copy (of the value)."""

    __slots__ = ('terms',)

    def __init__(self, terms):
        """Collect one or more merit terms (this module's or the reference's) into a single objective."""
        if isinstance(terms, _Term) or type(terms).__name__ in _TERM_CLASSES:
            terms = [terms]
        self.terms = [_as_term(t) for t in terms]

    def value(self, stack):
        """Total weighted sum-of-squares merit (a scalar)."""
        if not self.terms:
            return 0.0
        v = torch.empty(1, dtype=torch.float64, device=_ops.device())
        for j, t in enumerate(self.terms):
            t._launch(stack, capi.CM_OUT_VALUE | (capi.CM_ACCUMULATE if j else 0), value=v)
        return float(v.item())

    def residuals(self, stack):
        """Concatenated weighted residual vector across all terms (a device array)."""
        counted = [t._count(stack) for t in self.terms]
        out = torch.empty(sum(c for c, _ in counted), dtype=_rdtype(), device=_ops.device())
        o = 0
        for t, (c, ops) in zip(self.terms, counted):
            if c:
                t._launch(stack, capi.CM_OUT_RESIDUALS, residuals=out[o:o + c], ops=ops)
            o += c
        return out

    def value_and_grad(self, stack, grad_fn=thickness_gradient):
        """Total merit (a float) and its gradient (a device array of one value per layer) via grad_fn."""
        kind = _grad_flag(grad_fn)
        if not self.terms:
            return 0.0, torch.zeros(len(stack), dtype=_rdtype(), device=_ops.device())
        grad = torch.empty(len(stack), dtype=_rdtype(), device=_ops.device())
        v = torch.empty(1, dtype=torch.float64, device=_ops.device())
        for j, t in enumerate(self.terms):
            t._launch(stack, capi.CM_OUT_VALUE | kind | (capi.CM_ACCUMULATE if j else 0), value=v, grad=grad)
        return float(v.item()), grad


def as_merit(obj):
    """Normalize a term, list of terms, or MeritFunction (this module's or the reference's) into a MeritFunction."""
    if isinstance(obj, MeritFunction):
        return obj
    if isinstance(obj, _HostMerit):
        return obj.merit
    if isinstance(obj, _Term) or type(obj).__name__ in _TERM_CLASSES:
        return MeritFunction([obj])
    if type(obj).__name__ == 'MeritFunction':
        return MeritFunction(list(obj.terms))
    return MeritFunction(list(obj))


def _depth_runs(stack, z):
    """(zpart (2, nz) fp64, zlist int32) of depths z: the reference's layer rule clip(searchsorted(Z, z, 'right') - 1,
    0, N - 1), the partial thicknesses z - Z_j and Z_{j+1} - z in config.precision, and the depth indices grouped by
    layer after each layer's start offset."""
    N = len(stack)
    Z = np.concatenate([np.zeros(1, dtype=config.precision),
                        np.cumsum(np.asarray(stack.thicknesses, dtype=config.precision))])
    j = np.clip(np.searchsorted(Z, z, side='right') - 1, 0, N - 1)
    zpart = np.stack([z - Z[j], Z[j + 1] - z]).astype(np.float64)
    order = np.argsort(j, kind='stable')
    starts = np.searchsorted(j[order], np.arange(N + 1))
    zlist = np.concatenate([starts, order]).astype(np.int32)
    return _real(zpart), torch.as_tensor(zlist).to(_ops.device())


def needle_function(stack, targets, needle_material, z):
    """Merit derivative P(z) for inserting a thin layer of needle_material at depth(s) z (microns from the ambient
    side), for reflectance / transmittance terms: a device array shaped like atleast_1d(z); negative values lower the
    merit.  Depths outside the stack are evaluated in the clipped first or last layer, as the reference does."""
    merit = as_merit(targets)
    for t in merit.terms:
        if t._code not in (capi.CM_Q_R, capi.CM_Q_T):
            raise NotImplementedError('needle synthesis supports reflectance / transmittance targets')
    if len(stack) == 0:
        raise ValueError('needle_function requires at least one layer')
    z = np.atleast_1d(np.asarray(z, dtype=config.precision))
    if not merit.terms or not z.size:
        return torch.zeros(z.shape, dtype=_rdtype(), device=_ops.device())
    zpart, zlist = _depth_runs(stack, z.reshape(-1))
    P = torch.empty(z.size, dtype=_rdtype(), device=_ops.device())
    for j, t in enumerate(merit.terms):
        ops = t._operands(stack)
        ops.append(_cplx(_resolve(needle_material, t.wvl)))
        _ops.needle(t._code, t._ipol(), ops, zpart, zlist, P, accumulate=j > 0)
    return P.reshape(z.shape)


class _HostMerit:
    """A MeritFunction whose results are numpy arrays: what the reference's host optimizer loops (CoatingProblem,
    refine, synthesize) consume after set_backend_to_b200()."""

    __slots__ = ('merit',)

    def __init__(self, merit):
        self.merit = merit

    @property
    def terms(self):
        return self.merit.terms

    def value(self, stack):
        return self.merit.value(stack)

    def residuals(self, stack):
        return _ops.asnumpy(self.merit.residuals(stack))

    def value_and_grad(self, stack, grad_fn=thickness_gradient):
        v, g = self.merit.value_and_grad(stack, grad_fn=grad_fn)
        return v, _ops.asnumpy(g)


def _host_as_merit(obj):
    """as_merit for the reference's host loops: the merit evaluates on the device and hands back numpy."""
    return obj if isinstance(obj, _HostMerit) else _HostMerit(as_merit(obj))


def _host_needle_function(stack, targets, needle_material, z):
    """needle_function for the reference's synthesize loop, which takes np.argmin of P: P as a numpy array."""
    return _ops.asnumpy(needle_function(stack, targets, needle_material, z))
