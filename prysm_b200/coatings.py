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
import operator
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


# ---- optical monitoring (prysm/x/coatings monitoring.py) ----------------------------------------------------------
# Any number of as-built runs is one pb_monitor_runs launch, one CTA per run: the layers are deposited from the
# substrate up as a 2-vector sweep, so a layer step costs O(1) where the reference rebuilds the product of every layer
# below it.  Traces, cutoff levels and the realized reflectance of the as-built stacks are pb_stack_eval launches, and J
# with its scores one pb_monitor_jacobian launch: simulate_run is 2 launches (levels, runs) and one copy of the N
# thicknesses, monitoring_error_sensitivity and choose_monitor_wavelength 4 launches whatever the number of candidates,
# layers or grid points (choose_monitor_wavelength copies its scores once).  The monitor polarization follows the
# reference's _admittance ('p' in any case is p, anything else s), and a mode other than 'R' monitors T.

_STRATEGIES = {'level': capi.MON_LEVEL, 'turning': capi.MON_TURNING}
_RUN_KWARGS = ('turning_index', 'signal_errors', 'thickness_errors', 'n_points', 'max_factor', 'levels')


def _mon_pol(pol):
    return capi.TF_POL_P if pol.lower() == 'p' else capi.TF_POL_S


def _mon_signal(mode):
    """(pb_monitor_runs mode, pb_stack_eval output) of the monitored quantity."""
    return (capi.MON_R, capi.TF_OUT_REFL) if mode == 'R' else (capi.MON_T, capi.TF_OUT_TRANS)


def _monitor_operands(stack, wvls, theta):
    """The six pb_monitor_runs operands of the candidate monitor wavelengths wvls (a sequence): every index resolved on
    the host at each wavelength as given, as the reference resolves it for one run."""
    C, N = len(wvls), len(stack)
    n0 = np.empty(C, dtype=np.complex128)
    nsub = np.empty(C, dtype=np.complex128)
    table = np.empty((N, C), dtype=np.complex128)
    for c, w in enumerate(wvls):
        n0[c] = _resolve(stack.ambient_index, w)
        nsub[c] = _resolve(stack.substrate_index, w)
        for j, n in enumerate(stack.indices):
            table[j, c] = _resolve(n, w)
    d = np.asarray(stack.thicknesses, dtype=config.precision)
    return [_real(np.asarray(wvls, dtype=np.float64)), _real(np.full(C, theta, dtype=np.float64)), _cplx(n0),
            _cplx(nsub), _cplx(table), _real(d)]


def _cutoff(stack, ops, pol, mode):
    """(C, N) fp64 nominal cutoff levels of the monitor operands `ops` in one pb_stack_eval over the (C, N) samples:
    sample (c, k) is the stack with the layers above k at zero thickness, an exact identity in the sweep."""
    N = len(stack)
    d = np.asarray(stack.thicknesses, dtype=np.float64)
    D = np.where(np.arange(N)[:, None] >= np.arange(N)[None, :], d[:, None], 0.0)
    sops = [ops[0][:, None], ops[1][:, None], ops[2][:, None], ops[3][:, None], ops[4][:, :, None],
            _real(D)[:, None, :]]
    out = _mon_signal(mode)[1]
    return _ops.stack_eval(capi.TF_COATINGS, _mon_pol(pol), sops, (out,), torch.float64)[out]


def _err_rows(err, N):
    """per-layer errors as a (rows, N) fp64 device array, or None"""
    if err is None:
        return None
    e = _real(err)
    if e.shape[-1] < N:
        # the reference reads errors[k] for every layer k
        raise IndexError(f'index {e.shape[-1]} is out of bounds for axis 0 with size {e.shape[-1]}')
    # like the reference, entries past the N-th are not read
    return (e[:N].reshape(1, N) if e.ndim == 1 else e[:, :N]).contiguous()


def _as_built(stack, wvls, runs, per_cand, err, strategy='level', turning_index=1, theta=0.0, pol='s', mode='R',
              n_points=600, max_factor=1.8, levels=None, rdtype=None):
    """(runs, N) as-built thicknesses of the runs at the monitor wavelengths wvls, run r at wvls[r // per_cand]; err the
    (runs, N) fp64 errors of the strategy or None.  Arguments are checked before any launch."""
    rdtype = _rdtype() if rdtype is None else rdtype
    N = len(stack)
    if N == 0 or runs == 0:
        return torch.empty((runs, N), dtype=rdtype, device=_ops.device())
    code = _STRATEGIES.get(strategy)
    if code is None:
        raise ValueError("strategy must be 'level' or 'turning'")
    n_points = operator.index(n_points)
    if n_points < 0:
        raise ValueError(f'Number of samples, {n_points}, must be non-negative.')
    if code == capi.MON_LEVEL and n_points == 0:
        raise ValueError('attempt to get argmin of an empty sequence')
    if code == capi.MON_TURNING and turning_index < 1:
        # the reference indexes its list of turning points with turning_index - 1; below 1 that is refused here
        raise IndexError(f'turning_index must be 1 or more, got {turning_index}')
    mcode = _mon_signal(mode)[0]
    ops = _monitor_operands(stack, wvls, theta)
    lv = None
    if code == capi.MON_LEVEL:
        if levels is None:
            lv = _cutoff(stack, ops, pol, mode)
        else:
            lv = _real(levels).reshape(-1, N).expand(len(wvls), N).contiguous()
    return _ops.monitor_runs(code, mcode, _mon_pol(pol), ops, runs, per_cand, err, lv, n_points, 1e-12,
                             float(max_factor), int(turning_index), rdtype)


def _strategy_errors(strategy, signal_errors, thickness_errors):
    """the error vector the strategy reads: the level strategy ignores thickness errors, the turning one signal errors"""
    return signal_errors if strategy == 'level' else thickness_errors if strategy == 'turning' else None


def monitoring_trace(stack, layer, monitor_wvl, *, theta=0.0, pol='s', mode='R', n_points=400, max_factor=1.0):
    """Monitor signal versus deposited thickness while growing layer `layer` (ambient side first; the layers after it,
    Python's slice `layer + 1:`, lie below): (d grid, signal) as device arrays, one pb_stack_eval launch."""
    th = np.asarray(stack.thicknesses, dtype=config.precision)
    d_target = float(th[layer])
    d_grid = np.linspace(0.0, max_factor * d_target, n_points)
    below = list(stack.indices[layer + 1:])
    # the growing layer's thickness varies per sample; the layers below are broadcast
    D = np.empty((1 + len(below), d_grid.size), dtype=np.float64)
    D[0] = d_grid
    D[1:] = th[layer + 1:, None]
    grow = types.SimpleNamespace(indices=[stack.indices[layer]] + below, thicknesses=D,
                                 substrate_index=stack.substrate_index, ambient_index=stack.ambient_index)
    ops, _ = _operands(grow, monitor_wvl, theta)
    out = _mon_signal(mode)[1]
    sig = _ops.stack_eval(capi.TF_COATINGS, _mon_pol(pol), ops, (out,), _rdtype())[out]
    return torch.as_tensor(d_grid.astype(config.precision)).to(_ops.device()), sig


def _trace(d, signal):
    """d and signal as device arrays of one real dtype"""
    d = d if isinstance(d, torch.Tensor) else torch.as_tensor(np.asarray(d))
    s = signal if isinstance(signal, torch.Tensor) else torch.as_tensor(np.asarray(signal))
    dt = torch.promote_types(d.dtype, s.dtype)
    dt = dt if dt in (torch.float32, torch.float64) else torch.float64
    return d.to(_ops.device(), dt).reshape(-1), s.to(_ops.device(), dt).reshape(-1)


def turning_points(d, signal):
    """Deposited thicknesses at the turning points (extrema) of a monitor trace: a device array, one launch and one
    copy (of the count)."""
    d, s = _trace(d, signal)
    out, count = _ops.monitor_cut(capi.MON_TURNING, d, s)
    return out[:int(count.item())]


def level_cut(d, signal, level, target=None):
    """Deposited thickness where the monitor signal crosses `level`: the crossing nearest `target`, or the first one;
    with none, the thickness of the sample nearest the level.  A Python float, one launch and one copy."""
    d, s = _trace(d, signal)
    if d.numel() == 0:
        raise ValueError('attempt to get argmin of an empty sequence')
    out, _ = _ops.monitor_cut(capi.MON_LEVEL, d, s, float(level), float('nan') if target is None else float(target))
    return float(out[0].item())


def cutoff_levels(stack, monitor_wvl, *, theta=0.0, pol='s', mode='R', n_points=400):
    """Nominal monitor level at the end of each layer's deposition (a device array, one launch)."""
    N = len(stack)
    if N == 0:
        return torch.empty(0, dtype=_rdtype(), device=_ops.device())
    return _cutoff(stack, _monitor_operands(stack, [monitor_wvl], theta), pol, mode)[0].to(_rdtype())


def simulate_runs(stack, monitor_wvl, *, signal_errors=None, thickness_errors=None, strategy='level',
                  turning_index=1, theta=0.0, pol='s', mode='R', n_points=600, max_factor=1.8, levels=None):
    """Any number of monitored deposition runs in one launch (plus one for the cutoff levels): the (R, N) as-built
    thicknesses as a device array.  The errors the strategy reads are (N,) or (R, N) (the level strategy reads
    signal_errors, the turning strategy thickness_errors); monitor_wvl is one wavelength or one per run.  Run r equals
    simulate_run with row r of the errors at monitor wavelength r, bit for bit."""
    N = len(stack)
    wvls = list(np.ravel(monitor_wvl)) if np.ndim(monitor_wvl) else [monitor_wvl]
    err = _err_rows(_strategy_errors(strategy, signal_errors, thickness_errors), N) if N else None
    rows = 1 if err is None else err.shape[0]
    runs = max(rows, len(wvls))
    if rows not in (1, runs) or len(wvls) not in (1, runs):
        raise ValueError(f'{len(wvls)} monitor wavelengths and {rows} error rows do not make one set of runs')
    if err is not None and rows != runs:
        err = err.expand(runs, N).contiguous()
    return _as_built(stack, wvls, runs, runs if len(wvls) == 1 else 1, err, strategy=strategy,
                     turning_index=turning_index, theta=theta, pol=pol, mode=mode, n_points=n_points,
                     max_factor=max_factor, levels=levels)


def simulate_run(stack, monitor_wvl, *, strategy='level', turning_index=1, signal_errors=None, thickness_errors=None,
                 theta=0.0, pol='s', mode='R', n_points=600, max_factor=1.8, levels=None):
    """Simulate a monitored deposition run: the as-built stack, of the input stack's class, with host thicknesses."""
    N = len(stack)
    err = _err_rows(_strategy_errors(strategy, signal_errors, thickness_errors), N) if N else None
    th = _as_built(stack, [monitor_wvl], 1, 1, err, strategy=strategy, turning_index=turning_index, theta=theta,
                   pol=pol, mode=mode, n_points=n_points, max_factor=max_factor, levels=levels)
    return type(stack)(stack.indices, _ops.asnumpy(th[0]), stack.substrate_index, stack.ambient_index)


def _sensitivity(stack, wvls, design_wvls, strategy, theta, pol, design_pol, mode, eps, kwargs, want_J):
    """(J (C, W, N) or None, scores (C,)) of the candidate monitor wavelengths wvls: each candidate's base run and its N
    perturbed runs in one pb_monitor_runs launch, their realized reflectance in one pb_stack_eval, J and the scores in
    one pb_monitor_jacobian."""
    N, C = len(stack), len(wvls)
    # the realized reflectance is read as the reference's RTA reads it, which refuses any polarization but s and p
    ipol = _pol(design_pol)
    dw = np.atleast_1d(np.asarray(design_wvls, dtype=config.precision))
    if dw.ndim != 1:
        raise ValueError(f'design_wvls must be one-dimensional, got shape {dw.shape}')
    for k in kwargs:
        if k not in _RUN_KWARGS:
            raise TypeError(f"simulate_run() got an unexpected keyword argument '{k}'")
    # the reference hands each perturbed run its own error vector, so one in kwargs is a second value for it
    own = 'thickness_errors' if strategy == 'turning' else 'signal_errors'
    if own in kwargs and N:
        raise TypeError(f"simulate_run() got multiple values for keyword argument '{own}'")
    kw = {k: v for k, v in kwargs.items() if k not in ('signal_errors', 'thickness_errors')}
    if N == 0:
        J = torch.zeros((C, dw.size, 0), dtype=_rdtype(), device=_ops.device()) if want_J else None
        return J, torch.zeros(C, dtype=_rdtype(), device=_ops.device())
    E = np.zeros((N + 1, N), dtype=np.float64)
    E[1:] = np.eye(N) * np.asarray(eps, dtype=config.precision)
    err = _real(np.tile(E, (C, 1)))
    th = _as_built(stack, wvls, C * (N + 1), N + 1, err, strategy=strategy, theta=theta, pol=pol, mode=mode,
                   rdtype=torch.float64, **kw)
    # the realized reflectance of every as-built stack at the design wavelengths: (runs, W)
    ops, _ = _operands(stack, dw, theta)
    ops = [o[None] if o.ndim == 1 else o for o in ops[:4]] + [
        ops[capi.TF_IN_N][:, None] if ops[capi.TF_IN_N].ndim == 2 else ops[capi.TF_IN_N], th.t()[:, :, None]]
    Rr = _ops.stack_eval(capi.TF_COATINGS, ipol, ops, (capi.TF_OUT_REFL,),
                         torch.float64)[capi.TF_OUT_REFL]
    return _ops.monitor_jacobian(Rr, C, N, float(eps), _rdtype(), want_J)


def monitoring_error_sensitivity(stack, monitor_wvl, design_wvls, *, strategy='level', theta=0.0, pol='s',
                                 design_pol='s', mode='R', eps=1e-4, **kwargs):
    """Jacobian (len(design_wvls), N) of the realized reflectance with respect to each layer's termination error (a
    device array); four launches and no copy."""
    J, _ = _sensitivity(stack, [monitor_wvl], design_wvls, strategy, theta, pol, design_pol, mode, eps, kwargs, True)
    return J[0]


def choose_monitor_wavelength(stack, candidates, design_wvls, *, strategy='level', theta=0.0, pol='s',
                              design_pol='s', mode='R', eps=1e-4, **kwargs):
    """The candidate monitor wavelength of lowest error sensitivity sqrt(sum J^2) (a Python float) and every
    candidate's score (a device array): four launches for all candidates together and one copy (of the scores)."""
    wvls = list(candidates)
    if not wvls:
        raise ValueError('attempt to get argmin of an empty sequence')
    _, scores = _sensitivity(stack, wvls, design_wvls, strategy, theta, pol, design_pol, mode, eps, kwargs, False)
    best = float(np.asarray(candidates)[int(np.argmin(_ops.asnumpy(scores)))])
    return best, scores
