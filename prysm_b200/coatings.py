"""Thin-film coatings on the device: the stack and field engine of prysm.x.coatings (stack.py) and its analytic
gradients (diff.py).

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
