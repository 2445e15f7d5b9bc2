"""Jones and Mueller calculus on the device (reference prysm/x/polarization.py).

Layout.  A Jones array the engine returns has the reference's shape (..., 2, 2) and values, but its storage is
element-planar: a contiguous (2, 2, *S) buffer seen through a permuted view, so that each element J[..., i, j] is a
contiguous plane of the pixels S.  Mueller and Kronecker arrays are (4, 4, *S) buffers seen as (*S, 4, 4), and Jones
vectors (2, 1, *S) buffers seen as (*S, 2, 1).  Chains of engine operations therefore never re-layout: the four planes
go straight into one batched transform, and every kernel here streams whole planes.  `_planes` is the one place that
knows this: it returns the planes of an engine array as they are, and converts anything else (an interleaved
(..., 2, 2) array from numpy or from tensor arithmetic, real or complex, host or device) in one pb_jones_planar launch.

Everything on the pixels runs in four kernels (csrc/polarization.cu): pb_jones_planar, pb_jones_product (the 2x2
matrix and elementwise products, either operand optionally conjugate-transposed), pb_jones_elements (the constructors)
and pb_jones_reduce (Mueller, Kronecker, Pauli).  `jones_matmul` is the one name the reference does not have: on the
device its `a @ b` would be torch's batched matmul on strided views.
"""
import functools
import inspect
import math

import numpy as np
import torch

from . import _ops
from . import propagation
from ._capi import (JONES_CONST, JONES_PLANES, JONES_SCALAR, JONES_SCALAR_REAL, JONES_MATMUL, JONES_HADAMARD, JONES_OP_N,
                    JONES_OP_H, JONES_FILL, JONES_ROTATION, JONES_RETARDER, JONES_DIATTENUATOR, JONES_VVR, JONES_MUELLER,
                    JONES_KRON, JONES_PAULI)
from .conf import config

# supported functions for jones_adapter (polarization.py:10-16)
supported_propagation_funcs = [
    'focus',
    'unfocus',
    'focus_dft',
    'unfocus_dft',
    'angular_spectrum'
]

_REAL = (torch.float32, torch.float64)
_CPLX = {torch.float32: torch.complex64, torch.float64: torch.complex128,
         torch.complex64: torch.complex64, torch.complex128: torch.complex128}


# ---- layout ------------------------------------------------------------------------------------------------------

def _view(storage, tail=(2, 2)):
    """(prod(tail), *S) element-planar storage -> the (*S, *tail) view the reference's shape asks for."""
    S = tuple(storage.shape[1:])
    return storage.view(*tail, *S).permute(*range(len(tail), len(tail) + len(S)), *range(len(tail)))


def _storage(a):
    """The (4, *S) storage an element-planar (..., 2, 2) device tensor views, or None for any other layout."""
    if not isinstance(a, torch.Tensor) or not a.is_cuda or not a.is_complex():
        return None
    nd = a.ndim
    p = a.permute(nd - 2, nd - 1, *range(nd - 2))
    return p.reshape(4, *a.shape[:-2]) if p.is_contiguous() else None


def _is_jones(a):
    return np.ndim(a) >= 2 and tuple(a.shape[-2:]) == (2, 2)


def _planes(a, cdtype=None):
    """The 4 element planes (4, *S) of a Jones array (..., 2, 2) at `cdtype` (default: the complex type of a's
    precision).  An element-planar engine array is returned as it is (no launch); anything else is converted by one
    pb_jones_planar launch, whatever its strides, real or complex, host or device."""
    if not _is_jones(a):
        raise ValueError(f'a Jones array (..., 2, 2) is required, got shape {tuple(np.shape(a))}')
    if np.ndim(a) > 4:
        raise ValueError(f'Jones arrays of at most two pixel axes are supported, got shape {tuple(a.shape)}')
    st = _storage(a)
    if st is not None and (cdtype is None or st.dtype == cdtype):
        return st
    if isinstance(a, torch.Tensor):
        t = a
    else:
        h = np.asarray(a)
        if any(s < 0 for s in h.strides):
            h = np.ascontiguousarray(h)
        t = torch.from_numpy(h)
    if t.dtype not in _CPLX:
        t = t.to(torch.float64)
    if cdtype is None:
        cdtype = _CPLX[t.dtype]
    S = tuple(t.shape[:-2])
    t = t.to(_ops.device()) if not t.is_cuda else t
    while t.ndim < 4:
        t = t.unsqueeze(0)
    return _ops.jones_planar(t, cdtype).view(4, *S)


def _promote(*arrays):
    """numpy's complex result type of the array operands (the precision of the widest), config's when there are none."""
    dts = [str(a.dtype) for a in arrays if a is not None]
    if not dts:
        return config.complex_dtype
    wide = any(d.endswith(('float64', 'complex128', 'int64', 'int32')) for d in dts)
    return torch.complex128 if wide else torch.complex64


def _constant(a):
    """A 2x2 as four host complex values (a device tensor is copied to the host: four values)."""
    v = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    return np.asarray(v, dtype=np.complex128).reshape(4)


def _operand(a, cdtype, scalar_ok=False):
    """(kind, device tensor or None, 4 constants or None, pixel shape or None) of one product operand: a 2x2
    constant, a Jones array or (scalar_ok) one plane broadcast to all four elements."""
    if np.ndim(a) == 2 and tuple(a.shape) == (2, 2) and not scalar_ok:
        return JONES_CONST, None, _constant(a), None
    if not scalar_ok:
        st = _planes(a, cdtype)
        return JONES_PLANES, st, None, tuple(st.shape[1:])
    t = _ops.asdevice(a)
    if t.is_complex():
        return JONES_SCALAR, t.to(cdtype).contiguous(), None, tuple(t.shape)
    return JONES_SCALAR_REAL, t.to(_ops._REAL_OF[cdtype]).contiguous(), None, tuple(t.shape)


def _product(mode, a, b, cdtype, ops=(JONES_OP_N, JONES_OP_N)):
    """out = op(A) (x) op(B) at cdtype for two operands of `_operand`, as a new element-planar Jones array."""
    (ak, at, ac, aS), (bk, bt, bc, bS) = a, b
    if aS is not None and bS is not None and aS != bS:
        raise ValueError(f'Jones operands over different pixels: {aS} and {bS}')
    S = aS if aS is not None else (bS if bS is not None else ())
    consts = np.zeros(8, dtype=np.complex128)
    if ac is not None:
        consts[:4] = ac
    if bc is not None:
        consts[4:] = bc
    dev = at.device if at is not None else (bt.device if bt is not None else _ops.device())
    out = torch.empty((4, *S), dtype=cdtype, device=dev)
    _ops.jones_product(mode, math.prod(S), (ak, at, ops[0]), (bk, bt, ops[1]), out, consts)
    return _view(out)


# ---- constructors (polarization.py:19-347) -----------------------------------------------------------------------

def _real_plane(v):
    t = _ops.asdevice(v)
    if t.is_complex():
        raise ValueError('a real array is required')
    return t if t.dtype in _REAL else t.to(torch.float64)


def _elements(kind, params, shape=None, plane=None):
    """The (4, *S) storage of one constructor over the pixels `shape` (default: the plane's; none for a 2x2)."""
    if plane is not None:
        plane = _real_plane(plane).contiguous()
        S = tuple(plane.shape) if shape is None else tuple(shape)
        if math.prod(S) != plane.numel():
            raise ValueError(f'a plane of shape {tuple(plane.shape)} does not fill the pixels {S}')
    else:
        S = () if shape is None else tuple(shape)
    out = torch.empty((4, *S), dtype=config.complex_dtype, device=_ops.device())
    _ops.jones_elements(kind, math.prod(S), params, out, plane)
    return out


def _is_array(v):
    return isinstance(v, (np.ndarray, torch.Tensor)) and np.ndim(v) > 0


def linear_pol_vector(angle, degrees=True):
    """Linearly polarized Jones vector [cos, sin] at `angle` (polarization.py:45-77): shape (2,) for a scalar angle,
    (*angle.shape, 2, 1) for an array."""
    scale = np.pi / 180 if degrees else 1.0
    if _is_array(angle):
        out = _elements(JONES_ROTATION, (0.0, scale), plane=angle)   # planes 0, 1 of the rotation: cos, sin
        return _view(out[:2], (2, 1))
    out = _elements(JONES_ROTATION, (float(angle) * scale, 1.0))
    return out[:2]


def circular_pol_vector(handedness='left', shape=None):
    """Circularly polarized Jones vector (polarization.py:80-104).  Like the reference, only shape=None works: with a
    shape its second element assignment indexes the vector's size-1 last axis and raises IndexError."""
    if handedness not in ('left', 'right'):
        raise ValueError(f"unknown handedness {handedness}, use 'left' or 'right'")  # NOQA
    if shape is not None:
        raise IndexError(f'index 1 is out of bounds for axis {len(shape) + 1} with size 1')
    s = 1 / np.sqrt(2)
    out = _elements(JONES_FILL, np.array([s, 1j * s if handedness == 'left' else -1j * s, 0, 0]).view(np.float64))
    return out[:2]


def jones_rotation_matrix(theta, shape=None):
    """[[cos, sin], [-sin, cos]] of theta [rad] (polarization.py:133-160); theta may be a plane of the pixels."""
    if _is_array(theta):
        return _view(_elements(JONES_ROTATION, (0.0, 1.0), shape, plane=theta))
    return _view(_elements(JONES_ROTATION, (float(theta), 1.0), shape))


def linear_retarder(retardance, theta=0, shape=None):
    """R(-theta) diag(1, exp(i retardance)) R(theta) (polarization.py:163-196); retardance may be a plane."""
    if _is_array(retardance):
        return _view(_elements(JONES_RETARDER, (float(theta), 0.0), shape, plane=retardance))
    return _view(_elements(JONES_RETARDER, (float(theta), float(retardance)), shape))


def linear_diattenuator(alpha, theta=0, shape=None):
    """R(-theta) diag(1, alpha) R(theta) (polarization.py:199-231).  alpha may also be a plane of the pixels (the
    reference's range assert takes the truth value of its argument, so it accepts scalars only)."""
    if _is_array(alpha):
        a = _real_plane(alpha)
        lo, hi = float(a.min()), float(a.max())
        assert lo >= 0 and hi <= 1, f'alpha cannot be less than 0 or greater than 1, got values in [{lo}, {hi}]'
        return _view(_elements(JONES_DIATTENUATOR, (float(theta), 0.0), shape, plane=a))
    assert (alpha >= 0) and (alpha <= 1), f"alpha cannot be less than 0 or greater than 1, got: {alpha}"
    return _view(_elements(JONES_DIATTENUATOR, (float(theta), float(alpha)), shape))


def half_wave_plate(theta=0, shape=None):
    """polarization.py:234-251."""
    return linear_retarder(np.pi, theta=theta, shape=shape)


def quarter_wave_plate(theta=0, shape=None):
    """polarization.py:254-272."""
    return linear_retarder(np.pi / 2, theta=theta, shape=shape)


def linear_polarizer(theta=0, shape=None):
    """polarization.py:275-293."""
    return linear_diattenuator(0, theta=theta, shape=shape)


def vector_vortex_retarder(charge, theta, retardance=np.pi, rotate=0):
    """Phase-only vector vortex retarder over the azimuth plane theta (polarization.py:296-346), with the
    reference's values: its constant -i cos(retardance/2) term is on [0, 0] only (it assigns [0, 0] twice).  Unlike
    the reference, theta is not modified (it multiplies theta by the charge in place)."""
    return _view(_elements(JONES_VVR, (float(charge), float(retardance), float(rotate)), plane=theta))


def pauli_spin_matrix(index, shape=None):
    """Pauli spin matrix `index` (polarization.py:410-452)."""
    assert index in (0, 1, 2, 3), f"index should be 0,1,2, or 3. Got {index}"
    m = {0: (1, 0, 0, 1), 1: (1, 0, 0, -1), 2: (0, 1, 1, 0), 3: (0, -1j, 1j, 0)}[index]
    return _view(_elements(JONES_FILL, np.array(m, dtype=np.complex128).view(np.float64), shape))


# ---- products and reductions (polarization.py:349-475, 555-578) --------------------------------------------------

def jones_matmul(a, b, adjoint_a=False, adjoint_b=False):
    """Per-pixel 2x2 product a @ b of two Jones arrays (..., 2, 2) over the same pixels, or of a Jones array and a
    2x2 constant, in one launch; adjoint_a / adjoint_b use the conjugate transpose of that operand (the adjoints of
    the product: Aᴴ·G with respect to b, G·Bᴴ with respect to a).  The result is an element-planar Jones array."""
    cdtype = _promote(*(x for x in (a, b) if np.ndim(x) > 2))
    return _product(JONES_MATMUL, _operand(a, cdtype), _operand(b, cdtype), cdtype,
                    (JONES_OP_H if adjoint_a else JONES_OP_N, JONES_OP_H if adjoint_b else JONES_OP_N))


def apply_polarization_optic(field, pol_optic):
    """pol_optic * field elementwise, a 2-D scalar field broadcast to all four elements (polarization.py:555-578)."""
    cdtype = _promote(field, *([pol_optic] if np.ndim(pol_optic) > 2 else []))
    f = _operand(field, cdtype, scalar_ok=np.ndim(field) == 2)
    return _product(JONES_HADAMARD, _operand(pol_optic, cdtype), f, cdtype)


def broadcast_kron(a, b):
    """Per-pixel Kronecker product of two Jones arrays -> (..., 4, 4) (polarization.py:349-376)."""
    cdtype = _promote(a, b)
    pa, pb = _planes(a, cdtype), _planes(b, cdtype)
    if pa.shape != pb.shape:
        raise ValueError(f'Jones operands over different pixels: {tuple(pa.shape[1:])} and {tuple(pb.shape[1:])}')
    out = torch.empty((16, *pa.shape[1:]), dtype=cdtype, device=pa.device)
    _ops.jones_reduce(JONES_KRON, pa[0].numel(), pa, out, pb)
    return _view(out, (4, 4))


def jones_to_mueller(jones, broadcast=True):
    """real(U kron(conj J, J) U^-1) per pixel, in closed form (polarization.py:379-407).  Both values of `broadcast`
    give the same per-pixel result."""
    p = _planes(jones)
    out = torch.empty((16, *p.shape[1:]), dtype=_ops._REAL_OF[p.dtype], device=p.device)
    _ops.jones_reduce(JONES_MUELLER, p[0].numel(), p, out)
    return _view(out, (4, 4))


def pauli_coefficients(jones):
    """(c0, c1, c2, c3), each a contiguous array of the pixels (polarization.py:455-475)."""
    p = _planes(jones)
    out = torch.empty_like(p)
    _ops.jones_reduce(JONES_PAULI, p[0].numel(), p, out)
    return out[0], out[1], out[2], out[3]


# ---- propagation (polarization.py:478-552) -----------------------------------------------------------------------

def _fft_adjoint(direction):
    def run(prop_func, planes, args):
        Q = args.get('Q')
        ky, kx = planes.shape[1:]
        return _ops.fft2_batch(planes, (ky, kx), dir=direction, scale=1.0 / math.sqrt(ky * kx), shift_in=True,
                               shift_out=True, crop=propagation._shape_before_pad((ky, kx), Q))
    return run


def _executor(adjoint):
    def run(prop_func, planes, args):
        ex = args['executor']
        if not hasattr(ex, '_forward'):             # not an engine executor: one call per element
            return None
        planes = _planes(_view(planes), ex._dtype)
        out = torch.empty((4, *ex._out_shape(adjoint)), dtype=ex._dtype, device=planes.device)
        for i in range(4):
            (ex._adjoint if adjoint else ex._forward)(planes[i], out=out[i])
        return out
    return run


def _angular_spectrum(adjoint):
    def run(prop_func, planes, args):
        wvl, dx, z = args['wvl'], args['dx'], args['z']
        Q, tf, screen = args.get('Q', 2), args.get('tf'), args.get('screen')
        k = tuple(planes.shape[1:]) if (tf is not None or adjoint) else propagation._padded_shape(planes.shape[1:], Q)
        kw = {}
        if tf is not None:
            kw = dict(tf=_ops.asdevice(tf).to(planes.dtype).contiguous(), conj_tf=adjoint)
            crop = k
        else:
            ty, tx = _ops.angular_spectrum_vectors(k, wvl, dx, z, planes.dtype, planes.device)
            kw = dict(ty=ty, tx=tx, conj_tf=adjoint)
            crop = propagation._shape_before_pad(k, Q) if adjoint else k
        if screen is not None:
            kw['screen'] = _ops.ascomplex(_ops.asdevice(screen)).to(planes.dtype).contiguous()
        out = torch.empty((4, *crop), dtype=planes.dtype, device=planes.device)
        for i in range(4):
            _ops.angular_spectrum(planes[i], k, crop=crop, out=out[i], **kw)
        return out
    return run


def _stack(prop_func, planes, args):
    return prop_func(planes, **{k: v for k, v in args.items() if k != _first_param(prop_func)})


def _first_param(f):
    return next(iter(inspect.signature(f).parameters))


# how a (4, M, N) stack of element planes runs through each engine propagation function
_PLANE_RUNNERS = {
    propagation.focus: _stack,                      # the batched form: one pb_fft2_batch for the four planes
    propagation.unfocus: _stack,
    propagation.focus_adjoint: _fft_adjoint(+1),
    propagation.unfocus_adjoint: _fft_adjoint(-1),
    propagation.focus_dft: _executor(False),
    propagation.unfocus_dft_adjoint: _executor(False),
    propagation.unfocus_dft: _executor(True),
    propagation.focus_dft_adjoint: _executor(True),
    propagation.angular_spectrum: _angular_spectrum(False),
    propagation.angular_spectrum_adjoint: _angular_spectrum(True),
}


def jones_adapter(prop_func):
    """Wrap a propagation function so that it propagates Jones fields (polarization.py:478-538).

    A (..., 2, 2) array with ndim == 4 is a Jones field: its four elements are propagated independently and the
    result is an element-planar Jones array.  Arrays with ndim <= 3 go to prop_func unchanged (a 3-D array is the
    engine's stack of independent fields); anything else raises ValueError.  focus / unfocus and their adjoints run
    the four planes as one batched transform; the matrix-DFT and angular-spectrum functions run once per plane with
    the executor's bases (or the transfer function) shared, each writing its plane of one output.  Any other
    function is called once per plane."""
    runner = _PLANE_RUNNERS.get(prop_func)

    @functools.wraps(prop_func)
    def wrapper(*args, **kwargs):
        wavefunction = args[0]
        nd = np.ndim(wavefunction)
        if nd <= 3:
            return prop_func(*args, **kwargs)
        if nd != 4 or tuple(wavefunction.shape[-2:]) != (2, 2):
            raise ValueError(f'a Jones field (M, N, 2, 2) or an array of at most 3 dimensions is required, '
                             f'got shape {tuple(np.shape(wavefunction))}')
        planes = _planes(wavefunction)
        out = None
        if runner is not None:
            bound = inspect.signature(prop_func).bind(*args, **kwargs)
            bound.apply_defaults()
            out = runner(prop_func, planes, dict(bound.arguments))
        if out is None:
            rets = [prop_func(planes[i], *args[1:], **kwargs) for i in range(4)]
            out = torch.stack([_ops.asdevice(r) for r in rets])
        return _view(out)

    return wrapper


def add_jones_propagation(funcs_to_change=supported_propagation_funcs):
    """Wrap the named prysm_b200.propagation functions with jones_adapter (polarization.py:541-552)."""
    for name, func in list(vars(propagation).items()):
        if name in funcs_to_change:
            setattr(propagation, name, jones_adapter(func))
