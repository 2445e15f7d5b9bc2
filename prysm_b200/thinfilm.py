"""Thin-film r and t on the device: multilayer_stack_rt of prysm/thinfilm.py.

The transfer-matrix chain runs in one launch of `pb_stack_eval` (csrc/thinfilm.cu), one thread per sample, in fp64;
r and t are stored in `config.precision`.  Arguments, shapes and exceptions are the reference's: the AOI is in
degrees, the first axis of indices and thicknesses is the layer axis and any trailing axes are calculation axes.
Inputs may be numpy arrays, scalars or CUDA tensors.
"""
import math

import numpy as np
import torch

from . import _capi as capi
from . import _ops
from .conf import config


def _shape(a):
    return tuple(a.shape) if isinstance(a, torch.Tensor) else np.shape(a)


def _dev(a, dtype):
    """fp64 / complex128 device tensor of a (a CUDA tensor keeps its strides; only a dtype change copies it)."""
    if isinstance(a, torch.Tensor):
        t = a if a.is_cuda else a.to(_ops.device())
        return t if t.dtype == dtype else t.to(dtype)
    npdt = np.float64 if dtype == torch.float64 else np.complex128
    return torch.as_tensor(np.asarray(a, dtype=npdt, order='C')).to(_ops.device())


def _real(a):
    return _dev(a, torch.float64)


def _cplx(a):
    return _dev(a, torch.complex128)


def _layer_shapes(indices, thicknesses):
    """_as_layer_arrays (thinfilm.py:191-210) on shapes: the common (layers, *calc) shape."""
    si, st = _shape(indices), _shape(thicknesses)
    si = si if len(si) else (1,)
    st = st if len(st) else (1,)
    try:
        shape = np.broadcast_shapes(si, st)
    except ValueError as exc:
        raise ValueError('indices and thicknesses must be broadcastable to the same shape') from exc
    if len(shape) < 1 or shape[0] == 0:
        raise ValueError('indices and thicknesses must contain at least one film layer')
    return shape


def _as_layers(a, shape):
    """a with the leading unit axes numpy's broadcast to `shape` would add (a view: the kernel broadcasts by strides)."""
    t = a if isinstance(a, torch.Tensor) else np.asarray(a)
    if t.ndim == 0:
        t = t[None]
    return t.reshape((1,) * (len(shape) - t.ndim) + tuple(t.shape))


def _to_calc(a, calc):
    """A per-sample operand the reference broadcasts against the flattened (P,) calculation axis, viewed on calc."""
    if math.prod(_shape(a)) == 1:
        return a.reshape(()) if isinstance(a, torch.Tensor) else np.asarray(a).reshape(())
    return a.reshape(calc) if isinstance(a, torch.Tensor) else np.asarray(a).reshape(calc)


def multilayer_stack_rt(indices, thicknesses, wavelength, polarization, substrate_index, aoi=0, ambient_index=1):
    """Compute r and t for a given stack of materials.

    Parameters
    ----------
    indices : ndarray
        refractive index for each film layer.  The first axis is the layer
        axis; any trailing axes are vectorized calculation dimensions.
    thicknesses : ndarray
        thickness of each film layer, microns.  Must be broadcastable to the
        same shape as indices.
    wavelength : float
        wavelength of light, microns
    polarization : str, {'p', 's'}
        the polarization state
    substrate_index : float or ndarray
        refractive index of the medium after the final film layer.  May be a
        scalar, or broadcastable to the trailing dimensions of indices and
        thicknesses.
    aoi : float, optional
        angle of incidence, degrees
    ambient_index : float, optional
        The refractive index the film is immersed in, defaults to 1 (vacuum)

    Returns
    -------
    (torch.Tensor, torch.Tensor)
        r, t coefficients, complex in config.precision

    """
    polarization = polarization.lower()
    if polarization not in ('p', 's'):
        raise ValueError("unknown polarization, use p or s")
    layer_shape = _layer_shapes(indices, thicknesses)
    calc = tuple(layer_shape[1:])
    n = _as_layers(indices, layer_shape)
    d = _as_layers(thicknesses, layer_shape)
    wvl, theta, n0, nsub = wavelength, aoi, ambient_index, substrate_index
    if len(layer_shape) > 1:
        try:
            np.broadcast_shapes(_shape(nsub), calc)
            if len(_shape(nsub)) > len(calc):
                raise ValueError
        except ValueError as exc:
            raise ValueError('substrate_index must be broadcastable to the trailing layer dimensions') from exc
        # the reference flattens the calculation axes to (P,) and broadcasts the per-sample operands against that
        P = math.prod(calc)
        flat = np.broadcast_shapes((P,), _shape(wvl), _shape(theta), _shape(n0))
        if math.prod(flat) != P:
            raise ValueError(f'cannot reshape array of size {math.prod(flat)} into shape {calc}')
        wvl, theta, n0 = (_to_calc(a, calc) for a in (wvl, theta, n0))
    ops = [_real(wvl), _real(theta), _cplx(n0), _cplx(nsub), _cplx(n), _real(d)]
    rdtype = _ops.torch_dtype(config.precision)
    res = _ops.stack_eval(capi.TF_THINFILM, capi.TF_POL_P if polarization == 'p' else capi.TF_POL_S, ops,
                          (capi.TF_OUT_R, capi.TF_OUT_T), rdtype, theta_scale=math.pi / 180)
    r, t = res[capi.TF_OUT_R], res[capi.TF_OUT_T]
    if len(layer_shape) > 1:
        r, t = r.reshape(calc), t.reshape(calc)
    return r, t
