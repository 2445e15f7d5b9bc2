"""Coordinate grids on the device (reference prysm/coordinates.py:73-102, 344-378) -- the inputs of the pupil
synthesis that precedes the propagation path."""
import torch

from . import _ops
from .conf import config


def make_xy_grid(shape, *, dx=0, diameter=0, grid=True):
    """x, y = fftrange(n)*dx per axis in config precision (prysm/coordinates.py:344-378); one kernel for both
    meshgrids.  shape is (rows, cols); diameter, if given, sets dx = diameter / max(shape)."""
    if not isinstance(shape, tuple):
        shape = (shape, shape)
    if diameter != 0:
        dx = diameter / max(shape)
    g = _ops.xy_grid(shape, dx, config.real_dtype, _ops.device(), want='xy')
    if grid:
        return g['x'], g['y']
    return g['x'][0].contiguous(), g['y'][:, 0].contiguous()


def make_polar_grid(shape, *, dx=0, diameter=0):
    """r, t of the same grid without materialising x, y (cart_to_polar(*make_xy_grid(...)) in one kernel)."""
    if not isinstance(shape, tuple):
        shape = (shape, shape)
    if diameter != 0:
        dx = diameter / max(shape)
    g = _ops.xy_grid(shape, dx, config.real_dtype, _ops.device(), want='rt')
    return g['r'], g['t']


def warp(img, xnew, ynew):
    """Pull-warp a real image: out[i, j] = img at (row ynew[i, j], column xnew[i, j]) by cubic-spline interpolation,
    0 outside the image (prysm/coordinates.py:644-672: map_coordinates(img, (ynew, xnew)) at order 3,
    mode='constant', prefilter=True).  One prefilter and one interpolation kernel; the output has img's dtype."""
    return _ops.warp(img, xc=xnew, yc=ynew)


def interp_axes(x, y):
    """(x axis, y axis) as fp64 device vectors and the host float max|x, y ends| of two sorted 1-D axes (host arrays or
    tensors), the radius of uniform_cart_to_polar's lattice.  Only the axes cross to the host, never the data."""
    import numpy as np
    xh = np.asarray(_ops.asnumpy(x), dtype=np.float64).reshape(-1)
    yh = np.asarray(_ops.asnumpy(y), dtype=np.float64).reshape(-1)
    rmax = float(np.max(np.abs(np.asarray([xh.min(), xh.max(), yh.min(), yh.max()]))))
    return _ops.asdevice(xh), _ops.asdevice(yh), rmax, xh, yh


def polar_lattice_axes(rmax, nx, ny):
    """rho = linspace(0, rmax, nx) and phi = linspace(0, 2 pi, ny), fp64 device vectors (numpy's linspace, uploaded)."""
    import numpy as np
    return _ops.asdevice(np.linspace(0, rmax, nx)), _ops.asdevice(np.linspace(0, 2 * np.pi, ny))


def uniform_cart_to_polar(x, y, data):
    """Linear interpolation of data on the sorted 1-D axes x, y onto the polar lattice rho = linspace(0, max|x, y|,
    len(x)), phi = linspace(0, 2 pi, len(y)), 0 outside the axes (prysm/coordinates.py:269-316): one kernel, fp64
    coordinates and weights.  Returns (rho, phi, polar); rho, phi fp64, polar (len(y), len(x)) of data's dtype."""
    data = _ops.asdevice(data)
    xd, yd, rmax, _, _ = interp_axes(x, y)
    if tuple(data.shape) != (yd.numel(), xd.numel()):
        raise ValueError(f'data of shape {tuple(data.shape)} does not match axes of length ({yd.numel()}, {xd.numel()})')
    rho, phi = polar_lattice_axes(rmax, xd.numel(), yd.numel())
    return rho, phi, _ops.interp2d_linear(data, xd, yd, rmax=rmax)


def cart_to_polar(x, y, vec_to_grid=True):
    """rho = hypot(x, y), phi = arctan2(y, x) (prysm/coordinates.py:73-102); 1-D vectors broadcast to a grid."""
    x, y = _ops.asdevice(x), _ops.asdevice(y)
    if x.dtype not in (torch.float32, torch.float64):
        x = x.to(config.real_dtype)
    if vec_to_grid and x.ndim == 1:
        ny, nx = y.shape[0], x.shape[0]
        x, y = x[None, :].expand(ny, nx), y[:, None].expand(ny, nx)
    return _ops.cart_to_polar(x, y)
