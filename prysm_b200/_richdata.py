"""The container `Wavefront.intensity` and the otf functions return, with the reference's coordinates, slices, azimuthal
statistics and exact sampling on the device (reference prysm/_richdata.py:11-309, plotting excepted).

Every sampling step goes through one interpolator kernel with the semantics of scipy's
RegularGridInterpolator(method='linear'), so exact_xy, exact_polar, the slices' azimuthal statistics and
psf.estimate_size agree with one another.  Coordinates are fp64; values keep the data's dtype.  The 2-D data never
leaves the device: only the 1-D axes and the query points cross to the host.
"""
from collections.abc import Iterable

import numpy as np
import torch

from . import _capi as capi
from . import _ops
from .coordinates import cart_to_polar, interp_axes, polar_lattice_axes


def fix_interp_pair(x, y):
    """x, y with the same shape: a scalar is repeated for each value of the other (prysm/_richdata.py:11-38)."""
    if y is None:
        y = 0
    if x is None:
        x = 0
    if isinstance(x, Iterable) and not isinstance(y, Iterable):
        y = [y] * len(x)
    elif isinstance(y, Iterable) and not isinstance(x, Iterable):
        x = [x] * len(y)
    return x, y


def _device_data(data):
    data = _ops.asdevice(data)
    if not (data.is_floating_point() or data.is_complex()):
        data = data.to(torch.float64)
    return data.contiguous()


def _query(v):
    """a query coordinate (scalar, sequence, array or tensor) as a host fp64 array"""
    return np.asarray(_ops.asnumpy(v) if isinstance(v, torch.Tensor) else v, dtype=np.float64)


def _host_axes(x, y):
    """the 1-D axes of x, y (2-D grids give their first row / column) as host fp64 arrays"""
    if getattr(x, 'ndim', 1) == 2:
        x = x[0]
    if getattr(y, 'ndim', 1) == 2:
        y = y[:, 0]
    return _query(x).reshape(-1), _query(y).reshape(-1)


def _device_axes(xh, yh):
    xd, yd, _, _, _ = interp_axes(xh, yh)
    return xd, yd


def exact_xy(data, x, y, xq, yq):
    """data (on the axes of x, y) at the points (xq, yq) by linear interpolation; a point outside the axes raises
    scipy's ValueError before any launch.  0-d for scalar queries."""
    xq, yq = fix_interp_pair(xq, yq)
    xq, yq = np.broadcast_arrays(_query(xq), _query(yq))
    xh, yh = _host_axes(x, y)
    for dim, (ax, q) in enumerate(((yh, yq), (xh, xq))):
        if not np.logical_and(np.all(ax[0] <= q), np.all(q <= ax[-1])):
            raise ValueError(f'One of the requested xi is out of bounds in dimension {dim}')
    xd, yd = _device_axes(xh, yh)
    return _ops.interp2d_linear(_device_data(data), xd, yd, _ops.asdevice(xq), _ops.asdevice(yq)).reshape(xq.shape)


def exact_polar(data, x, y, rho, phi=None):
    """data at the polar points (rho, phi), x = rho cos phi and y = rho sin phi in fp64 on the host."""
    rho, phi = fix_interp_pair(rho, phi)
    rho, phi = _query(rho), _query(phi)
    return exact_xy(data, x, y, rho * np.cos(phi), rho * np.sin(phi))


def _check_1d_bounds(ax, q):
    """scipy.interpolate.interp1d's bounds error"""
    below, above = q < ax[0], q > ax[-1]
    if below.any():
        raise ValueError(f"A value ({q[np.argmax(below)]}) in x_new is below the interpolation range's minimum value "
                         f"({ax[0]}).")
    if above.any():
        raise ValueError(f"A value ({q[np.argmax(above)]}) in x_new is above the interpolation range's maximum value "
                         f"({ax[-1]}).")


def exact_x(data, x, y, xq):
    """data along the centre row (argmin |y|) at xq, linear between samples."""
    xh, yh = _host_axes(x, y)
    xq = _query(xq)
    _check_1d_bounds(xh, xq.reshape(-1))
    data = _device_data(data)
    xd, yd = _device_axes(xh, yh)
    c = int(np.argmin(np.abs(yh)))
    return _ops.interp2d_linear(data[c:c + 1], xd, yd[c:c + 1], _ops.asdevice(xq),
                                _ops.asdevice(np.full(xq.shape, yh[c])), ld=data.shape[1]).reshape(xq.shape)


def exact_y(data, x, y, yq):
    """data along the centre column (argmin |x|) at yq, linear between samples."""
    xh, yh = _host_axes(x, y)
    yq = _query(yq)
    _check_1d_bounds(yh, yq.reshape(-1))
    data = _device_data(data)
    xd, yd = _device_axes(xh, yh)
    c = int(np.argmin(np.abs(xh)))
    return _ops.interp2d_linear(data[:, c:c + 1], xd[c:c + 1], yd, _ops.asdevice(np.full(yq.shape, xh[c])),
                                _ops.asdevice(yq), ld=data.shape[1]).reshape(yq.shape)


class RichData:
    """Array plus its sample spacing and wavelength, with coordinates, slices and exact sampling."""
    _default_twosided = True

    def __init__(self, data, dx, wavelength):
        self.dx = dx
        self.wavelength = wavelength
        self._x = self._y = self._r = self._t = None
        self._data = None
        self.data = data

    @property
    def data(self):
        """Sampled data."""
        return self._data

    @data.setter
    def data(self, data):
        old_shape = None if self._data is None else tuple(self._data.shape)
        self._data = data
        if old_shape is not None and old_shape != tuple(data.shape):
            self._x = self._y = self._r = self._t = None

    @property
    def shape(self):
        return tuple(self.data.shape)

    @property
    def size(self):
        return int(np.prod(self.shape))

    def _grids(self):
        g = _ops.xy_grid(self.shape, self.dx, torch.float64, _ops.asdevice(self.data).device, want='xy')
        self._x, self._y = g['x'], g['y']

    @property
    def x(self):
        """X coordinates, 2-D fp64 (make_xy_grid)."""
        if self._x is None:
            self._grids()
        return self._x

    @x.setter
    def x(self, x):
        self._x = x
        self._r = self._t = None

    @property
    def y(self):
        """Y coordinates, 2-D fp64 (make_xy_grid)."""
        if self._y is None:
            self._grids()
        return self._y

    @y.setter
    def y(self, y):
        self._y = y
        self._r = self._t = None

    @property
    def r(self):
        """Radial coordinates, 2-D (cart_to_polar of x, y)."""
        if self._r is None:
            self._r, self._t = cart_to_polar(self.x, self.y)
        return self._r

    @r.setter
    def r(self, r):
        self._r = r

    @property
    def t(self):
        """Azimuthal coordinates, 2-D (cart_to_polar of x, y)."""
        if self._t is None:
            self._r, self._t = cart_to_polar(self.x, self.y)
        return self._t

    @t.setter
    def t(self, t):
        self._t = t

    @property
    def support_x(self):
        return float(self.shape[1] * self.dx)

    @property
    def support_y(self):
        return float(self.shape[0] * self.dx)

    @property
    def support(self):
        return max((self.support_x, self.support_y))

    def numpy(self):
        """Host copy of the data."""
        return _ops.asnumpy(self.data)

    def copy(self):
        return RichData(self.data.clone(), self.dx, self.wavelength)

    def slices(self, twosided=None):
        """Slices of the data through the centre and over azimuth (prysm/_richdata.py:166-187)."""
        if twosided is None:
            twosided = self._default_twosided
        return Slices(data=self.data, x=self.x[0], y=self.y[:, 0], twosided=twosided)

    def exact_polar(self, rho, phi=None):
        """Data at the polar points (rho, phi) (prysm/_richdata.py:234-254)."""
        return exact_polar(self.data, self.x, self.y, rho, phi)

    def exact_xy(self, x, y=None):
        """Data at the points (x, y) (prysm/_richdata.py:256-275)."""
        return exact_xy(self.data, self.x, self.y, x, y)

    def exact_x(self, x):
        """Data at x along the centre row (prysm/_richdata.py:277-292)."""
        return exact_x(self.data, self.x, self.y, x)

    def exact_y(self, y):
        """Data at y along the centre column (prysm/_richdata.py:294-309)."""
        return exact_y(self.data, self.x, self.y, y)


class Slices:
    """Slices of 2-D data: along the centre row and column, and statistics over azimuth on the polar lattice of
    uniform_cart_to_polar (prysm/_richdata.py:414-585).  The first azimuthal statistic read runs one kernel for count,
    mean, variance, min and max and keeps them; the median is computed when it is asked for."""

    def __init__(self, data, x, y, twosided=True):
        self._source = data
        self._x, self._y = x, y
        self._xh = np.asarray(_ops.asnumpy(x), dtype=np.float64)
        self._yh = np.asarray(_ops.asnumpy(y), dtype=np.float64)
        self.center_y, self.center_x = int(np.argmin(np.abs(self._yh))), int(np.argmin(np.abs(self._xh)))
        self.twosided = twosided
        self._polar = None          # (x axis, y axis, rmax) on the device
        self._r = self._p = None
        self._stats = None
        self._median = None

    def _lattice(self):
        if self._polar is None:
            xd, yd, rmax, _, _ = interp_axes(self._xh, self._yh)
            self._polar = (xd, yd, rmax)
            self._r, self._p = polar_lattice_axes(rmax, len(self._xh), len(self._yh))
        return self._polar

    def check_polar_calculated(self):
        """Set up the polar lattice (rho, phi); the polar plane itself is never formed."""
        self._lattice()

    def _stat(self, row):
        if len(self._yh) > capi.AZ_MAX_NY:
            raise ValueError(f'azimuthal statistics hold a column on chip: at most {capi.AZ_MAX_NY} phi samples (rows), '
                             f'got {len(self._yh)}')
        xd, yd, rmax = self._lattice()
        self._source = _device_data(self._source)
        if row == 5:
            if self._median is None:
                self._median = _ops.azimuthal_stats(self._source, xd, yd, rmax, capi.AZ_MEDIAN)[5]
            return self._r, self._median
        if self._stats is None:
            self._stats = _ops.azimuthal_stats(self._source, xd, yd, rmax,
                                               capi.AZ_COUNT | capi.AZ_MEAN | capi.AZ_VAR | capi.AZ_MIN | capi.AZ_MAX)
        return self._r, self._stats[row]

    @property
    def x(self):
        """(x, data along the centre row)."""
        if self.twosided:
            return self._x, self._source[self.center_y, :]
        return self._x[self.center_x:], self._source[self.center_y, self.center_x:]

    @property
    def y(self):
        """(y, data along the centre column)."""
        if self.twosided:
            return self._y, self._source[:, self.center_x]
        return self._y[self.center_y:], self._source[self.center_y:, self.center_x]

    @property
    def azavg(self):
        """(rho, mean over azimuth ignoring NaN)."""
        return self._stat(1)

    @property
    def azmedian(self):
        """(rho, median over azimuth ignoring NaN)."""
        return self._stat(5)

    @property
    def azmin(self):
        """(rho, minimum over azimuth ignoring NaN)."""
        return self._stat(3)

    @property
    def azmax(self):
        """(rho, maximum over azimuth ignoring NaN)."""
        return self._stat(4)

    @property
    def azpv(self):
        """(rho, max - min over azimuth)."""
        r, mx = self.azmax
        _, mn = self.azmin
        return r, mx - mn

    @property
    def azvar(self):
        """(rho, variance over azimuth ignoring NaN, ddof 0)."""
        return self._stat(2)

    @property
    def azstd(self):
        """(rho, standard deviation over azimuth ignoring NaN)."""
        r, v = self._stat(2)
        return r, v.sqrt()
