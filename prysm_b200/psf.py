"""PSF reductions on the path (reference prysm/psf.py:174-237)."""
from . import _ops


def centroid(data, dx=None, unit='spatial'):
    """Centre of mass; 'pixels' is corner indexed, 'spatial' = dx*(com - shape//2)
    (prysm/psf.py:174-203; scipy.ndimage.center_of_mass = first moments / sum)."""
    if not hasattr(data, 'ndim'):
        dx = data.dx if dx is None else dx
        data = data.data
    data = _ops.asdevice(data)
    s0, sy, sx = _ops.moments(data)
    com = (sy / s0, sx / s0)
    if unit != 'spatial':
        return com
    return tuple(dx * (c - s // 2) for c, s in zip(com, data.shape))


def autocrop(data, px):
    """Window of full width px around the centroid (prysm/psf.py:206-237); a view when it fits."""
    import torch
    data = _ops.asdevice(data)
    cy, cx = (int(c) for c in centroid(data, unit='pixels'))
    w = px // 2
    y0, x0 = cy - w, cx - w
    y1, x1 = y0 + px, x0 + px
    pad_y = (max(0, -y0), max(0, y1 - data.shape[0]))
    pad_x = (max(0, -x0), max(0, x1 - data.shape[1]))
    if any(pad_y) or any(pad_x):
        data = torch.nn.functional.pad(data, (pad_x[0], pad_x[1], pad_y[0], pad_y[1]))
        y0, y1, x0, x1 = y0 + pad_y[0], y1 + pad_y[0], x0 + pad_x[0], x1 + pad_x[0]
    return data[y0:y1, x0:x1]


FIRST_AIRY_ZERO = 1.220
SECOND_AIRY_ZERO = 2.233
THIRD_AIRY_ZERO = 3.238
FIRST_AIRY_ENCIRCLED = 0.8377850436212378
SECOND_AIRY_ENCIRCLED = 0.9099305350850819
THIRD_AIRY_ENCIRCLED = 0.9376474743695488

AIRYDATA = {
    1: (FIRST_AIRY_ZERO, FIRST_AIRY_ENCIRCLED),
    2: (SECOND_AIRY_ZERO, SECOND_AIRY_ENCIRCLED),
    3: (THIRD_AIRY_ZERO, THIRD_AIRY_ENCIRCLED)
}


def _size_level(metric):
    """(level, relative) of estimate_size's metric: a fraction of the polar maximum, or an absolute value."""
    import numbers
    import numpy as np
    name = metric.lower() if isinstance(metric, str) else None
    if name == 'fwhm':
        return 0.5, True
    if name == '1/e':
        return 1 / np.e, True
    if name == '1/e^2':
        return 1 / (np.e ** 2), True
    if isinstance(metric, numbers.Number):
        return float(metric), False
    raise ValueError('unknown metric, use fwhm, 1/e, or 1/e^2')


def estimate_size(data, metric, dx=None, x=None, y=None, criteria='last'):
    """The mean radius at which data falls through `metric` ('fwhm', '1/e', '1/e^2' of the maximum, or a value) along
    the rays of uniform_cart_to_polar's lattice, at the first or last crossing of each ray (prysm/psf.py:27-90).  One
    call of four kernels; only the count and the mean come back to the host.  x, y are the 1-D axes (fftrange * dx in
    fp64 when not given)."""
    import numpy as np
    import torch
    from .coordinates import interp_axes
    criteria = criteria.lower()
    level, relative = _size_level(metric)
    if criteria not in ('first', 'last'):
        raise ValueError('unknown criteria, use first or last')
    if not hasattr(data, 'ndim'):
        data = data.data
    data = _ops.asdevice(data)
    if data.dtype not in (torch.float32, torch.float64):
        data = data.to(torch.float64)
    if x is None and y is None:
        y, x = ((np.arange(s, dtype=np.float64) - s // 2) * dx for s in data.shape)
    if getattr(x, 'ndim', 1) == 2:
        x = x[0]
    if getattr(y, 'ndim', 1) == 2:
        y = y[:, 0]
    xd, yd, rmax, _, _ = interp_axes(x, y)
    count, mean = _ops.polar_crossings(data, xd, yd, rmax, level, relative, criteria == 'last')
    if count == 0:
        raise ValueError('metric does not cross the sampled data')
    return np.float64(mean)


def fwhm(data, dx=None, x=None, y=None, criteria='last'):
    """Full width at half maximum: twice estimate_size(metric='fwhm') (prysm/psf.py:93-117)."""
    return estimate_size(x=x, y=y, dx=dx, data=data, metric='fwhm', criteria=criteria) * 2


def one_over_e(data, dx=None, x=None, y=None, criteria='last'):
    """1/e diameter (prysm/psf.py:120-144)."""
    return estimate_size(x=x, y=y, dx=dx, data=data, metric='1/e', criteria=criteria) * 2


def one_over_e_sq(data, dx=None, x=None, y=None, criteria='last'):
    """1/e^2 diameter (prysm/psf.py:147-171)."""
    return estimate_size(x=x, y=y, dx=dx, data=data, metric='1/e^2', criteria=criteria) * 2


def analytic(kind, v, a, b):
    """One analytic radial function (pb_analytic_radial) of v, a number, sequence, array or tensor, in fp64 stored at
    config precision; a number gives a float."""
    import numbers
    import torch
    from .conf import config
    if isinstance(v, numbers.Number):
        out = _ops.analytic_radial(kind, _ops.asdevice([float(v)]), a, b, torch.float64)
        return float(out[0])
    return _ops.analytic_radial(kind, _ops.asdevice(v), a, b, config.real_dtype)


def airydisk(unit_r, fno, wavelength):
    """|2 jinc(pi r / (wavelength fno))|^2 (prysm/psf.py:240-259), one kernel."""
    from . import _capi
    return analytic(_capi.AR_AIRYDISK, unit_r, wavelength, fno)


def airydisk_efield(unit_r, fno, wavelength):
    """2 jinc(pi r / (wavelength fno)) (prysm/psf.py:262-265), one kernel."""
    from . import _capi
    return analytic(_capi.AR_AIRYDISK_EFIELD, unit_r, wavelength, fno)


def airydisk_ft(r, fno, wavelength):
    """The Fourier transform of the Airy disk, (2 / pi)(acos s - s sqrt(1 - s^2)) with s = |r| wavelength fno clamped
    at 1 (prysm/psf.py:268-292), one kernel."""
    from . import _capi
    return analytic(_capi.AR_AIRYDISK_FT, r, wavelength, fno)
