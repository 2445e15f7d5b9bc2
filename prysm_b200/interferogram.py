"""Interferometric metrology on the device (reference prysm/interferogram.py, the random surfaces, PSD fits, Zygo I/O
and plotting excepted).

A measured or simulated map that is already a CUDA tensor stays on the device through the whole chain: its statistics,
tilt and power removal, PVr, PSD, band-limited RMS, filtering and slopes.  What comes back to the host is scalars
(statistics, fit coefficients, the four crop indices) and the 1-D frequency axes.  The reference's quirks are kept
(SURVEY Appendix B): fit_plane has no piston term, fit_sphere fits on linspace(-1, 1) axes whatever dx is,
bandlimited_rms takes one spacing from the y axis, std is the population std and rms is about zero.
"""
import warnings

import numpy as np
import torch

from . import _capi as capi
from . import _ops
from ._richdata import RichData
from .polynomials import fringe_to_nm, lstsq, solve_gram
from .util import mean, nan_stats, pv, rms, Sa, std  # noqa: F401

HeNe = 0.6328
_FILTERS = {'lp': capi.FILT_LOWPASS, 'lowpass': capi.FILT_LOWPASS, 'hp': capi.FILT_HIGHPASS,
            'highpass': capi.FILT_HIGHPASS, 'bp': capi.FILT_BANDPASS, 'bandpass': capi.FILT_BANDPASS,
            'br': capi.FILT_BANDREJECT, 'bandreject': capi.FILT_BANDREJECT}


def _real(a):
    a = _ops.asdevice(a)
    if a.dtype not in (torch.float32, torch.float64):
        a = a.to(torch.float64)
    return a


def _item(t, idx):
    return float(t[idx].item())


def _check_bool_index(shape, mask_shape):
    """numpy's IndexError for a boolean mask (the reference's `data[mask]`, `work[r < flow]`) of another shape"""
    if tuple(mask_shape) == tuple(shape):
        return
    if len(mask_shape) > len(shape):
        raise IndexError(f'too many indices for array: array is {len(shape)}-dimensional, but {len(mask_shape)} were '
                         'indexed')
    ax = next((i for i, (a, b) in enumerate(zip(shape, mask_shape)) if a != b), None)
    if ax is None:
        raise ValueError(f'a mask of shape {tuple(mask_shape)} selects whole rows; the engine takes one of the data '
                         f'shape {tuple(shape)}')
    raise IndexError(f'boolean index did not match indexed array along axis {ax}; size of axis is {shape[ax]} but size '
                     f'of corresponding boolean axis is {mask_shape[ax]}')


def _rmax_square_array(r):
    """r[ny - 1, nx // 2], the radius pvr and window_2d_welch normalise by"""
    return _item(r, (r.shape[0] - 1, r.shape[1] // 2))


def fit_plane(x, y, z):
    """The least-squares plane c0 x + c1 y through the finite samples of z (no piston term)."""
    z = _real(z)
    x, y = _ops.asdevice(x), _ops.asdevice(y)
    c = lstsq([x, y], z)
    return _ops.metro_pointwise(capi.PW_AXPBY, u=x, v=y, a=c[0], b=c[1], dtype=z.dtype)


def _sphere_coefs(z):
    """(rho^2 on linspace(-1, 1) axes, the coefficients of the fit of [rho^2, 1] to the finite samples of z)"""
    ny, nx = z.shape
    rho2 = _ops.metro_pointwise(capi.PW_RHO2, shape=(ny, nx), dtype=z.dtype, a=2.0 / (nx - 1) if nx > 1 else 0.0,
                                b=2.0 / (ny - 1) if ny > 1 else 0.0)
    return rho2, lstsq([rho2, None], z)


def fit_sphere(z):
    """(finite mask, c0 rho^2 at the finite samples) of the fit of [rho^2, 1] on linspace(-1, 1) axes."""
    z = _real(z)
    rho2, c = _sphere_coefs(z)
    pts = torch.isfinite(z)
    return pts, _ops.metro_pointwise(capi.PW_AXPBY, u=rho2, a=c[0])[pts]


def _corners(shape):
    """the four 2 % corner rectangles of make_window's automatic choice, with numpy's slice semantics"""
    ny, nx = shape
    ys, xs = int(round(ny * 0.02, 0)), int(round(nx * 0.02, 0))
    out = []
    for sy in (slice(None, ys), slice(-ys, None)):
        for sx in (slice(None, xs), slice(-xs, None)):
            y0, y1, _ = sy.indices(ny)
            x0, x1, _ = sx.indices(nx)
            out += [y0, max(y0, y1), x0, max(x0, x1)]
    return out


def _window_args(shape, dx, which, alpha):
    """(kind, user array, rmax, corners) of pb_psd_prologue for make_window's `which`"""
    ny, nx = shape
    rmax = abs((ny - 1 - ny // 2) * dx)       # r[ny - 1, nx // 2] of the fftrange * dx grid
    if which is None:
        return capi.WIN_AUTO, None, rmax, _corners(shape)
    if type(which) is str:
        wl = which.lower()
        if wl == 'welch':
            return capi.WIN_WELCH, None, rmax, None
        if wl in ('hann', 'hanning'):
            return capi.WIN_HANN, None, rmax, None
        raise ValueError('unknown window type')
    return capi.WIN_USER, _ops.asdevice(which), rmax, None


def make_window(signal, dx, which=None, alpha=4):
    """The PSD window: Welch (alpha), Hann, or with which=None Welch when the four 2 % corners of signal are all
    == 0 and Hann otherwise, decided on the device.  An array `which` is returned as given."""
    signal = _real(signal)
    kind, user, rmax, corners = _window_args(signal.shape, dx, which, alpha)
    if kind == capi.WIN_USER:
        return which
    _, w, _ = _ops.psd_prologue(signal, kind, None, dx, alpha, rmax, corners, want_shifted=False, want_window=True)
    return w


def _ft_axes(dx, shape, dev):
    """the fp64 forward_ft_unit axes (ux, uy) on the host and on the device"""
    ny, nx = shape
    ux = np.fft.fftshift(np.fft.fftfreq(nx, dx))
    uy = np.fft.fftshift(np.fft.fftfreq(ny, dx))
    return ux, uy, _ops.asdevice(ux).to(dev), _ops.asdevice(uy).to(dev)


def _psd_data(height, dx, window=None):
    """psd without the 2-D axes: (psd, ux, uy, ux_dev, uy_dev).  Launches: the window prologue (one more for the
    automatic choice), pb_fft2, the epilogue."""
    height = _real(height)
    kind, user, rmax, corners = _window_args(height.shape, dx, window, 4)
    shifted, _, s2 = _ops.psd_prologue(height, kind, user, dx, 4, rmax, corners)
    F = _ops.fft2(shifted)
    out = _ops.psd_epilogue(F, s2, 1 / dx)
    ux, uy, uxd, uyd = _ft_axes(dx, height.shape, out.device)
    return out, ux, uy, uxd, uyd


def psd(height, dx, window=None):
    """(ux, uy, psd): the power spectral density ifftshift(fft2(fftshift(height w))) |.|^2 / (sum w^2 fs^2) on the 2-D
    frequency grids.  Any NaN in height makes every sample NaN."""
    out, _, _, uxd, uyd = _psd_data(height, dx, window)
    ny, nx = out.shape
    return uxd[None, :].expand(ny, nx), uyd[:, None].expand(ny, nx), out


def _band_limits(rmax, wllow, wlhigh, flow, fhigh):
    """(flow, fhigh) with the reference's precedence and warnings (prysm/interferogram.py:214-241)"""
    default_max = rmax
    if wllow is not None or wlhigh is not None:
        if wllow is None:
            flow = 0
        else:
            fhigh = 1 / wllow
        if wlhigh is None:
            fhigh = default_max()
        else:
            flow = 1 / wlhigh
    elif flow is not None or fhigh is not None:
        if flow is None:
            flow = 0
        if fhigh is None:
            fhigh = default_max()
    else:
        raise ValueError('must specify either period (wavelength) or frequency')
    if flow is None:
        warnings.warn('no lower limit given, using 0 for low frequency')
        flow = 0
    if fhigh is None:
        warnings.warn('no upper limit given, using limit imposed by data.')
        fhigh = default_max()
    return flow, fhigh


def bandlimited_rms(r, psd, wllow=None, wlhigh=None, flow=None, fhigh=None):
    """The RMS of the band flow <= r <= fhigh of a PSD: the trapezoid over both axes with one spacing, taken from r
    at the centre and at the centre row - 1 (the y spacing), for both."""
    r, psd = _real(r), _real(psd)
    _check_bool_index(psd.shape, r.shape)
    flow, fhigh = _band_limits(lambda: float(nan_stats(r)[3]), wllow, wlhigh, flow, fhigh)
    if r.ndim == 2:
        c0, c1 = r.shape[0] // 2, r.shape[1] // 2
        dx = abs(_item(r, (c0 - 1, c1)) - _item(r, (c0, c1)))
    else:
        c = r.shape[0] // 2
        dx = abs(_item(r, c - 1) - _item(r, c))
    s = _ops.band_trapz(psd, r=r, flow=flow, fhigh=fhigh)
    return float(np.sqrt(s * dx * dx if r.ndim == 2 else s * dx))


def window_2d_welch(r, alpha=8):
    """1 - |r / rmax|^alpha, rmax = r[ny - 1, nx // 2]; negative in the corners."""
    r = _real(r)
    return _ops.metro_pointwise(capi.PW_WELCH, x=r, a=_rmax_square_array(r), b=alpha)


def hann2d(M, N):
    """Hann window in 2-D: cos(pi / min(M, N) * hypot(n, m))^2, zero beyond min(M, N) // 2."""
    from .conf import config
    dtype = _ops.torch_dtype(config.precision)
    return _ops.filter_h((M, N), capi.FILT_W, dtype, _ops.device())[0]


def ideal_lpf_iir2d(r, dx, fc_over_nyq):
    """Ideal impulse response of a 2-D low-pass filter, jinc(r pi fc / dx) fc^2 pi / 2."""
    r = _real(r)
    return _ops.filter_h(r.shape, capi.FILT_H, r.dtype, r.device, r=r, dx=dx, fcn0=fc_over_nyq)[0]


def _filter_type(typ):
    tl = typ.lower()
    if tl not in _FILTERS:
        raise ValueError(f"unknown filter type {typ!r}: one of 'lowpass', 'lp', 'highpass', 'hp', 'bandpass', 'bp', "
                         "'bandreject', 'br'")
    return _FILTERS[tl]


def _filter_transforms(r, dx, fc, ftyp, dtype):
    """(Hl, Hh): the unshifted transforms of hann2d * the ideal low-pass response at the one or two cut-offs, formed
    at the real dtype"""
    nyq = 1 / (2 * dx)
    two = ftyp in (capi.FILT_BANDPASS, capi.FILT_BANDREJECT)
    f0, f1 = (fc[0] / nyq, fc[1] / nyq) if two else (fc / nyq, None)
    h0, h1 = _ops.filter_h(r.shape, capi.FILT_W | capi.FILT_H, dtype, r.device, r=r, dx=dx, fcn0=f0, fcn1=f1)
    return _ops.fft2(h0), (_ops.fft2(h1) if two else None)


def designfilt2d(r, dx, fc, typ='lowpass'):
    """The rotationally symmetric transfer function H = |fft2(hann2d h)| (unshifted) combined by typ."""
    ftyp = _filter_type(typ)
    r = _real(r)
    Hl, Hh = _filter_transforms(r, dx, fc, ftyp, r.dtype)
    return _ops.filter_apply(ftyp, Hl, Hh)


class Interferogram(RichData):
    """A phase map with the metrology of prysm's Interferogram; methods change `data` and return self."""

    def __init__(self, phase, dx=0, wavelength=HeNe, intensity=None, meta=None):
        if not wavelength:
            if meta:
                wavelength = meta.get('wavelength', None)
                if wavelength is None:
                    wavelength = meta.get('Wavelength')
                if wavelength is not None:
                    wavelength *= 1e6
        super().__init__(data=_real(phase), dx=dx, wavelength=wavelength)
        self.intensity = intensity
        self.meta = meta
        self._latcaled = dx != 0

    @property
    def dropout_percentage(self):
        """Percentage of the samples that are NaN."""
        return float(nan_stats(self.data)[5] / self.data.numel() * 100)

    @property
    def pv(self):
        """Peak-to-valley of the finite samples (DIN/ISO St)."""
        return pv(self.data)

    @property
    def rms(self):
        """RMS about zero of the finite samples (DIN/ISO Sq)."""
        return rms(self.data)

    @property
    def Sa(self):
        """Mean absolute deviation from the mean (DIN/ISO Sa)."""
        return Sa(self.data)

    @property
    def strehl(self):
        """Strehl ratio exp(-(2 pi std / wavelength)^2), the data in nm and the wavelength in um."""
        wvl = self.wavelength * 1e3
        return float(np.exp(-(2 * np.pi * std(self.data) / wvl) ** 2))

    @property
    def std(self):
        """Population standard deviation of the finite samples."""
        return std(self.data)

    def pvr(self, normalization_radius=None):
        """Peak-to-valley residual (C. Evans, OF&T 2008, OWA4): pv of a 36-term Fringe Zernike fit plus 3 times the
        RMS of its residual, inside r <= normalization_radius (default r[ny - 1, nx // 2], square data only)."""
        r, t = self.r, self.t
        if normalization_radius is None:
            if self.shape[0] != self.shape[1]:
                raise ValueError('pvr: if normalization_radius is None, data must be square')
            normalization_radius = _rmax_square_array(r)
        d = self.data
        rn = _ops.metro_pointwise(capi.PW_DIV, x=r, a=normalization_radius)
        data = _ops.metro_pointwise(capi.PW_RADIUS, x=d, u=rn, a=1.0)
        nms = [fringe_to_nm(j) for j in range(1, 38)]
        basis = _ops.zernike_seq(nms, rn, t, norm=False, polar=True).to(d.dtype)
        coefs = solve_gram(_ops.masked_gram([basis[k].reshape(-1) for k in range(len(nms))], data.reshape(-1)),
                           len(nms))
        projected = _ops.weighted_sum(basis, coefs)
        _ops.metro_pointwise(capi.PW_RADIUS, x=projected, u=rn, a=1.0, out=projected)
        fit_err = _ops.metro_pointwise(capi.PW_SUB, x=data, u=projected, a=1.0)
        return pv(projected) + 3 * rms(fit_err)

    def _set(self, data):
        self.data = data
        return self

    def fill(self, _with=0):
        """Replace NaN samples with `_with`."""
        return self._set(_ops.metro_pointwise(capi.PW_FILL, x=self.data, a=_with, out=self.data))

    def crop(self):
        """Crop to the rectangle bounding the finite samples."""
        left, right, top, bottom = _ops.finite_bounds(self.data)
        if left == right == top == bottom == 0:
            return self
        ny, nx = self.shape
        lr, tb = slice(left, ny - right), slice(top, nx - bottom)
        xy = None if self._x is None else (self.x[lr, tb], self.y[lr, tb])
        rt = None if self._r is None else (self.r[lr, tb], self.t[lr, tb])
        self.data = self.data[lr, tb].contiguous()
        if xy is not None:
            self.x, self.y = (a.contiguous() for a in xy)
        if rt is not None:
            self.r, self.t = (a.contiguous() for a in rt)
        return self

    def recenter(self):
        """Shift x and y so that the sample at (ny // 2, nx // 2) is at the origin."""
        c = tuple(s // 2 for s in self.shape)
        x, y = self.x, self.y
        self.x = _ops.metro_pointwise(capi.PW_SUB, x=x, a=_item(x, c))
        self.y = _ops.metro_pointwise(capi.PW_SUB, x=y, a=_item(y, c))
        self._r = self._t = None
        return self

    def remove_piston(self):
        """Subtract the mean of the finite samples."""
        return self._set(_ops.metro_pointwise(capi.PW_SUB, x=self.data, a=mean(self.data), out=self.data))

    def remove_tiptilt(self):
        """Subtract the least-squares plane c0 x + c1 y."""
        x, y = self.x, self.y
        c = lstsq([x, y], self.data)
        return self._set(_ops.metro_pointwise(capi.PW_SUB, x=self.data, u=x, v=y, a=c[0], b=c[1], out=self.data))

    def remove_power(self):
        """Subtract c0 rho^2 of the fit of [rho^2, 1] on linspace(-1, 1) axes."""
        rho2, c = _sphere_coefs(self.data)
        return self._set(_ops.metro_pointwise(capi.PW_SUB, x=self.data, u=rho2, a=c[0], out=self.data))

    def mask(self, mask):
        """Set the samples where mask is False to NaN."""
        m = _ops.asdevice(mask)
        _check_bool_index(self.shape, m.shape)
        return self._set(_ops.metro_pointwise(capi.PW_KEEP, x=self.data, m=m, out=self.data))

    def strip_latcal(self):
        """Revert to pixels: dx = 1 and fresh x, y."""
        self.dx = 1.
        g = _ops.xy_grid(self.shape, self.dx, torch.float64, self.data.device, want='xy')
        self.x, self.y = g['x'], g['y']
        self._latcaled = False
        return self

    def latcal(self, plate_scale):
        """Lateral calibration: pixels of `plate_scale` (unit)s."""
        self.strip_latcal()
        self.x = _ops.metro_pointwise(capi.PW_AXPBY, u=self.x, a=plate_scale)
        self.y = _ops.metro_pointwise(capi.PW_AXPBY, u=self.y, a=plate_scale)
        self.dx = plate_scale
        self._latcaled = True
        return self

    def pad(self, value=np.nan, *, samples=None, shape=None):
        """Pad to `shape`, or by `samples`, filling with value; then latcal(dx)."""
        from .fttools import pad2d
        if samples is None and shape is None:
            raise ValueError('Neither samples nor shape specified')
        if samples is not None and shape is not None:
            raise ValueError('Both sampels and shape provided: only one can be given')
        if samples is not None:
            if isinstance(samples, int):
                samples = (samples, samples)
            shape = tuple(s + p for s, p in zip(self.shape, samples))
        self.data = pad2d(self.data, value=value, out_shape=shape)
        return self.latcal(self.dx)

    def spike_clip(self, nsigma=3):
        """Set to NaN the samples with |x| > nsigma * std."""
        thr = nsigma * self.std
        return self._set(_ops.metro_pointwise(capi.PW_CLIP, x=self.data, a=thr, out=self.data))

    def psd(self):
        """The PSD as a RichData on the frequency grids, one-sided slices by default."""
        out, _, _, uxd, uyd = _psd_data(self.data, self.dx)
        ny, nx = out.shape
        p = RichData(out, 0, self.wavelength)
        p.x = uxd[None, :].expand(ny, nx)
        p.y = uyd[:, None].expand(ny, nx)
        p.dx = np.zeros(nx)             # ux[1] - ux[0] of the 2-D grid, as the reference sets it
        p._default_twosided = False
        return p

    def filter(self, fc, typ='lowpass'):
        """Filter with designfilt2d(self.r, self.dx, fc, typ): the real part of ifft2(fft2(data) H)."""
        ftyp = _filter_type(typ)
        Hl, Hh = _filter_transforms(self.r, self.dx, fc, ftyp, self.data.dtype)
        D = _ops.filter_apply(ftyp, Hl, Hh, D=_ops.fft2(self.data))
        ny, nx = self.shape
        out = _ops.fft2(D, dir=+1, scale=1.0 / (ny * nx))
        return self._set(_ops.metro_pointwise(capi.PW_REAL, x=torch.view_as_real(out), shape=(ny, nx),
                                              dtype=self.data.dtype))

    def bandlimited_rms(self, wllow=None, wlhigh=None, flow=None, fhigh=None):
        """The band-limited RMS from the PSD, r = hypot of the frequency axes taken on the fly."""
        out, ux, uy, uxd, uyd = _psd_data(self.data, self.dx)
        ny, nx = out.shape
        flow, fhigh = _band_limits(lambda: float(np.hypot(np.abs(ux).max(), np.abs(uy).max())),
                                   wllow, wlhigh, flow, fhigh)
        dx = abs(float(np.hypot(ux[nx // 2], uy[ny // 2 - 1])) - float(np.hypot(ux[nx // 2], uy[ny // 2])))
        s = _ops.band_trapz(out, fx=uxd, fy=uyd, flow=flow, fhigh=fhigh)
        return float(np.sqrt(s * dx * dx))

    def total_integrated_scatter(self, wavelength, incident_angle=0):
        """TIS = 1 - exp(-(4 pi cos(angle) blr / wavelength)^2), the band up to 1000 / wavelength (um to mm)."""
        upper_limit = 1000 / wavelength
        kernel = 4 * np.pi * np.cos(np.radians(incident_angle))
        kernel *= self.bandlimited_rms(fhigh=upper_limit) / wavelength
        return 1 - np.exp(-kernel ** 2)

    def slope(self):
        """(x slope, y slope, their hypot) as RichData, np.gradient(data, dx)."""
        gx, gy, gr = _ops.gradient2d(self.data, self.dx)
        return RichData(gx, self.dx, None), RichData(gy, self.dx, None), RichData(gr, self.dx, None)
