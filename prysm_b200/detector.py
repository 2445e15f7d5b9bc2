"""Detector sampling at the end of the image chain (reference prysm/detector.py): binning to detector pixels, its
adjoint, the analytic pixel / optical-low-pass-filter transfer functions that `apply_transfer_functions` consumes, the
pixel footprint, lookup tables, and `Detector.expose`, which turns an aerial image into camera frames with shot and read
noise on the device."""
import numbers

import numpy as np
import torch

from . import _ops


def _factors(factor, ndim=2):
    if isinstance(factor, numbers.Number):
        return (int(factor),) * ndim
    f = tuple(int(v) for v in factor)
    if len(f) != ndim:
        raise ValueError(f'factor must have {ndim} entries for a {ndim}-D array')
    return f


def _lut_overflow(code, lut):
    return IndexError(f'index {code} is out of bounds for axis 0 with size {lut.numel()}')


def apply_lut(img, lut):
    """np.take(lut, img) for an image of an unsigned integer dtype (prysm/detector.py:8-26): one gather kernel.  A table
    shorter than the image dtype's range is checked, and a code past its end raises IndexError as np.take does."""
    img = _ops.asdevice(img)
    lut = _ops.asdevice(lut).reshape(-1)
    if img.dtype not in (torch.uint8, torch.uint16, torch.uint32):
        raise TypeError(f'apply_lut takes an image of an unsigned integer dtype, got {img.dtype}')
    check = lut.numel() < 2 ** (8 * img.element_size())
    out, bad = _ops.apply_lut(img, lut, check)
    if bad is not None:
        raise _lut_overflow(bad, lut)
    return out


def _code_dtype(bits):
    if bits <= 8:
        return torch.uint8
    if bits <= 16:
        return torch.uint16
    if bits <= 32:
        return torch.uint32
    raise ValueError("numpy's random functionality is inadequate for > 32 unsigned bits")


class Detector:
    """Model of a detector (prysm/detector.py:29-148)."""

    def __init__(self, dark_current, read_noise, bias, fwc, conversion_gain, bits, exposure_time, prnu=None, dcnu=None,
                 lut=None):
        """dark_current e-/s; read_noise e- (Gaussian sigma); bias e-; fwc e- (full well); conversion_gain e-/DN; bits of
        the ADC; exposure_time s; prnu / dcnu: optional maps the light / the dark current are multiplied by (broadcast
        against the image); lut: optional table of output DN by ideal DN."""
        self.dark_current = dark_current
        self.read_noise = read_noise
        self.bias = bias
        self.fwc = fwc
        self.conversion_gain = conversion_gain
        self.bits = bits
        self.exposure_time = exposure_time
        self.prnu = prnu
        self.dcnu = dcnu
        self.lut = lut

    def expose(self, aerial_img, frames=1):
        """Frames of the aerial image (e-/s, QE included), shape (frames, *aerial_img.shape), squeezed when frames == 1;
        uint8 / uint16 / uint32 DN by `bits` (or the LUT's dtype).  One kernel draws every frame: per pixel
        lam = aerial t [* prnu] + dark t [* dcnu], shot noise ~ Poisson(lam) (exact), read noise ~ N(0, read_noise),
        then bias, the full well, the gain and the ADC range, as the reference does.

        The random numbers are the engine's own (Philox4x32-10): equal to the reference's in distribution, not sample
        for sample.  The key of each call is drawn from numpy's global `np.random` state, so `np.random.seed(s)`
        makes runs reproducible and successive calls differ.  The call reads the kernel's error flags back, its only
        synchronisation; it cannot be captured into a CUDA graph, whose replays would repeat the same noise."""
        if torch.cuda.is_available() and torch.cuda.is_current_stream_capturing():
            raise RuntimeError('Detector.expose cannot be captured into a CUDA graph: its random key comes from the '
                               'host, so every replay would repeat the same noise')
        code = _code_dtype(self.bits)
        if self.read_noise < 0:
            raise ValueError('scale < 0')
        frames = int(frames)
        aerial = _ops.asdevice(aerial_img)
        maps = [None if m is None else _ops.asdevice(m) for m in (self.prnu, self.dcnu)]
        dt = aerial.dtype if aerial.is_floating_point() else torch.float64
        for m in maps:
            if m is not None:
                dt = torch.promote_types(dt, m.dtype if m.is_floating_point() else torch.float64)
        if dt not in (torch.float32, torch.float64):
            dt = torch.float64
        aerial = aerial.to(dt).contiguous()
        maps = [None if m is None else m.to(dt) for m in maps]
        lut = None if self.lut is None else _ops.asdevice(self.lut).reshape(-1)
        t = float(self.exposure_time)
        params = [t, float(self.dark_current) * t, float(self.read_noise), float(self.bias), float(self.fwc),
                  1 / self.conversion_gain, float(2 ** self.bits - 1)]
        lo, hi = (int(v) for v in np.random.randint(0, 2 ** 32, size=2, dtype=np.uint64))
        key = hi << 32 | lo
        key = key - 2 ** 64 if key >= 2 ** 63 else key
        out, flags = _ops.expose(aerial, maps[0], maps[1], params, frames, key, code, lut)
        if flags[0] & 2:
            raise ValueError('lam value too large')
        if flags[0] & 1:
            raise ValueError('lam < 0 or lam is NaN')
        if flags[0] & 4:
            raise _lut_overflow(flags[1], lut)
        return out[0] if frames == 1 else out


def pixel(x, y, width_x, width_y):
    """Spatial representation of a pixel (prysm/detector.py:197-219): the boolean (x <= wx/2) & (x >= -wx/2) &
    (y <= wy/2) & (y >= -wy/2), with the half widths rounded to the coordinates' dtype as numpy compares them."""
    x = _ops.asdevice(x)
    y = _ops.asdevice(y)
    dt = torch.promote_types(x.dtype, y.dtype)
    if dt not in (torch.float32, torch.float64):
        dt = torch.float64
    x, y = x.to(dt), y.to(dt)
    npdt = np.float32 if dt == torch.float32 else np.float64

    def half(w):
        w = w / 2
        return float(np.asarray(w, dtype=np.result_type(npdt, w)))
    return _ops.pixel(x, y, half(width_x), half(width_y))


def bindown(array, factor, mode='avg'):
    """Bin a 2-D array by `factor` (int or (fy, fx)); the shape must be an integer multiple (prysm/detector.py:222-274)."""
    if mode.lower() in ('avg', 'average', 'mean'):
        mean = True
    elif mode.lower() == 'sum':
        mean = False
    else:
        raise ValueError('mode must be average or sum.')
    fy, fx = _factors(factor)
    return _ops.bindown(array, fy, fx, mean)


def tile(array, factor, scaling='sum'):
    """Repeat every sample `factor` times per axis -- the adjoint of bindown (prysm/detector.py:277-338)."""
    fy, fx = _factors(factor)
    if scaling == 'sum':
        sf = 1 / (fy * fx)
    elif scaling in ('avg', 'average', 'mean'):
        sf = 1
    else:
        raise ValueError('scaling must be average or sum')
    return _ops.tile(array, fy, fx, sf)


def pixel_ft(fx, fy, width_x, width_y):
    """sinc(fx wx) sinc(fy wy) on broadcastable frequency vectors fx (1, N), fy (M, 1) (prysm/detector.py:174-194)."""
    return _ops.separable_tf(0, fx, fy, width_x, width_y)


def olpf_ft(fx, fy, width_x, width_y):
    """cos(2 wx fx) cos(2 wy fy) (prysm/detector.py:151-171)."""
    return _ops.separable_tf(1, fx, fy, width_x, width_y)
