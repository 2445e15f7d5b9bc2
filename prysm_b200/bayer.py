"""Bayer colour-filter-array operations on the device (reference prysm/bayer.py): white balance in place, interleaving
and de-interleaving colour planes, de-interlace and Malvar-He-Cutler demosaicing, and the assembly of super-resolved
colour planes.  Shapes follow numpy's slicing of the reference exactly, odd sides included."""
import numpy as np
import torch

from . import _ops
from .conf import config

top_left = (slice(0, None, 2), slice(0, None, 2))
top_right = (slice(0, None, 2), slice(1, None, 2))
bottom_left = (slice(1, None, 2), slice(0, None, 2))
bottom_right = (slice(1, None, 2), slice(1, None, 2))

ErrBadCFA = NotImplementedError('only rggb, bggr bayer patterns currently implemented')

# The 5x5 filters of Malvar, He & Cutler (ICASSP 2004, fig. 2), times 8; csrc/sensor.cu holds the same taps.  Each is
# symmetric under a 180-degree rotation, so convolving and correlating with it agree.
MALVAR_KERNELS = {
    'G_at_R_or_B': np.array([[0, 0, -1, 0, 0], [0, 0, 2, 0, 0], [-1, 2, 4, 2, -1], [0, 0, 2, 0, 0], [0, 0, -1, 0, 0]],
                            dtype=np.float64),
    'R_at_G_in_RB': np.array([[0, 0, .5, 0, 0], [0, -1, 0, -1, 0], [-1, 4, 5, 4, -1], [0, -1, 0, -1, 0],
                              [0, 0, .5, 0, 0]]),
    'R_at_G_in_BR': np.array([[0, 0, -1, 0, 0], [0, -1, 4, -1, 0], [.5, 0, 5, 0, .5], [0, -1, 4, -1, 0],
                              [0, 0, -1, 0, 0]]),
    'R_at_B_in_BB': np.array([[0, 0, -1.5, 0, 0], [0, 2, 0, 2, 0], [-1.5, 0, 6, 0, -1.5], [0, 2, 0, 2, 0],
                              [0, 0, -1.5, 0, 0]]),
}


def _bggr(cfa):
    if cfa == 'rggb':
        return False
    if cfa == 'bggr':
        return True
    raise ErrBadCFA


def _sites(values, bggr):
    """(r, g1, g2, b)-ordered values -> the order of the CFA sites top-left, top-right, bottom-left, bottom-right."""
    r, g1, g2, b = values
    return [b, g1, g2, r] if bggr else [r, g1, g2, b]


def _float_device(a, name):
    """The device tensor a white balance scales in place, and the numpy array to write back into (or None)."""
    host = a if isinstance(a, np.ndarray) else None
    t = _ops.asdevice(a)
    if not t.is_floating_point():
        raise TypeError(f'{name} must have a float dtype to be scaled in place, got {t.dtype}')
    if host is None and not t.is_contiguous():
        raise ValueError(f'{name} must be contiguous to be scaled in place')
    if t.dtype not in (torch.float32, torch.float64):
        raise TypeError(f'{name} must be float32 or float64, got {t.dtype}')
    return t, host


def _saturation(saturation, count):
    if saturation is None:
        raise ValueError('When doing safe WB prescaling, saturation must be not-none')
    if not hasattr(saturation, '__iter__'):
        saturation = [saturation] * count
    else:
        saturation = list(saturation)
        if len(saturation) != count:
            raise ValueError(f"saturation must be scalar or contain {('four', 'three')[count == 3]} values")
    if any(s <= 0 for s in saturation):
        raise ValueError('saturation must be positive')
    return [float(s) for s in saturation]


def _empty_plane():
    return ValueError('zero-size array to reduction operation maximum which has no identity')


def wb_prescale(mosaic, wr, wg1, wg2, wb, cfa='rggb', safe=False, saturation=None):
    """White-balance prescaling of an (m, n) float mosaic in place (prysm/bayer.py).  A device tensor is scaled where
    it is; a numpy array is scaled on the device and written back.  safe=True reduces every gain by
    max(1, max_p(max(plane p) gain_p / saturation_p)), with the maxima and the ratio computed on the device."""
    cfa = cfa.lower()
    sat = _saturation(saturation, 4) if safe else None
    bggr = _bggr(cfa)
    t, host = _float_device(mosaic, 'mosaic')
    if t.ndim != 2:
        raise ValueError(f'mosaic must be 2-D, got shape {tuple(t.shape)}')
    if safe and (t.shape[0] < 2 or t.shape[1] < 2):
        raise _empty_plane()
    _ops.white_balance(t, 0, _sites((wr, wg1, wg2, wb), bggr), None if sat is None else _sites(sat, bggr))
    if host is not None:
        host[...] = t.cpu().numpy()


def wb_postscale(rgb, wr, wg, wb, safe=False, saturation=None):
    """White-balance post scaling of an (..., 3) float RGB image in place (prysm/bayer.py); safe=True clamps the gains
    so that no channel exceeds its saturation, with the maxima and the ratio computed on the device."""
    sat = _saturation(saturation, 3) if safe else None
    t, host = _float_device(rgb, 'rgb')
    if t.ndim < 1 or t.shape[-1] != 3:
        raise ValueError(f'rgb must have 3 channels along its last axis, got shape {tuple(t.shape)}')
    if safe and t.numel() == 0:
        raise _empty_plane()
    _ops.white_balance(t, 1, (wr, wg, wb), sat)
    if host is not None:
        host[...] = t.cpu().numpy()


def _out_buffer(output, shape, dtype, dev):
    """(device tensor the kernel writes, numpy array to copy it into or None)."""
    if output is None:
        return torch.empty(shape, dtype=dtype, device=dev), None
    if isinstance(output, np.ndarray):
        if output.shape != tuple(shape):
            raise ValueError(f'output has shape {output.shape}, expected {tuple(shape)}')
        return torch.empty(shape, dtype=torch.from_numpy(np.empty(0, dtype=output.dtype)).dtype, device=dev), output
    if tuple(output.shape) != tuple(shape):
        raise ValueError(f'output has shape {tuple(output.shape)}, expected {tuple(shape)}')
    if not output.is_cuda or output.stride(-1) != 1:
        raise ValueError('output must be a CUDA tensor with unit stride along its last axis')
    return output, None


def _planes(arrays, dtype):
    return [_ops.asdevice(a).to(dtype).contiguous() for a in arrays]


def _finish(t, host):
    if host is None:
        return t
    host[...] = t.cpu().numpy()
    return host


def composite_bayer(r, g1, g2, b, cfa='rggb', output=None):
    """Interleave densely sampled (m, n) colour planes into one (m, n) mosaic (prysm/bayer.py): one kernel."""
    cfa = cfa.lower()
    bggr = _bggr(cfa)
    r = _ops.asdevice(r)
    out, host = _out_buffer(output, tuple(r.shape), r.dtype, r.device)
    planes = _planes((r, g1, g2, b), out.dtype)
    for p in planes:
        if p.shape != out.shape:
            raise ValueError(f'every plane must have shape {tuple(out.shape)}, got {tuple(p.shape)}')
    _ops.bayer_interleave(_sites(planes, bggr), False, out)
    return _finish(out, host)


def decomposite_bayer(img, cfa='rggb'):
    """The four colour planes of a mosaic as strided views of the device tensor (prysm/bayer.py): no kernel, no copy."""
    cfa = cfa.lower()
    bggr = _bggr(cfa)
    img = _ops.asdevice(img)
    tl, tr, bl, br = img[0::2, 0::2], img[0::2, 1::2], img[1::2, 0::2], img[1::2, 1::2]
    if bggr:
        return br, tr, bl, tl
    return tl, tr, bl, br


def recomposite_bayer(r, g1, g2, b, cfa='rggb', output=None):
    """Recomposite (m, n) raw colour planes into a (2m, 2n) mosaic, the reciprocal of decomposite_bayer: one kernel."""
    r = _ops.asdevice(r)
    m, n = r.shape
    cfa = cfa.lower()
    out, host = _out_buffer(output, (2 * m, 2 * n), r.dtype, r.device)
    bggr = _bggr(cfa)
    planes = _planes((r, g1, g2, b), out.dtype)
    for p in planes:
        if p.shape != (m, n):
            raise ValueError(f'every plane must have shape {(m, n)}, got {tuple(p.shape)}')
    _ops.bayer_interleave(_sites(planes, bggr), True, out)
    return _finish(out, host)


_DEINTERLACE_IN = (torch.float32, torch.float64, torch.uint8, torch.uint16, torch.uint32)


def demosaic_deinterlace(img, cfa='rggb'):
    """(m/2, n/2, 3) RGB with the two greens averaged (prysm/bayer.py): one kernel.  As in the reference, the green sum
    is formed in the mosaic's dtype and integer mosaics give float64; an odd side is a shape mismatch of the planes."""
    cfa = cfa.lower()
    bggr = _bggr(cfa)
    img = _ops.asdevice(img)
    if img.ndim != 2:
        raise ValueError(f'img must be 2-D, got shape {tuple(img.shape)}')
    m, n = img.shape
    if m % 2 or n % 2:
        raise ValueError(f'the colour planes of a {m} x {n} mosaic do not have one shape')
    if img.dtype not in _DEINTERLACE_IN:
        raise TypeError(f'demosaic_deinterlace does not take {img.dtype}')
    if img.stride(1) != 1:
        img = img.contiguous()
    out_dtype = img.dtype if img.is_floating_point() else torch.float64
    return _ops.demosaic_deinterlace(img, bggr, out_dtype)


def assemble_superresolved(r, g1, g2, b, zoomfactor, cfa='rggb', out=None):
    """(m, n, 3) RGB from super-resolved colour planes (prysm/bayer.py): r, b and g2 are moved onto g1's site by a
    Fourier shift of zoomfactor samples (one batched transform, a separable phase ramp, one batched inverse) and one
    kernel assembles the real parts, green as (g2' + g1) / 2.  Only rggb, compared as given (not lower-cased), as in the
    reference."""
    if cfa == 'rggb':
        shifts = ((-zoomfactor, 0), (0, zoomfactor), (-zoomfactor, zoomfactor))     # r, b, g2 -> g1
    else:
        raise NotImplementedError('assemble_superresolved: only rggb patterns supported at this time')
    r = _ops.asdevice(r)
    dt = r.dtype if r.dtype in (torch.float32, torch.float64) else torch.float64
    m, n = r.shape
    dst, host = _out_buffer(out, (m, n, 3), r.dtype, r.device)
    if dst.dtype != dt or not dst.is_contiguous():
        raise ValueError(f'out must be a contiguous {dt} array')
    stack = torch.stack(_planes((r, b, g2), dt))
    g1 = _ops.asdevice(g1).to(dt).contiguous()
    spec = _ops.fft2_batch(stack)
    cdt = spec.dtype
    shifted = torch.empty_like(spec)
    for i, (sy, sx) in enumerate(shifts):
        vy = _ops.asdevice(_ramp(m, sy), cdt)
        vx = _ops.asdevice(_ramp(n, sx), cdt)
        _ops.mul_outer(spec[i], vy, vx, out=shifted[i])
    back = _ops.fft2_batch(shifted, dir=1, scale=1.0 / (m * n))
    _ops.bayer_assemble(back[0], back[2], back[1], g1, dst)
    return _finish(dst, host)


def _ramp(N, shift):
    """exp(-2 pi i shift k / N) over scipy.ndimage.fourier_shift's frequency index k (k - N from (N + 1) // 2 on), the
    argument reduced to [-1/2, 1/2] turns in fp64 before the exponential."""
    k = np.arange(N, dtype=np.float64)
    k[(N + 1) // 2:] -= N
    turns = -float(shift) * k / N
    turns -= np.rint(turns)
    return np.exp(2j * np.pi * turns)


_MALVAR_IN = (torch.float32, torch.float64, torch.uint8, torch.uint16)


def demosaic_malvar(img, cfa='rggb'):
    """(m, n, 3) RGB from an (m, n) mosaic by Malvar-He-Cutler demosaicing (prysm/bayer.py), in one pass: each output
    pixel evaluates the two 5x5 filters its CFA site needs, in fp64, with scipy.ndimage's reflect boundary.  Integer
    input is promoted to config.precision."""
    cfa = cfa.lower()
    bggr = _bggr(cfa)
    img = _ops.asdevice(img)
    if img.ndim != 2:
        raise ValueError(f'img must be 2-D, got shape {tuple(img.shape)}')
    if img.is_complex():
        raise TypeError('demosaic_malvar takes a real mosaic')
    if img.is_floating_point():
        out_dtype = img.dtype if img.dtype in (torch.float32, torch.float64) else torch.float64
    else:
        out_dtype = config.real_dtype
    if img.dtype not in _MALVAR_IN or (img.dtype == torch.float64 and out_dtype == torch.float32):
        img = img.to(out_dtype)
    if img.stride(1) != 1:
        img = img.contiguous()
    return _ops.demosaic_malvar(img, bggr, out_dtype)
