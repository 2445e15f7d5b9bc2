"""PSF -> MTF / PTF / OTF on the H100 engine (reference prysm/otf.py:11-202).

One fused centred FFT of the real PSF (shifts folded into the passes, no complex copy of the
input) and one normalisation kernel that divides by the centre sample and takes abs / angle.
"""
from . import _ops
from ._richdata import RichData


def _unwrap_psf(psf, dx):
    """prysm/otf.py:16-25."""
    if not hasattr(psf, 'ndim'):
        dx = psf.dx
        psf = psf.data
    if dx is None:
        raise ValueError('dx is None: dx must be provided if psf is an array')
    return _ops.asdevice(psf), dx


def transform_psf(psf, dx=None):
    """fftshift(fft2(ifftshift(psf))), unnormalised; df = 1000/(rows*dx) (prysm/otf.py:28-33)."""
    psf, dx = _unwrap_psf(psf, dx)
    data = _ops.fft2(psf, tuple(psf.shape), dir=-1, scale=1.0, shift_in=True, shift_out=True)
    return data, 1000 / (data.shape[0] * dx)


def transform_psf_adjoint(data_bar):
    """fftshift(ifft2(ifftshift(g), norm='forward')) (prysm/otf.py:36-59)."""
    g = _ops.ascomplex(_ops.asdevice(data_bar))
    return _ops.fft2(g, tuple(g.shape), dir=+1, scale=1.0, shift_in=True, shift_out=True)


def _normalized(psf, dx, which):
    data, df = transform_psf(psf, dx)
    mtf, ptf, otf = _ops.otf_normalize(data, which)
    return mtf, ptf, otf, data, df


def mtf_from_psf(psf, dx=None, return_more=False):
    """prysm/otf.py:77-104."""
    mtf, _, _, data, df = _normalized(psf, dx, 1)
    rd = RichData(data=mtf, dx=df, wavelength=None)
    return (rd, data) if return_more else rd


def ptf_from_psf(psf, dx=None, return_more=False):
    """prysm/otf.py:107-137."""
    _, ptf, _, data, df = _normalized(psf, dx, 2)
    rd = RichData(data=ptf, dx=df, wavelength=None)
    return (rd, data) if return_more else rd


def otf_from_psf(psf, dx=None, return_more=False):
    """prysm/otf.py:140-167."""
    _, _, otf, data, df = _normalized(psf, dx, 4)
    rd = RichData(data=otf, dx=df, wavelength=None)
    return (rd, data) if return_more else rd


def mtf_ptf_otf_from_psf(psf, dx=None, return_more=False):
    """All three from one forward transform (prysm/otf.py:170-202)."""
    mtf, ptf, otf, data, df = _normalized(psf, dx, 7)
    out = (RichData(mtf, df, None), RichData(ptf, df, None), RichData(otf, df, None))
    return out + (data,) if return_more else out


def _forward_data(psf, dx, data):
    if data is None:
        data, _ = transform_psf(psf, dx)
    return _ops.ascomplex(_ops.asdevice(data))


def mtf_from_psf_adjoint(mtf_bar, psf=None, dx=None, data=None):
    """Gradient at the PSF plane of a gradient on the centre-normalised MTF: one seed kernel (modulus +
    normalisation terms) and the adjoint transform (prysm/otf.py:205-242)."""
    seed = _ops.otf_adjoint_seed(1, mtf_bar, _forward_data(psf, dx, data))
    return transform_psf_adjoint(seed).real


def ptf_from_psf_adjoint(ptf_bar, psf=None, dx=None, data=None):
    """prysm/otf.py:245-279."""
    seed = _ops.otf_adjoint_seed(2, ptf_bar, _forward_data(psf, dx, data))
    return transform_psf_adjoint(seed).real


def otf_from_psf_adjoint(otf_bar, psf=None, dx=None, data=None):
    """prysm/otf.py:282-316."""
    seed = _ops.otf_adjoint_seed(4, _ops.ascomplex(_ops.asdevice(otf_bar)), _forward_data(psf, dx, data))
    return transform_psf_adjoint(seed).real


def encircled_energy_adjoint(ee_bar, psf=None, dx=None, radius=None, data=None):
    """Encircled energy is linear in the MTF: the per-radius gradients fold into one MTF-plane gradient (one
    kernel), then mtf_from_psf_adjoint (prysm/otf.py:417-471)."""
    import numbers
    import numpy as np
    if data is not None:
        if dx is None:
            raise ValueError('dx is None: dx must be provided to set the frequency grid')
        data = _ops.ascomplex(_ops.asdevice(data))
        dxv = dx
    else:
        arr, dxv = _unwrap_psf(psf, dx)
        data, _ = transform_psf(arr, dxv)
    shape = tuple(data.shape)
    df = 1000 / (shape[0] * dxv)
    if isinstance(radius, numbers.Number):
        radius, ee_bar = (radius,), (ee_bar,)
    radii = np.asarray(list(radius), dtype=np.float64) / 1e3
    bars = np.asarray(list(ee_bar), dtype=np.float64)[:len(radii)]
    radii = radii[:len(bars)]                                   # zip() semantics of the reference loop
    rd = data.real.dtype
    mtf_bar = _ops.encircled_energy_adjoint_seed(shape, df, radii, bars, rd, data.device)
    return mtf_from_psf_adjoint(mtf_bar, data=data)


def encircled_energy(psf, dx, radius, return_more=False):
    """Baliga & Cohn encircled energy at `radius` [um] (scalar or iterable) from the MTF of the PSF
    (prysm/otf.py:346-387): one reduction kernel per call covers all radii."""
    import numbers
    import numpy as np
    mtf, data = mtf_from_psf(psf, dx, return_more=True)
    scalar = isinstance(radius, numbers.Number)
    radii = np.atleast_1d(np.asarray(radius, dtype=np.float64)) / 1e3
    out = _ops.encircled_energy(mtf.data, mtf.dx, radii)
    out = float(out[0]) if scalar else out
    return (out, data) if return_more else out


def analytical_encircled_energy_circular_aperture(fno, wavelength, points):
    """1 - J0(p)^2 - J1(p)^2, p = points pi / fno / wavelength (prysm/otf.py:474-493), one kernel."""
    from . import _capi
    from .psf import analytic
    return analytic(_capi.AR_EE_CIRCULAR, points, wavelength, fno)


def diffraction_limited_mtf(fno, wavelength, frequencies=None, samples=128):
    """The MTF of a circular pupil at frequencies [cy/mm], or (frequencies, mtf) at `samples` frequencies from 0 to
    the extinction 1 / (wavelength / 1000 fno) when none are given (prysm/otf.py:496-543), one kernel."""
    import numpy as np
    from . import _capi
    from .psf import analytic
    if frequencies is None:
        extinction = 1 / (wavelength / 1000 * fno)
        nf = np.linspace(0, 1, samples)
        return _ops.asdevice(nf * extinction), analytic(_capi.AR_DIFFLIM_NORMALIZED, nf, 0.0, 0.0)
    return analytic(_capi.AR_DIFFLIM_MTF, frequencies, wavelength, fno)
