"""GPU: the reference's analytic pins of the path (tests/test_physics.py:14-74, SURVEY.md 8(c) pin (ii)) run on the
device pipeline -- grid, circular aperture, focus, intensity, psf -> mtf all on the GPU -- against closed forms evaluated
in this test with numpy/scipy:
    Airy disk      (2 J1(u)/u)^2, u = pi r / (wvl F#)                       prysm/psf.py:240-265
    diffraction-limited MTF  2/pi (acos(v) - v sqrt(1 - v^2)), v = f wvl F#   prysm/otf.py:496-562
to the reference's own 1e-3, plus its array-orientation test."""
import numpy as np
import pytest
import torch
from scipy.special import j1

from gpu_fixtures import pb, host  # noqa: F401

pytestmark = pytest.mark.gpu
PARAMS = [(10.0, 1.000, 0.5), (10.0, 1.000, 1.0), (3.00, 1.125, 3.0)]


def centre_slices(a, dx):
    ny, nx = a.shape
    u = (np.arange(nx) - nx // 2) * dx
    return u, a[ny // 2, :], a[:, nx // 2]


def aperture(pb, epd):
    x, y = pb.coordinates.make_xy_grid(128, diameter=epd)
    r, _ = pb.coordinates.cart_to_polar(x, y)
    return pb.geometry.circle(epd / 2, r), float(x[0, 1] - x[0, 0])


@pytest.mark.parametrize('efl,epd,wvl', PARAMS)
def test_diffprop_matches_airydisk(pb, efl, epd, wvl):
    fno = efl / epd
    amp, dx = aperture(pb, epd)
    wf = pb.propagation.Wavefront.from_amp_and_phase(amp.to(torch.float64), None, wvl, dx).pad2d(Q=3)
    wf = wf * (3 * np.sqrt(amp.numel()) / float(amp.sum()))          # peak-normalise like the reference
    psf = wf.focus(efl, Q=1)
    u, sx, sy = centre_slices(host(psf.intensity.data), psf.dx)
    ue = u * np.pi / wvl / fno
    with np.errstate(invalid='ignore', divide='ignore'):
        analytic = np.where(np.abs(ue) < 1e-8, 1.0, (2 * j1(ue) / ue) ** 2)
    assert np.allclose(sx, analytic, atol=1e-3) and np.allclose(sy, analytic, atol=1e-3)


@pytest.mark.parametrize('efl,epd,wvl', PARAMS)
def test_diffprop_matches_analytic_mtf(pb, efl, epd, wvl):
    fno = efl / epd
    amp, dx = aperture(pb, epd)
    psf = pb.propagation.Wavefront.from_amp_and_phase(amp, None, wvl, dx).focus(efl, Q=3).intensity
    mtf = pb.otf.mtf_from_psf(psf.data, psf.dx)
    u, sx, sy = centre_slices(host(mtf.data), mtf.dx)
    v = np.minimum(np.abs(u) / (1 / (wvl / 1000 * fno)), 1.0)
    analytic = (2 / np.pi) * (np.arccos(v) - v * np.sqrt(1 - v ** 2))
    assert np.allclose(sx, analytic, atol=1e-3) and np.allclose(sy, analytic, atol=1e-3)


def test_array_orientation_consistency_tilt(pb):
    """arr[y, x] everywhere: +y tilt in the pupil moves the PSF towards +y (tests/test_physics.py:56-74)."""
    N, Q = 128, 3
    x, y = pb.coordinates.make_xy_grid(N, diameter=2.1)
    r, _ = pb.coordinates.cart_to_polar(x, y)
    amp = pb.geometry.circle(1, r)
    psf = pb.propagation.Wavefront.from_amp_and_phase(amp, 1000 * y, 0.5, float(x[0, 1] - x[0, 0])).focus(1, Q=Q).intensity
    idx = int(torch.argmax(psf.data))
    iy, ix = divmod(idx, psf.data.shape[1])
    assert ix == (N * Q) // 2 and iy > (N * Q) // 2
