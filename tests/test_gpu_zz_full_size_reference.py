"""GPU: BASELINE configs C4 and C5 at FULL size against the reference's own fp64 outputs (tests/golden/full_c4.npz,
full_c5.npz: windows, strided samples, sums written by oracle/make_golden.py full_c45), complex64 path.

  C4  2048^2 pupil -> CZT -> 2048^2 field at two wavelengths, weighted incoherent sum (polychromatic_psf)
  C5  4096^2 field x unit-modulus phase screen -> free_space(dz = 5 mm)

Inputs are bit-identical on both sides: the golden run used the OPD (and the screen's OPD) rounded to float32 once, which
is exactly what the complex64 path is fed here, so the differences below are transform error only.
Bounds = full-array parity figures (same inputs, the reference fp64 run as arbiter) times at most 1.5; every one is
inside the north-star 1e-6.  Measured by this test on an H100 (windows / strided samples):
    C4 CZT fields        measured 2.9e-7 / 3.5e-7   bound 5.5e-7      (the reference's own fp32 run: 1.2e-4 / 4.0e-4)
    C4 weighted PSF sum  measured 7.9e-7            bound 1.0e-6      (reference fp32: 2.2e-4)
    C5 free-space plane  measured 4.1e-7            bound 1.0e-6      (reference fp32: 4.0e-6)
    C5 final CZT focus   measured 5.0e-7            bound 6.5e-7      (reference fp32: 2.5e-5)"""
import numpy as np
import pytest

import prysm_oracle as O
from conftest import load_golden, within
from gpu_fixtures import pb, host  # noqa: F401

pytestmark = pytest.mark.gpu
HeNe = 0.6328


@pytest.fixture(scope='module', autouse=True)
def precision_32(pb):
    pb.config.precision = 32


def test_c4_czt_fields_and_incoherent_sum_vs_reference(pb):
    g = load_golden('full_c4.npz')
    P = pb.propagation
    N = M = 2048
    amp, opd, dx = O.synthetic_pupil(N, np.float32)
    cy = M // 2
    for w in (0.5, 0.7):
        tag = f'w{int(w * 10)}_'
        wf = P.Wavefront.from_amp_and_phase(amp, opd, w, dx)
        f = host(wf.focus_dft(wf.prepare_executor(100.0, 2.5, M, kind='czt')).data)
        den = float(g[tag + 'absmax'])
        assert f.shape == (M, M)
        within(f'c4.{tag}field_stride', np.abs(f[::64, ::64] - g[tag + 'field_stride']).max() / den, 5.5e-7)
        within(f'c4.{tag}field_window', np.abs(f[cy - 32:cy + 32, cy - 32:cy + 32] - g[tag + 'field_win']).max() / den, 5.5e-7)
        I = (f.real.astype(np.float64) ** 2 + f.imag.astype(np.float64) ** 2).sum()
        assert I == pytest.approx(float(g[tag + 'I_sum']), rel=1e-6)
    from prysm_b200.polychromatic import polychromatic_psf
    tot = host(polychromatic_psf(amp, opd, [0.5, 0.7], [0.25, 0.75], dx, 100.0, 2.5, M, kind='czt')).astype(np.float64)
    smax = float(g['sum_max'])
    within('c4.sum_stride', np.abs(tot[::64, ::64] - g['sum_stride']).max() / smax, 1e-6)
    within('c4.sum_window', np.abs(tot[cy - 32:cy + 32, cy - 32:cy + 32] - g['sum_win']).max() / smax, 1e-6)
    assert tot.sum() == pytest.approx(float(g['sum_total']), rel=1e-6)


def test_c5_screen_and_free_space_plane_vs_reference(pb):
    g = load_golden('full_c5.npz')
    P = pb.propagation
    N = 4096
    amp, opd, dx = O.synthetic_pupil(N, np.float32)
    wf = P.Wavefront.from_amp_and_phase(amp, opd, HeNe, dx)
    phi32 = np.random.default_rng(1000).normal(0, 0.1, (N, N)).astype(np.float32)
    scr_opd = (phi32.astype(np.float64) * (HeNe * 1e3 / (2 * np.pi))).astype(np.float32)   # exp(i*phi): OPD[nm] = phi*wvl/(2 pi)
    scr = P.Wavefront.phase_screen(scr_opd, HeNe, dx)
    plane = (wf * scr).free_space(dz=float(g['dz']), Q=1)         # the screen multiply rides in the first transform pass
    out = host(plane.data)
    den = float(g['absmax'])
    c = N // 2
    assert out.shape == (N, N)
    within('c5.plane_stride', np.abs(out[::128, ::128] - g['field_stride']).max() / den, 1e-6)
    within('c5.plane_window', np.abs(out[c - 32:c + 32, c - 32:c + 32] - g['field_win']).max() / den, 1e-6)
    within('c5.plane_edge', np.abs(out[c, 1000:1100] - g['edge']).max() / den, 1e-6)
    E = (out.real.astype(np.float64) ** 2 + out.imag.astype(np.float64) ** 2).sum()
    assert E == pytest.approx(float(g['E_out']), rel=1e-6)
    # the chain's final focus: CZT 4096^2 -> 512^2
    foc = host(plane.focus_dft(plane.prepare_executor(100.0, float(g['focal_dx']), 512, kind='czt')).data)
    fden = float(g['focus_absmax'])
    within('c5.focus_window', np.abs(foc[256 - 32:256 + 32, 256 - 32:256 + 32] - g['focus_win']).max() / fden, 6.5e-7)
    within('c5.focus_stride', np.abs(foc[::16, ::16] - g['focus_stride']).max() / fden, 6.5e-7)
    If = (foc.real.astype(np.float64) ** 2 + foc.imag.astype(np.float64) ** 2).sum()
    assert If == pytest.approx(float(g['focus_I_sum']), rel=2e-6)
