"""GPU parity: the CUDA path (through the C ABI) against the reference's golden outputs and the
CPU oracle on identical seeded inputs.

Tolerances (relative L-inf = max|a-b|/max|b|, SURVEY.md section 8d):
    complex128 path vs the reference's fp64 golden ........ 1e-12
    complex64  path vs the fp64 oracle on the same inputs .. 1e-6   (BASELINE.json north_star)
"""
import numpy as np
import pytest
import torch

import prysm_oracle as O
from conftest import rel_linf, load_golden, within
from gpu_fixtures import pb, host  # noqa: F401

pytestmark = pytest.mark.gpu

HeNe = 0.6328
TOL64 = 1e-12
TOL32 = 1e-6


def Qof(v):
    v = float(v)
    return int(v) if v == int(v) else v


# ------------------------------------------------------------------------------------------
# focus family: golden (fp64) and oracle (fp32 inputs)
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize('i', range(9))
def test_focus_family_c128_vs_reference_golden(pb, small, i):
    P = pb.propagation
    a, Q, g = small[f'focus{i}_in'], Qof(small[f'focus{i}_Q']), small[f'focus{i}_gin']
    assert rel_linf(host(P.focus(a, Q)), small[f'focus{i}_focus']) < TOL64
    assert rel_linf(host(P.unfocus(a, Q)), small[f'focus{i}_unfocus']) < TOL64
    assert rel_linf(host(P.focus_adjoint(g, Q)), small[f'focus{i}_focus_adjoint']) < TOL64
    assert rel_linf(host(P.unfocus_adjoint(g, Q)), small[f'focus{i}_unfocus_adjoint']) < TOL64


@pytest.mark.parametrize('i', range(9))
def test_focus_family_c64_vs_oracle(pb, small, i):
    P = pb.propagation
    a = small[f'focus{i}_in'].astype(np.complex64)
    g = small[f'focus{i}_gin'].astype(np.complex64)
    Q = Qof(small[f'focus{i}_Q'])
    out = P.focus(a, Q)
    assert out.dtype == torch.complex64
    assert rel_linf(host(out), O.focus(a.astype(np.complex128), Q)) < TOL32
    assert rel_linf(host(P.unfocus(a, Q)), O.unfocus(a.astype(np.complex128), Q)) < TOL32
    assert rel_linf(host(P.focus_adjoint(g, Q)), O.focus_adjoint(g.astype(np.complex128), Q)) < TOL32
    assert rel_linf(host(P.unfocus_adjoint(g, Q)), O.unfocus_adjoint(g.astype(np.complex128), Q)) < TOL32


@pytest.mark.parametrize('shape,Q', [((1, 1), 1), ((2, 2), 1), ((1, 8), 2), ((3, 5), 2), ((16, 4), 1), ((5, 5), 1),
                                     ((100, 60), 1), ((33, 65), 2), ((128, 128), 1), ((512, 256), 2)])
@pytest.mark.parametrize('cdt', [np.complex64, np.complex128])
def test_focus_ragged_and_edge_shapes(pb, shape, Q, cdt):
    rng = np.random.default_rng(shape[0] * 1000 + shape[1])
    a = (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype(cdt)
    tol = TOL32 if cdt is np.complex64 else TOL64
    ref = O.focus(a.astype(np.complex128), Q)
    assert rel_linf(host(pb.propagation.focus(a, Q)), ref) < tol
    ref = O.unfocus(a.astype(np.complex128), Q)
    assert rel_linf(host(pb.propagation.unfocus(a, Q)), ref) < tol


def test_focus_unfocus_roundtrip_is_identity(pb):
    """reference tests/test_propagation.py:24-29"""
    rng = np.random.default_rng(5)
    a = (rng.random((64, 64)) + 1j * rng.random((64, 64))).astype(np.complex128)
    P = pb.propagation
    wf = P.Wavefront(a, HeNe, 0.1)
    back = wf.focus(1, 1).unfocus(1, 1)
    assert rel_linf(host(back.data), a) < 1e-13
    assert back.space == 'pupil' and back.dx == pytest.approx(0.1)


@pytest.mark.parametrize('Q', [1, 1.5, 2])
def test_focus_adjoint_dot_product(pb, Q):
    """<Ax, y> == <x, A^H y> on odd rectangular shapes (reference tests/test_propagation.py:32-55)."""
    rng = np.random.default_rng(11)
    x = rng.standard_normal((9, 12)) + 1j * rng.standard_normal((9, 12))
    P = pb.propagation
    Ax = host(P.focus(x, Q))
    y = rng.standard_normal(Ax.shape) + 1j * rng.standard_normal(Ax.shape)
    AHy = host(P.focus_adjoint(y, Q))
    assert abs(np.vdot(y, Ax) - np.vdot(AHy, x)) < 1e-12 * abs(np.vdot(y, Ax)) + 1e-12
    Bx = host(P.unfocus(x, Q))
    BHy = host(P.unfocus_adjoint(y, Q))
    assert abs(np.vdot(y, Bx) - np.vdot(BHy, x)) < 1e-12 * abs(np.vdot(y, Bx)) + 1e-12


# ------------------------------------------------------------------------------------------
# Wavefront object path
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize('prec', [64, 32])
def test_wavefront_chain(pb, small, prec):
    P = pb.propagation
    pb.config.precision = prec
    tol = TOL64 if prec == 64 else TOL32
    rdt = np.float64 if prec == 64 else np.float32
    amp, opd, dx = small['wf_amp'], small['wf_opd'].astype(rdt), float(small['wf_dx'])
    ref_field = O.from_amp_and_phase(amp, opd.astype(np.float64), HeNe)
    ref_psf = O.focus(ref_field, 2)
    wf = P.Wavefront.from_amp_and_phase(amp, opd, HeNe, dx)
    psf = wf.focus(100.0, Q=2)                      # fused synthesis path (lazy field)
    assert psf.space == 'psf'
    assert psf.dx == pytest.approx(float(small['wf_psf_dx']), rel=1e-12)
    assert rel_linf(host(psf.data), ref_psf) < tol
    assert rel_linf(host(wf.data), ref_field) < tol  # materialised field
    assert rel_linf(host(P.Wavefront(wf.data, HeNe, dx).focus(100.0, Q=2).data), ref_psf) < tol
    I = psf.intensity
    assert rel_linf(host(I.data), O.intensity(ref_psf)) < tol
    assert I.dx == psf.dx and I.wavelength == HeNe
    if prec == 64:
        assert rel_linf(host(psf.data), small['wf_psf_field']) < TOL64
        assert rel_linf(host(I.data), small['wf_psf_intensity']) < TOL64
        assert rel_linf(host(psf.unfocus(100.0, Q=1).data), small['wf_back_field']) < TOL64
    # fused |.|^2 outputs
    I2 = P.psf_from_amp_and_phase(amp, opd, HeNe, 2)
    assert rel_linf(host(I2), O.intensity(ref_psf)) < tol
    acc = torch.zeros_like(I2)
    P.psf_from_amp_and_phase(amp, opd, HeNe, 2, weight=0.25, out=acc)
    P.focus_intensity(wf.data, 2, weight=0.75, out=acc)
    assert rel_linf(host(acc), O.intensity(ref_psf)) < 2 * tol
    pb.config.precision = 64


def test_wavefront_errors_and_operators(pb):
    """reference tests/test_propagation.py:285-315"""
    P = pb.propagation
    a = np.ones((8, 8), dtype=np.complex128)
    wf = P.Wavefront(a, HeNe, 0.1)
    with pytest.raises(ValueError, match='can only propagate from a psf to pupil plane'):
        wf.unfocus(1, 1)
    with pytest.raises(ValueError, match='can only propagate from a pupil to psf plane'):
        wf.focus(1, 1).focus(1, 1)
    with pytest.raises(ValueError, match='dz must be provided'):
        wf.free_space()
    with pytest.raises(TypeError):
        wf * 'a string'
    other = P.Wavefront(a, HeNe, 0.2)
    with pytest.raises(ValueError, match='physicality'):
        wf * other
    two = P.Wavefront(2 * a, HeNe, 0.1)
    assert np.allclose(host((wf * two).data), 2) and np.allclose(host((wf + two).data), 3)
    assert np.allclose(host((wf - two).data), -1) and np.allclose(host((wf / two).data), 0.5)
    assert np.allclose(host((3 * wf).data), 3) and np.allclose(host((1 / two).data), 0.5)
    assert np.allclose(host((wf * torch.full((8, 8), 1j, dtype=torch.complex128, device='cuda')).data), 1j)
    p = wf.pad2d(2, inplace=False)
    assert p.data.shape == (16, 16) and float(p.data.abs().sum()) == 64
    assert p.crop(8, inplace=False).data.shape == (8, 8)
    assert rel_linf(host(p.crop(8, inplace=False).data), a) == 0


def test_thin_lens_and_phase_screen(pb, small):
    P = pb.propagation
    g = O.fftrange(64) * float(small['wf_dx'])
    x, y = np.meshgrid(g, g)
    lens = P.Wavefront.thin_lens(250.0, HeNe, x, y)
    assert rel_linf(host(lens.data), small['lens']) < 1e-11
    assert lens.dx == pytest.approx(float(small['wf_dx']))
    scr = P.Wavefront.phase_screen(small['wf_opd'], HeNe, 0.1)
    assert rel_linf(host(scr.data), O.phase_screen(small['wf_opd'], HeNe)) < TOL64


# ------------------------------------------------------------------------------------------
# angular spectrum
# ------------------------------------------------------------------------------------------
def test_angular_spectrum_c128_vs_reference_golden(pb, small):
    P = pb.propagation
    f = small['as_in']
    for Q in (1, 2):
        assert rel_linf(host(P.angular_spectrum(f, HeNe, 0.05, 12.5, Q)), small[f'as_Q{Q}']) < TOL64
    pb.config.precision = 64
    assert rel_linf(host(P.angular_spectrum_transfer_function((24, 32), HeNe, 0.05, 12.5)), small['as_tf']) < TOL64
    assert rel_linf(host(P.angular_spectrum(f, HeNe, 0.05, 12.5, tf=small['as_tf'])), small['as_with_tf']) < TOL64
    assert rel_linf(host(P.angular_spectrum_adjoint(small['as_gin'], HeNe, 0.05, 12.5, 2)), small['as_adjoint_Q2']) < TOL64
    assert rel_linf(host(P.angular_spectrum(small['as9_in'], HeNe, 0.05, 3.0, 1)), small['as9_Q1']) < TOL64
    assert rel_linf(host(P.angular_spectrum(small['as9_in'], HeNe, 0.05, 3.0, 1.5)), small['as9_Q15']) < TOL64


def test_angular_spectrum_c64_and_identities(pb, small):
    P = pb.propagation
    f = small['as_in'].astype(np.complex64)
    for Q in (1, 2):
        ref = O.angular_spectrum(f.astype(np.complex128), HeNe, 0.05, 12.5, Q)
        assert rel_linf(host(P.angular_spectrum(f, HeNe, 0.05, 12.5, Q)), ref) < TOL32
    # zero distance is the identity (reference tests/test_propagation.py:210-218)
    assert rel_linf(host(P.angular_spectrum(small['as_in'], HeNe, 0.05, 0.0, 1)), small['as_in']) < 1e-13
    # adjoint dot-product test with and without tf (reference tests/test_propagation.py:178-243)
    rng = np.random.default_rng(2)
    x = rng.standard_normal((9, 12)) + 1j * rng.standard_normal((9, 12))
    Ax = host(P.angular_spectrum(x, HeNe, 0.05, 3.0, 1.5))
    y = rng.standard_normal(Ax.shape) + 1j * rng.standard_normal(Ax.shape)
    AHy = host(P.angular_spectrum_adjoint(y, HeNe, 0.05, 3.0, 1.5))
    assert abs(np.vdot(y, Ax) - np.vdot(AHy, x)) < 1e-12 * abs(np.vdot(y, Ax))
    wf = P.Wavefront(small['as_in'], HeNe, 0.05)
    out = wf.free_space(dz=12.5, Q=2)
    assert rel_linf(host(out.data), small['as_Q2']) < TOL64 and out.dx == 0.05 and out.space == 'pupil'


# ------------------------------------------------------------------------------------------
# executors
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize('i', range(4))
@pytest.mark.parametrize('kind', ['mdft', 'czt'])
@pytest.mark.parametrize('prec', [64, 32])
def test_executors_vs_reference_golden(pb, small, i, kind, prec):
    P = pb.propagation
    pb.config.precision = prec
    cdt = np.complex128 if prec == 64 else np.complex64
    tol = TOL64 if prec == 64 else TOL32
    a, g = small[f'ex{i}_in'].astype(cdt), small[f'ex{i}_gin'].astype(cdt)
    pdx, fdx, wvl, efl, sx, sy = (float(v) for v in small[f'ex{i}_params'])
    ex = P.prepare_executor(pdx, a.shape, fdx, g.shape, wvl, efl, (sx, sy), kind)
    assert ex.pupil_dx == pdx and ex.focal_dx == fdx
    within(f'executors.{kind}{i}.p{prec}.fwd', rel_linf(host(ex(a)), small[f'ex{i}_{kind}_fwd']), tol)
    within(f'executors.{kind}{i}.p{prec}.adj', rel_linf(host(ex.adjoint(g)), small[f'ex{i}_{kind}_adj']), tol)
    assert ex.nbytes() > 0
    pb.config.precision = 64


@pytest.mark.parametrize('i', range(2))
def test_fftdft_vs_reference_golden(pb, small, i):
    P = pb.propagation
    pb.config.precision = 64
    a, g = small[f'fd{i}_in'], small[f'fd{i}_gin']
    pdx, fdx, wvl, efl, sx, sy = (float(v) for v in small[f'fd{i}_params'])
    ex = P.prepare_executor(pdx, a.shape, fdx, g.shape, wvl, efl, (sx, sy), 'fftdft')
    assert rel_linf(host(ex(a)), small[f'fd{i}_fwd']) < TOL64
    assert rel_linf(host(ex.adjoint(g)), small[f'fd{i}_adj']) < TOL64


def test_executor_equivalences_and_structure(pb):
    """FFT focus == MDFT == CZT == FFTDFT at FFT-equivalent sampling; multiply-order flags; nbytes;
    non power-of-two FFTDFT length (reference tests/test_fttools.py:26-85,140-182; test_propagation.py:98-166)."""
    P, F = pb.propagation, pb.fttools
    pb.config.precision = 64
    rng = np.random.default_rng(3)
    a = rng.standard_normal((16, 16)) + 1j * rng.standard_normal((16, 16))
    fdx = HeNe * 100.0 / (0.1 * 32)
    ref = host(P.focus(a, 2))
    outs = {k: host(P.prepare_executor(0.1, 16, fdx, 32, HeNe, 100.0, kind=k)(a)) for k in ('mdft', 'czt', 'fftdft')}
    for k, v in outs.items():
        assert rel_linf(v, ref) < 1e-12, k
    # K = 20 (not a power of two) through Bluestein
    fdx20 = HeNe * 100.0 / (0.1 * 20)
    m = host(P.prepare_executor(0.1, (12, 10), fdx20, (20, 9), HeNe, 100.0, kind='mdft')(a[:12, :10]))
    f = host(P.prepare_executor(0.1, (12, 10), fdx20, (20, 9), HeNe, 100.0, kind='fftdft')(a[:12, :10]))
    assert rel_linf(f, m) < 1e-12
    x = np.arange(-8, 8) * 0.1
    fx = np.arange(-4, 4) * 0.3
    ex = F.MDFT(x, x, fx, fx)
    assert ex.Ex.shape == (8, 16) and ex.Ey.shape == (8, 16) and ex.nbytes() == 2 * 8 * 16 * 16
    assert ex._forward_left_first == (8 * 16 * (16 + 8) <= 16 * 8 * (16 + 8))
    assert rel_linf(host(ex.Ex), np.exp(-2j * np.pi * np.outer(fx, x))) < 1e-14
    # adjoint(forward) = N^2 * I on a full unit cell (reference tests/test_fttools.py:35-44)
    n = 16
    xx = np.arange(-8, 8, dtype=float)
    ex = F.MDFT(xx, xx, xx / n, xx / n)
    assert rel_linf(host(ex.adjoint(ex(a))), a * n * n) < 1e-12
    with pytest.raises(ValueError, match='not FFT-compatible'):
        F.FFTDFT(xx, xx, xx / 10.3, xx / 10.3)
    with pytest.raises(ValueError, match='sign must be -1 or \\+1'):
        F.CZT(xx, xx, xx, xx, sign=2)
    with pytest.raises(ValueError):
        ex(np.ones((3, 3), dtype=np.complex128))


def test_legacy_fixed_sampling_aliases(pb, small):
    """BASELINE.json names focus_fixed_sampling (v0.19-v0.21 API)."""
    P = pb.propagation
    pb.config.precision = 64
    a, g = small['ex1_in'], small['ex1_gin']
    pdx, fdx, wvl, efl, sx, sy = (float(v) for v in small['ex1_params'])
    out = P.focus_fixed_sampling(a, pdx, efl, wvl, fdx, g.shape, (sx, sy), 'mdft')
    assert rel_linf(host(out), small['ex1_mdft_fwd']) < TOL64
    back = P.unfocus_fixed_sampling(g, fdx, efl, wvl, pdx, a.shape, (sx, sy), 'czt')
    assert rel_linf(host(back), small['ex1_czt_adj']) < TOL64
    wf = P.Wavefront(a, wvl, pdx)
    o2 = wf.focus_fixed_sampling(efl, fdx, g.shape, (sx, sy), 'czt')
    assert rel_linf(host(o2.data), small['ex1_czt_fwd']) < TOL64 and o2.dx == fdx and o2.space == 'psf'


# ------------------------------------------------------------------------------------------
# psf / otf reductions, incoherent sum
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize('prec', [64, 32])
def test_otf_family(pb, small, prec):
    otf = pb.otf
    rdt = np.float64 if prec == 64 else np.float32
    tol = 1e-11 if prec == 64 else 2e-6
    I = small['wf_psf_intensity'].astype(rdt)
    pdx = float(small['wf_psf_dx'])
    mtf = otf.mtf_from_psf(I, pdx)
    assert mtf.dx == pytest.approx(float(small['wf_mtf_df']))
    ref_mtf, _ = O.mtf_from_psf(I.astype(np.float64), pdx)
    assert np.abs(host(mtf.data) - ref_mtf).max() < tol          # MTF abs L-inf (MTF <= 1)
    m, p, o = otf.mtf_ptf_otf_from_psf(pb.propagation.RichData(pb.asdevice(I), pdx, HeNe))
    assert torch.equal(m.data, mtf.data)                         # bit-identical to the single (reference tests/test_otf.py:141-158)
    assert torch.equal(p.data, otf.ptf_from_psf(I, pdx).data) and torch.equal(o.data, otf.otf_from_psf(I, pdx).data)
    c = I.shape[0] // 2
    assert complex(host(o.data)[c, c]) == 1 + 0j and float(host(m.data)[c, c]) == 1.0 and float(host(p.data)[c, c]) == 0.0
    if prec == 64:
        assert np.abs(host(m.data) - small['wf_mtf']).max() < 1e-11
        assert rel_linf(host(o.data), small['wf_otf']) < 1e-11
        sel = small['wf_mtf'] > 1e-6
        assert np.abs(host(p.data) - small['wf_ptf'])[sel].max() < 1e-6
    data, df = otf.transform_psf(I, pdx)
    assert rel_linf(host(data), O.transform_psf(I.astype(np.float64), pdx)[0]) < (1e-12 if prec == 64 else 1e-6)
    with pytest.raises(ValueError, match='dx is None'):
        otf.mtf_from_psf(I)


def test_centroid_and_mode_sum(pb, small):
    I, pdx = small['wf_psf_intensity'], float(small['wf_psf_dx'])
    assert np.allclose(pb.psf.centroid(I, pdx), small['wf_centroid'], rtol=1e-9, atol=1e-10)
    assert np.allclose(pb.psf.centroid(I, unit='pixels'), small['wf_centroid_px'], rtol=1e-12)
    out = pb.polynomials.sum_of_2d_modes(pb.asdevice(small['modes']), small['weights'])
    assert rel_linf(host(out), small['modes_sum']) < 1e-14
    rng = np.random.default_rng(0)
    big = rng.random((70, 33, 17)).astype(np.float32)   # > 64 modes exercises the chunked accumulate
    w = rng.random(70)
    out = pb.polynomials.sum_of_2d_modes(pb.asdevice(big), w)
    assert rel_linf(host(out), np.tensordot(big.astype(np.float64), w, axes=(0, 0))) < 1e-6


# ------------------------------------------------------------------------------------------
# BASELINE.json sizes against the reference's stored fp64 windows and size-independent properties
# ------------------------------------------------------------------------------------------
def _window(a, w):
    cy, cx = a.shape[0] // 2, a.shape[1] // 2
    return a[cy - w // 2:cy + w // 2, cx - w // 2:cx + w // 2]


def test_c1_256_focus_fp64(pb):
    g = load_golden('full_c1.npz')
    amp, opd, dx = O.synthetic_pupil(256, np.float64)
    P = pb.propagation
    pb.config.precision = 64
    psf = P.Wavefront.from_amp_and_phase(amp, opd, HeNe, dx).focus(100.0, Q=2)
    f = host(psf.data)
    assert f.shape == (512, 512) and psf.dx == pytest.approx(float(g['psf_dx']))
    assert np.abs(_window(f, 64) - g['field_win']).max() / float(g['field_absmax']) < 1e-9
    assert np.abs(f[::16, ::16] - g['field_stride']).max() / float(g['field_absmax']) < 1e-9
    I = host(psf.intensity.data)
    assert I.sum() == pytest.approx(float(g['E_in']), rel=1e-12)


def test_c2_2048_focus_fp32_headline(pb):
    """BASELINE configs[1]: 2048^2 Zernike-aberrated pupil -> 4096^2 PSF, complex64, against the
    reference's fp64 run (windows, strided samples, energy, MTF)."""
    g = load_golden('full_c2.npz')
    N = 2048
    amp, opd, dx = O.synthetic_pupil(N, np.float32)
    P = pb.propagation
    pb.config.precision = 32
    wf = P.Wavefront.from_amp_and_phase(amp, opd, HeNe, dx)
    field = wf.data                               # complex64 pupil (materialised)
    assert field.dtype == torch.complex64
    psf = P.Wavefront(field, HeNe, dx).focus(100.0, Q=2)
    assert psf.data.shape == (4096, 4096) and psf.data.dtype == torch.complex64
    assert psf.dx == pytest.approx(float(g['psf_dx']), rel=1e-12)
    f = host(psf.data)
    amax = float(g['field_absmax'])
    # bounds: full-array parity figures on identical inputs (field 1.4e-7, PSF 2.3e-7) x 1.5; measured here on an H100:
    # field window 1.4e-7, PSF window 2.5e-7
    within('c2.field_window', np.abs(_window(f, 64) - g['field_win']).max() / amax, 2.1e-7)
    within('c2.field_stride', np.abs(f[::N // 16, ::N // 16] - g['field_stride']).max() / amax, 2.1e-7)
    I = host(psf.intensity.data).astype(np.float64)
    within('c2.psf_window', np.abs(_window(I, 64) - g['I_win']).max() / float(g['I_max']), 3.5e-7)   # PSF relative L-inf
    within('c2.energy', abs(I.sum() / float(g['E_in']) - 1), 5e-7)                                   # energy conservation
    within('c2.rowsum', np.abs(I.sum(axis=1)[::8] - g['I_rowsum']).max() / g['I_rowsum'].max(), 5e-7)
    within('c2.colsum', np.abs(I.sum(axis=0)[::8] - g['I_colsum']).max() / g['I_colsum'].max(), 5e-7)
    mtf = host(pb.otf.mtf_from_psf(psf.intensity).data)
    within('c2.mtf_window', np.abs(_window(mtf, 64) - g['mtf_win']).max(), 1e-6)                      # MTF abs L-inf
    within('c2.mtf_row', np.abs(mtf[mtf.shape[0] // 2, ::8] - g['mtf_row']).max(), 1e-6)
    # fused synth -> focus -> |.|^2 gives the same PSF
    I2 = host(P.psf_from_amp_and_phase(amp, opd, HeNe, 2)).astype(np.float64)
    within('c2.fused_psf_vs_two_step', np.abs(I2 - I).max() / float(g['I_max']), 3.5e-7)
    # size-independent properties at full size: unitarity and linearity
    back = psf.unfocus(100.0, Q=1)
    within('c2.unfocus_round_trip', rel_linf(host(pb.fttools.crop_center(back.data, N)), host(field)), 1e-6)
    pb.config.precision = 64


def test_c3_4096_mdft_to_512(pb):
    """BASELINE configs[2]: 4096^2 -> 512^2 fixed-sampling focus via MDFT, complex64."""
    g = load_golden('full_c3.npz')
    N, M = 4096, 512
    amp, opd, dx = O.synthetic_pupil(N, np.float32)
    P = pb.propagation
    pb.config.precision = 32
    wf = P.Wavefront.from_amp_and_phase(amp, opd, HeNe, dx)
    ex = wf.prepare_executor(100.0, float(g['focal_dx']), M, kind='mdft')
    assert ex.norm == pytest.approx(float(g['norm']), rel=1e-6)
    out = wf.focus_dft(ex)
    f = host(out.data)
    amax = float(g['field_absmax'])
    assert f.shape == (M, M) and out.dx == float(g['focal_dx'])
    # tensor-core MDFT (3xTF32), bound 1e-6 (the reference's own fp32 run: 1.0e-6); measured on an H100: window 4.3e-7,
    # stride 1.1e-7; the CZT of the same window: 2.5e-7
    within('c3.mdft_field_window', np.abs(_window(f, 64) - g['field_win']).max() / amax, 1e-6)
    within('c3.mdft_field_stride', np.abs(f[::16, ::16] - g['field_stride']).max() / amax, 1e-6)
    # CZT reaches the same answer (reference identity CZT == MDFT)
    ex2 = wf.prepare_executor(100.0, float(g['focal_dx']), M, kind='czt')
    f2 = host(wf.focus_dft(ex2).data)
    within('c3.czt_vs_mdft', np.abs(f2 - f).max() / amax, 1.2e-6)
    within('c3.czt_field_stride', np.abs(f2[::16, ::16] - g['field_stride']).max() / amax, 4.5e-7)
    pb.config.precision = 64


def test_polychromatic_recipe_small(pb):
    """docs/source/how-tos/Polychromatic Propagation.ipynb:86-98 at reduced size: loop over wavelengths,
    CZT focus to a common grid, weighted incoherent sum."""
    P = pb.propagation
    pb.config.precision = 32
    N, M = 128, 128
    amp, opd, dx = O.synthetic_pupil(N, np.float32)
    wvls = np.linspace(0.5, 0.7, 5)
    wts = np.full(5, 0.2)
    ref = np.zeros((M, M))
    acc = None
    planes = []
    for w, wt in zip(wvls, wts):
        ex_ref = O.prepare_executor(dx, (N, N), 2.5, (M, M), w, 100.0, kind='czt')
        ref += wt * O.intensity(ex_ref(O.from_amp_and_phase(amp, opd.astype(np.float64), w)))
        wf = P.Wavefront.from_amp_and_phase(amp, opd, w, dx)
        ex = wf.prepare_executor(100.0, 2.5, M, kind='czt')
        planes.append(wf.focus_dft(ex).intensity.data)
    total = pb.polynomials.sum_of_2d_modes(torch.stack(planes), wts)
    within('polychromatic_small', rel_linf(host(total), ref), TOL32)
    pb.config.precision = 64


# ------------------------------------------------------------------------------------------
# tensor-core matrix DFT against the CUDA-core GEMM and the oracle
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize('N,M', [(256, 128), (512, 256), (1024, 128)])
def test_mdft_tensor_core_path(pb, N, M):
    F = pb.fttools
    pb.config.precision = 32
    rng = np.random.default_rng(N + M)
    x = (np.arange(N) - N // 2) * 0.1
    f = (np.arange(M) - M // 2) * (0.37 / (N * 0.1))
    a = (rng.standard_normal((N, N)) + 1j * rng.standard_normal((N, N))).astype(np.complex64)
    ref = O.MDFT(x, x, f, f, -1, 0.5)(a.astype(np.complex128))
    tc = F.MDFT(x, x, f, f, -1, 0.5)
    assert tc._tc is not None, 'tensor-core plan should cover this shape'
    simt = F.MDFT(x, x, f, f, -1, 0.5, use_tensor_cores=False)
    assert simt._tc is None
    within(f'mdft_tc.{N}_{M}', rel_linf(host(tc(a)), ref), TOL32)          # 3xTF32 + chunked fp32 accumulation
    within(f'mdft_simt.{N}_{M}', rel_linf(host(simt(a)), ref), TOL32)
    # ragged shapes fall back to the CUDA-core GEMM
    assert F.MDFT(x[:100], x[:100], f[:50], f[:50])._tc is None
    pb.config.precision = 64


def test_mdft_tensor_core_stream_k(pb):
    """1024^2 -> 512^2 and its adjoint take the stream-K form of the GEMM on an H100: the first stage has 64 (forward)
    and 64 (adjoint, 512 rows x 2048 basis rows) tiles of 128 x 128, under 80 % of 132 SMs and at least a quarter of
    them, so one CTA per SM walks contiguous chunk ranges and tile owners gather the partials of their neighbours.
    Against the fp64 oracle, and bit for bit across repeated applies (the partials are added in a fixed order)."""
    F = pb.fttools
    pb.config.precision = 32
    N, M = 1024, 512
    rng = np.random.default_rng(7)
    x = (np.arange(N) - N // 2) * 0.1
    f = (np.arange(M) - M // 2) * (0.37 / (N * 0.1))
    a = (rng.standard_normal((N, N)) + 1j * rng.standard_normal((N, N))).astype(np.complex64)
    g = (rng.standard_normal((M, M)) + 1j * rng.standard_normal((M, M))).astype(np.complex64)
    ref = O.MDFT(x, x, f, f, -1, 0.5)
    tc = F.MDFT(x, x, f, f, -1, 0.5)
    assert tc._tc is not None and tc._tc_adj is not None, 'tensor-core plans should cover both directions'
    fwd = host(tc(a))
    adj = host(tc.adjoint(g))
    within(f'mdft_tc_streamk.{N}_{M}.fwd', rel_linf(fwd, ref(a.astype(np.complex128))), TOL32)
    within(f'mdft_tc_streamk.{N}_{M}.adj', rel_linf(adj, ref.adjoint(g.astype(np.complex128))), TOL32)
    for _ in range(2):
        assert np.array_equal(host(tc(a)), fwd)
        assert np.array_equal(host(tc.adjoint(g)), adj)
    pb.config.precision = 64
