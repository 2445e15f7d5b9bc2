"""CPU: the references of tests/sensing_reference.py against closed forms, the committed Bessel fixture against mpmath
(when it imports) and scipy, the lenslet-screen restatement against the reference's fixtures, and every defect model
against the GPU test's ceilings: each faithful model stays under its ceiling and each defect lands 10x or more above."""
import numpy as np
import pytest
import scipy.special as sps

import sensing_reference as S
from conftest import load_golden
from gpu_fixtures import crand
from test_gpu_sensing_vs_fp64 import CEIL


# ---- launch rules --------------------------------------------------------------------------------------------------
def test_launch_rules():
    assert (S.CENTROID_NCOLS_V4, S.CENTROID_NCOLS_MAX) == (614, 1075)
    assert [S.centroid_route(4096, k) for k in S.CENTROID_NCOLS] == [4, 1, 1, None]
    assert S.centroid_route(1025, 10) == 1 and S.centroid_route(1024, 10, aligned=False) == 1
    assert [S.overlap_launches(P) for P in S.OVERLAP_P] == [2, 2, 2, 2, 2, 2, 3, 4]
    assert [S.lp_launches(P) for P in S.LP_P] == [1, 1, 2, 3]
    assert [S.psi_width(t) for t in S.PSI_TYPES] == [4, 2, 8, 4]
    assert S.psi_route(4096, 'uint16') == 8 and S.psi_route(4097, 'uint16') == 1
    assert S.overlap_chunks(1024 ** 2 + 1) == S.THREADS + 1


# ---- closed forms --------------------------------------------------------------------------------------------------
def test_overlap_closed_forms():
    E = crand(5000, 1)
    orth = np.exp(2j * np.pi * np.arange(5000) / 5000)
    eta, maj, _, _ = S.overlap_ref(E, np.stack((E, 2.5j * E)))
    assert np.allclose(eta.astype(float), 1, rtol=0, atol=1e-18) and np.all(maj <= 1 + 1e-15)
    eta, _, _, _ = S.overlap_ref(np.ones(5000), orth[None])
    assert abs(float(eta[0])) < 1e-25


def test_psi_recovers_phase():
    ph = np.linspace(-3, 3, 101)
    for N in (3, 13, 64):
        g, s, c = S.fringes(N, 101, ph, np.float64)
        num, den, _, _ = S.psi_ref(g, s, c)
        assert np.max(np.abs(np.arctan2(num, den).astype(float) - ph)) < 1e-14


def test_centroid_single_pixel():
    xv, yv = np.arange(40.0) - 20, np.arange(20.0) - 10
    xc, yc = S.centres(10, 4), S.centres(10, 2)
    fr = np.zeros((1, 20, 40))
    fr[0, 13, 27] = 5.0
    d, f, _ = S.centroid_ref(fr, xv, yv, xc, yc, 10)
    i, j = S.owners(xv, xc, 10)[27], S.owners(yv, yc, 10)[13]
    assert d[0, 0, j, i] == xv[27] - xc[i] and d[0, 1, j, i] == yv[13] - yc[j] and f[0, j, i] == 5
    assert np.isnan(d[0, 0, 0, 0]) and f[0, 0, 0] == 0


def test_reconstruct_identity():
    s = np.random.default_rng(1).standard_normal((3, 50))
    idx = np.arange(50)
    out, mag = S.reconstruct_ref(s, idx, None, np.eye(50))
    assert np.array_equal(out.astype(float), s) and np.array_equal(mag.astype(float), np.abs(s))


def test_grating_mod_semantics():
    g = S.grating_rect_ref(np.array([-0.1, 0.0, -0.0, 0.3, 1e16]), 0.0, 0.3, 0.15, 1.0, 0.0, 0.5, 1e-12)
    assert list(g[:4]) == [0.0, 0.5, 0.5, 0.5]


# ---- the Bessel fixture --------------------------------------------------------------------------------------------
def test_bessel_fixture_vs_mpmath():
    pytest.importorskip('mpmath')
    z = load_golden(S.BESSEL_FIXTURE)
    rng = np.random.default_rng(0)
    for i in rng.choice(len(z['val']), 60, replace=False):
        want = S.mp_ratio(z['kind'][i], z['l'][i], z['arg'][i], z['rho'][i])
        assert abs(z['val'][i] - want) <= np.spacing(abs(want)), i


def test_bessel_fixture_vs_scipy():
    z = load_golden(S.BESSEL_FIXTURE)
    k, l, a, r, v = z['kind'], z['l'], z['arg'], z['rho'], z['val']
    j = k == 0
    sj = sps.jv(l[j], a[j] * r[j]) / sps.jv(l[j], a[j])
    kk = ~j
    sk = sps.kve(l[kk], a[kk] * r[kk]) / sps.kve(l[kk], a[kk]) * np.exp(a[kk] * (1 - r[kk]))
    ok = np.abs(v[j]) > 1e-280
    assert np.max(np.abs(sj[ok] - v[j][ok]) / np.maximum(np.abs(v[j][ok]), 1e-3)) < 1e-10
    assert np.max(np.abs(sk - v[kk]) / np.abs(v[kk])) < 1e-12


# ---- the lenslet screen restatement ------------------------------------------------------------------------------
@pytest.mark.parametrize('case', ('rect_edges', 'circle_edges'))
def test_screen_restatement_vs_fixtures(case):
    """the restatement's fp64 phase, through exp, matches the reference's screens (edges on samples, claimed by two to
    four lenslets) to 1e-12"""
    import shack_hartmann_oracle as O
    shape, dx, pitch, n, efl, aperture, kw, shift = O.CASES[case]
    assert kw is None and not shift
    x, y = O.grid(shape, dx)
    total = S.lenslet_phase(x, y, pitch, (n, n), efl, aperture)
    cr, ci = S.lenslet_field_ref(total, (-1j * 2 * np.pi / (O.WAVELENGTH / 1e3)).imag)
    got = load_golden('shack_hartmann.npz')['screen_' + case]
    assert max(np.max(np.abs(got.real - cr)), np.max(np.abs(got.imag - ci))) < 1e-12


# ---- defect models against the ceilings ----------------------------------------------------------------------------
def overlap_case(n, P, seed=3):
    E = crand(n, seed)
    M = crand((P, n), seed + 1)
    M[:, ::3] += 0.5 * E[::3]
    return E, M


@pytest.mark.parametrize('defect,n,P', [('f32', 3 * 4096 + 5, 3), ('drop_last_chunk', 4097, 2),
                                        ('stage2_256', 1024 ** 2 + 1, 1), ('e_twice', 5, 257)])
def test_overlap_defects(defect, n, P):
    E, M = overlap_case(n, P)
    eta, maj, _, _ = S.overlap_ref(E, M)
    assert S.overlap_fig(S.overlap_model(E, M), eta, maj) < CEIL['overlap']
    assert S.overlap_fig(S.overlap_model(E, M, defect), eta, maj) > 10 * CEIL['overlap']


def test_centroid_straddle_defect():
    W, pitch, V = 1030, 24, 1
    xv, yv = np.arange(W, dtype=np.float64) - W // 2, np.arange(48.0) - 23.5
    xc, yc = S.centres(pitch, W // pitch + 1), S.centres(pitch, 2)
    fr = np.random.default_rng(2).uniform(0, 1, (1, 48, W))
    d, _, sc = S.centroid_ref(fr, xv, yv, xc, yc, pitch)
    assert S.centroid_fig(S.centroid_model(fr, xv, yv, xc, yc, pitch, V), d, sc) < CEIL['centroid64']
    assert S.centroid_fig(S.centroid_model(fr, xv, yv, xc, yc, pitch, V, 'straddle'), d, sc) > 10 * CEIL['centroid32']


def test_psi_int_f64_defect():
    rng = np.random.default_rng(9)
    g = (2 ** 31 - 1 - rng.integers(0, 1000, (64, 500))).astype(np.int32)
    s = (rng.integers(-1, 2, 64) * 2 ** 26 + rng.integers(-999, 1000, 64) * 2 + 1).astype(np.float64)
    c = (rng.integers(0, 2, 64) * 2 ** 26 + rng.integers(-999, 1000, 64) * 2 + 1).astype(np.float64)
    en, ec = S.psi_int_ref(g, s, c)
    assert np.abs(en).max() > 2 ** 53
    fn, fc = S.psi_int_model(g, s, c, 'f64')
    assert not np.array_equal(fn, en) or not np.array_equal(fc, ec)


@pytest.mark.parametrize('defect', ('offset0', 'forward_below'))
def test_lp_defects(defect):
    z = load_golden(S.BESSEL_FIXTURE)
    sel = np.flatnonzero((z['kind'] == 0) & (z['l'] >= 2) & (z['l'] <= 30))
    sel = sel[np.linspace(0, len(sel) - 1, 200).astype(int)]
    cases = np.stack((z['l'][sel], z['arg'][sel], z['rho'][sel]), axis=1)
    ref = z['val'][sel]
    fig = lambda v: np.max(np.abs(v - ref) / np.maximum(np.abs(ref), 1.0))  # noqa: E731
    assert fig(S.lp_model(cases)) < CEIL['lp']
    assert not np.all(np.abs(S.lp_model(cases, defect) - ref) <= 10 * CEIL['lp'] * np.maximum(np.abs(ref), 1.0))


def test_reconstruct_gather_defect():
    rng = np.random.default_rng(4)
    idx = rng.permutation(512)[:257]
    R, ref = rng.standard_normal((10, 257)), rng.standard_normal(257) * 0.1
    s = rng.standard_normal((2, 512))
    want, mag = S.reconstruct_ref(s, idx, ref, R)
    fig = lambda v: float(np.max(np.abs(v - want) / mag))  # noqa: E731
    assert fig(S.reconstruct_model(s, idx, ref, R)) < CEIL['recon']
    assert fig(S.reconstruct_model(s, idx, ref, R, 'gather_m')) > 10 * CEIL['recon']
