"""CPU: the references of tests/test_gpu_streaming_vs_fp64.py (tests/streaming_reference.py) against closed forms and
the adjoint (dot-product) identity, and proof that the GPU test's ceilings would catch a subtly wrong kernel: each
faithful model lands under its ceiling and each modelled defect at least 10x above it."""
import math

import numpy as np
import pytest
import scipy.special as sps

import streaming_reference as S
from gpu_fixtures import crand
from streaming_reference import LD, LDBL, PB_C64, PB_C128, CEIL_ELEM, CEIL_RED


def rand(shape, seed, dt=np.float64):
    return np.random.default_rng(seed).standard_normal(shape).astype(dt)


# ---- launch geometry ------------------------------------------------------------------------------------------------
def test_launch_geometry():
    sm = 132
    assert S.grid_for(1, sm) == 1 and S.grid_for(S.sweep(sm), sm) == sm * 16
    assert S.grid_for(S.sweep(sm) + 1, sm) == sm * 16
    assert S.reduction_grid(S.reduction_cap(sm) + 1, sm) == sm * 4
    assert S.mode_projection_gx(10 ** 6, 1, sm) == sm * 4
    assert S.mode_projection_gx(10 ** 6, sm * 4 + 1, sm) == 1
    assert tuple(S.shapes(sm)) == S.SHAPE_NAMES
    counts = {a * b for a, b in S.shapes(sm).values()}
    for cap in (S.reduction_cap(sm), S.sweep(sm)):
        assert {cap - 1, cap, cap + 1} <= counts
    assert S.shapes(sm)['4096sq'] == (4096, 4096)


# ---- closed forms ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('shape', ((1, 1), (1, 1000), (1000, 1), (31, 33), (1023, 769)))
def test_moments_of_a_ramp(shape):
    ny, nx = shape
    d = np.add.outer(np.arange(ny) * 0.0, np.arange(nx, dtype=np.float64))      # d[y, x] = x
    (s0, sy, sx), (c0, _, _) = S.moments_ref(d)
    assert s0 == ny * nx * (nx - 1) // 2
    assert sy == (nx * (nx - 1) // 2) * (ny * (ny - 1) // 2)
    assert sx == ny * (nx - 1) * nx * (2 * nx - 1) // 6
    assert c0 == s0


def test_encircled_energy_of_a_delta_mtf():
    """an MTF that is 1 at the centre only: r j1(2 pi r 1e-16) / 1e-16 df^2 = pi r^2 df^2"""
    for shape in ((64, 64), (63, 65)):
        mtf = np.zeros(shape)
        mtf[S.centre_index(shape)] = 1
        radii = np.array([0.001, 0.01, 0.3])
        ee, cond = S.ee_ref(mtf, 0.5, radii)
        np.testing.assert_allclose(ee.astype(float), np.pi * radii ** 2 * 0.25, rtol=1e-15)
        assert np.all(cond >= np.abs(ee) * (1 - 1e-15))      # |j1(x)| <= x/2: equal here to rounding


@pytest.mark.parametrize('shape', ((16, 16), (15, 17), (1, 9), (8, 1)))
def test_packed_product_is_the_product_of_two_transforms(shape):
    rng = np.random.default_rng(3)
    o, h = rng.random(shape) * 1e5, rng.random(shape)
    s = 7.25
    Z = S.ft2_ld(S.ld(o) + 1j * s * S.ld(h))
    got = S.packed_product_ref(Z, 2.0, s)
    ref = 2.0 * S.ft2_ld(o) * S.ft2_ld(h)
    assert S.rel_linf(np.asarray(got, np.complex128), ref) < 1e-15
    assert float(np.abs(got - ref).max() / np.abs(ref).max()) < 1e-16      # long double, 1e5 : 1 in Z


@pytest.mark.parametrize('f', ((1, 7), (7, 1), (3, 5)))
def test_bindown_then_tile(f):
    fy, fx = f
    a = np.arange(2 * fy * 3 * fx, dtype=np.float64).reshape(2 * fy, 3 * fx)
    s = S.bindown_ref(a, fy, fx, mean=False)
    for (i, j), v in np.ndenumerate(s):
        assert v == a[i * fy:(i + 1) * fy, j * fx:(j + 1) * fx].sum()
    m = S.bindown_ref(a, fy, fx, mean=True)
    t = S.tile_ref(m, fy, fx, 1.0)
    assert t.shape == a.shape
    assert float(np.abs(S.bindown_ref(t, fy, fx, False) - s).max()) < 1e-12


def test_separable_tf_closed_forms():
    f = np.array([-2.0, -1.0, -0.5, 0.0, 0.5, 1.0, 2.0])
    tf = S.separable_tf_ref(0, f, f, 1.0, 1.0)
    assert tf[3, 3] == 1
    assert np.all(np.abs(tf[[0, 1, 5, 6], :]) < 1e-18)                # sinc zeros at integers
    np.testing.assert_allclose(tf[3].astype(float), np.sinc(f), rtol=1e-15, atol=1e-16)
    assert np.all(S.separable_tf_ref(0, f, f, 0.0, 0.0) == 1)
    np.testing.assert_allclose(S.separable_tf_ref(1, f, f, 0.3, 0.7).astype(float),
                               np.outer(np.cos(1.4 * f), np.cos(0.6 * f)), rtol=1e-15)


def test_resample_reference_edges():
    m = crand((5, 7), 1)
    ny, nx = m.shape
    # grid nodes come back exactly, the last row / column and -0.0 are inside, a coordinate one ulp (of the row /
    # column) outside either edge, or NaN, is the fill
    hy, hx = ny // 2, nx // 2
    xs = np.array([-hx, nx - 1 - hx, -0.0, nx - 1 - hx + np.spacing(nx - 1.0), np.nan, 0.5])
    ys = np.array([ny - 1 - hy, -hy, -0.0, 0.0, 0.0, np.nextafter(-hy, -np.inf)])
    got = S.resample_ref(m, xs, ys, 0.0, 0.0, 1.0, 9 + 9j)
    assert got[0] == m[ny - 1, 0] and got[1] == m[0, nx - 1] and got[2] == m[hy, hx]
    assert np.all(got[3:] == 9 + 9j)


def test_mask_one_minus_and_conj_commute():
    """conj(1 - m) = 1 - conj(m): the kernel's order of the two flags cannot matter; what can be wrong is a 1 - m
    that forgets to negate the imaginary part (the 'one_minus_re' defect below)"""
    a, m = crand(50, 1), crand(50, 2)
    ref = S.mask_multiply_ref(a, m, conj=True, one_minus=True)
    np.testing.assert_allclose(ref.astype(complex), a * (1 - np.conj(m)), rtol=1e-15)


# ---- adjoint identities ---------------------------------------------------------------------------------------------
def jvp(fwd, x, dx, eps):
    """long-double central difference (fwd(x + eps dx) - fwd(x - eps dx)) / 2 eps"""
    x, dx = S.ld(x), S.ld(dx)
    return (fwd(x + eps * dx) - fwd(x - eps * dx)) / (2 * eps)


def pair(a, b):
    """Re sum conj(a) b, and the sum of the terms' magnitudes"""
    t = (np.conj(S.ld(a)) * S.ld(b)).real
    return t.sum(), np.abs(t).sum()


def check_identity(ybar, jv, xbar, dx, tol=1e-9):
    """<ybar, J dx> = <J^T ybar, dx>, to tol relative to the sums of the terms' magnitudes"""
    (lhs, cl), (rhs, cr) = pair(ybar, jv), pair(xbar, dx)
    assert abs(lhs - rhs) <= tol * (cl + cr), (float(lhs), float(rhs))


def psf_for(shape, seed):
    rng = np.random.default_rng(seed)
    y, x = np.indices(shape) - np.array(shape)[:, None, None] // 2
    return np.exp(-(x * x + y * y) / (0.1 * shape[0] * shape[1])) + 0.05 * rng.random(shape)


@pytest.mark.parametrize('shape', ((16, 16), (15, 17)))
@pytest.mark.parametrize('which', (1, 2, 4))
def test_otf_from_psf_adjoint_identity(which, shape):
    psf, dpsf = psf_for(shape, 1), rand(shape, 2)
    bar = crand(shape, 3) if which == 4 else rand(shape, 3)
    pick = {1: 0, 2: 1, 4: 2}[which]

    def fwd(p):
        return S.mtf_ptf_otf_from_psf_ld(p)[pick]
    eps = LDBL(1e-10 if which == 2 else 1e-8)      # the phase is strongly curved where |D| is small
    jv = jvp(fwd, psf, dpsf, eps)
    if which == 2:      # angles: the difference of two phases, wrapped
        d = fwd(S.ld(psf) + eps * S.ld(dpsf)) - fwd(S.ld(psf) - eps * S.ld(dpsf))
        jv = (d - 2 * S.G.PI_LD * np.round(d / (2 * S.G.PI_LD))) / (2 * eps)
    check_identity(bar, jv, S.otf_from_psf_adjoint_ld(which, bar, psf), dpsf)


def test_encircled_energy_adjoint_identity():
    shape, dx = (32, 32), 0.5
    psf, dpsf = psf_for(shape, 4), rand(shape, 5)
    radii = np.array([0.002, 0.005, 0.011])
    ee_bar = np.array([0.3, -1.2, 2.0])
    jv = jvp(lambda p: S.encircled_energy_ld(np.asarray(p, np.float64), dx, radii), psf, dpsf, LDBL(1e-6))
    check_identity(ee_bar, jv, S.encircled_energy_adjoint_ld(ee_bar, psf, dx, radii), dpsf, tol=1e-8)


def test_from_amp_and_phase_adjoints():
    shape, k = (9, 11), 2 * np.pi / 0.6328e3
    amp, phase = 0.5 + np.random.default_rng(1).random(shape), 400 * rand(shape, 2)
    bar, dv = crand(shape, 3), rand(shape, 4)

    def field(a, p):
        return S.ld(a) * S.expi_ld(S.ld(p) * LDBL(k) / (2 * S.G.PI_LD))
    f = field(amp, phase)
    # phase: the kernel returns i * (true gradient), kept for parity with the reference
    g = S.field_adjoint_ref(0, f, bar, None, k)
    assert np.all(g.real == 0)
    check_identity(bar, jvp(lambda p: field(amp, p), phase, dv, LDBL(1e-6)), g.imag, dv)
    # amplitude, both branches: from the field (P / |P|) and from the phase
    jv = jvp(lambda a: field(a, phase), amp, dv, LDBL(1e-6))
    check_identity(bar, jv, S.field_adjoint_ref(1, f, bar, None, k), dv)
    check_identity(bar, jv, S.field_adjoint_ref(2, None, bar, phase, k), dv)
    f0 = f.copy()
    f0[0, 0] = 0
    assert S.field_adjoint_ref(1, f0, bar, None, k)[0, 0] == 0


def test_thin_lens_adjoint_identity():
    w, f = 0.6328e-3, 50.0
    x = np.linspace(-2, 2, 13)[None, :] + np.zeros((11, 1))
    y = np.linspace(-1.5, 1.5, 11)[:, None] + np.zeros((1, 13))
    rsq = S.ld(x * x + y * y)
    bar = crand(x.shape, 1)

    def lens(ff):
        return S.expi_ld(-rsq / (2 * ff) / LDBL(w))
    jv = (lens(LDBL(f) + LDBL(1e-6)) - lens(LDBL(f) - LDBL(1e-6))) / LDBL(2e-6)
    L = lens(LDBL(f))
    fbar = math.pi / (w * f * f) * S.dot_ref(bar, L, rsq)[0].imag
    check_identity(bar, jv, fbar, 1.0)


def test_intensity_adjoint_identity():
    E, dE, ibar = crand((7, 9), 1), crand((7, 9), 2), rand((7, 9), 3)
    jv = jvp(lambda e: np.abs(e) ** 2, E, dE, LDBL(1e-7))
    check_identity(ibar, jv, S.mask_multiply_ref(E, ibar, scale=2.0), dE)


def test_sum_of_2d_modes_adjoint_identity():
    modes, bar, dw = rand((5, 8, 9), 1), rand((8, 9), 2), rand(5, 3)
    jv = np.tensordot(S.ld(dw), S.ld(modes), axes=1)
    check_identity(bar, jv, S.mode_projection_ref(modes, bar)[0], dw, tol=1e-15)


# ---- faithful models under the ceilings, defects far above -----------------------------------------------------------
def defect_cases():
    """(name, ceiling, figure of the faithful model, figure of the defect)"""
    out = []
    shape = (16, 18)
    D = S.ft2_ld(psf_for(shape, 7)).astype(np.complex128)
    for which in (1, 2, 4):
        bar = crand(shape, 8) if which == 4 else rand(shape, 8)
        ref = S.otf_adjoint_seed_ref(which, bar, D)[0]
        faithful = np.asarray(ref, np.complex128)
        for d in ('no_centre', 'centre_nm1'):
            bad = np.asarray(S.otf_adjoint_seed_ref(which, bar, D, defect=d)[0], np.complex128)
            out.append((f'otf_seed/{which}/{d}', CEIL_ELEM[PB_C128], S.rel_linf(faithful, ref), S.rel_linf(bad, ref)))
    a, b, w = crand(4000, 1), crand(4000, 2), rand(4000, 3)
    ref, cond = S.dot_ref(a, b, w)
    out.append(('dot/conj_swap', CEIL_RED, S.red_fig(S.dot_model(a, b, w), ref, cond),
                S.red_fig(S.dot_model(a, b, w, 'conj_swap'), ref, cond)))
    for scale in (1e20, 1e-21):
        x, y = (crand(1000, 4) * scale).astype(np.complex64), (crand(1000, 5) * scale).astype(np.complex64)
        ref = S.binary_ref('truediv', x, y)
        out.append((f'truediv/{scale:g}/den_r', CEIL_ELEM[PB_C64], S.rel_linf(S.div_model(x, y, np.float32), ref),
                    S.rel_linf(S.div_model(x, y, np.float32, 'den_r'), ref)))
    a, m = crand(500, 6), crand(500, 7)
    ref = S.mask_multiply_ref(a, m, one_minus=True)
    out.append(('mask/one_minus_re', CEIL_ELEM[PB_C128], S.rel_linf(a * (1 - m), ref),
                S.rel_linf(np.asarray(S.mask_multiply_ref(a, m, one_minus=True, defect='one_minus_re'), complex), ref)))
    cmap = crand((6, 8), 9)
    xs = np.array([3.0, 3.0, -4.0, 0.5])
    ys = np.array([2.0, -3.0, 2.0, 2.0])
    ref = S.ld(S.resample_ref(cmap, xs, ys, 0.0, 0.0, 1.0, 0j))
    out.append(('resample/clamp_m1', CEIL_ELEM[PB_C128], S.rel_linf(S.resample_ref(cmap, xs, ys, 0, 0, 1, 0j), ref),
                S.rel_linf(S.resample_ref(cmap, xs, ys, 0, 0, 1, 0j, defect='clamp_m1'), ref)))
    modes, wts = rand((129, 300), 10), rand(129, 11)
    ref = S.weighted_sum_ref(modes, wts)
    out.append(('weighted_sum/no_accumulate', CEIL_ELEM[PB_C128], S.rel_linf(S.weighted_sum_model(modes, wts), ref),
                S.rel_linf(S.weighted_sum_model(modes, wts, 'no_accumulate'), ref)))
    for shape in ((16, 16), (15, 17), (1, 9)):
        Z = crand(shape, 12)
        ref = S.packed_product_ref(Z)
        out.append((f'packed/{shape}/mirror_nm1', CEIL_ELEM[PB_C128], S.rel_linf(np.asarray(ref, np.complex128), ref),
                    S.rel_linf(np.asarray(S.packed_product_ref(Z, defect='mirror_nm1'), np.complex128), ref)))
    return out


CASES = defect_cases()


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_defects_are_caught(case):
    name, ceiling, faithful, bad = case
    print(f'{name}: faithful {faithful:.2e}, defect {bad:.2e}, ceiling {ceiling:.0e}')
    assert faithful < ceiling, (name, faithful)
    assert bad >= 10 * ceiling, (name, bad)


def test_j1_reference():
    """scipy's j1 against its power series at small argument and a zero near 3.8317"""
    x = np.array([1e-16, 1e-8, 1e-3])
    np.testing.assert_allclose(sps.j1(x), x / 2 - x ** 3 / 16 + x ** 5 / 384, rtol=1e-15)
    assert abs(sps.j1(3.8317059702075123)) < 1e-15
