"""GPU: the streaming kernels every reverse pass and PSF metric runs through -- the adjoint seeds and elementwise twins
of csrc/adjoint_ops.cu, the non-transform kernels of csrc/elementwise.cu and the image chain of csrc/imagechain.cu --
held to the high-precision references of tests/streaming_reference.py over whole arrays.

Shapes come from the device's SM count: element counts on both sides of the one-sweep caps of grid_for (sm*16
blocks of 256) and of the reductions (sm*4 blocks), 1 x 1, 1 x n, n x 1, a partial warp, an odd shape, and 2048^2 and
4096^2, which take many grid-stride sweeps.  Inputs are drawn in fp64 and rounded to the run's dtype; the reference
gets the rounded values.

Figures: a reduction is |got - ref| / sum|terms| (ceiling 1e-13: both dtypes accumulate in fp64; encircled energy
1e-12 over a majorant of the terms, which includes the error of the device's fp64 j1); an elementwise output is max|got -
ref| / max|ref| (ceilings 1e-6 float32, 1e-14 float64: a few ulps of R).  Bounds are 1.5x the figures measured on an
H100 (`MEASURED`, recorded with PB_TEST_MEASUREMENTS) and never above the ceilings; every reduction folds its blocks in a
fixed order, so a figure is the same on every run.  The last test fails when a figure reached has no MEASURED entry.  Outputs that are exact by construction (re / im, the focal grids of radial_window,
tile, a closed-form sum beyond 2^31 elements) are compared bit for bit.

Every call also pins its launches (_ops.launch_count): one per entry point, two for otf_adjoint_seed, ceil(k/64) for
weighted_sum.

Ranges of the measured figures, H100 80GB HBM3 at a 700 W power limit: reductions 5.5e-18-1.3e-15 of sum|terms| (EE 8.5e-14); float64
elementwise 8.2e-17-4.9e-15; float32 elementwise 2.6e-8-4.4e-7.  Before complex
division was formed in fp64, test_otf_float32_psf_scale failed at 1e21 (mtf NaN) and 1e-22 (ptf 4.1e-3), and
test_truediv_range failed for float32 at 1e20 and 1e-21 (non-finite quotients).
"""
import math
import os

import numpy as np
import pytest
import torch

import streaming_reference as S
from accuracy import Ledger
from gpu_fixtures import pb, dev, host, launches, sm_count  # noqa: F401
from gpu_fixtures import crand as _crand
from streaming_reference import PB_C64, PB_C128, CEIL_ELEM, CEIL_RED, CEIL_EE

pytestmark = pytest.mark.gpu

DTS = (PB_C64, PB_C128)
DN = S.DT_NAME
TC = {PB_C64: torch.complex64, PB_C128: torch.complex128}
TR = {PB_C64: torch.float32, PB_C128: torch.float64}
SMALL = ('1x1', '1xn', 'nx1', '31x33', '1023x769')

# ---- measured figures (H100 80GB HBM3, 700 W power limit); bounds are 1.5x these, capped at the ceiling ----------
MEASURED = {
    'c128/balance_scale': 9.89e-17,
    'c128/binary_add': 8.94e-17,
    'c128/binary_mul': 1.22e-16,
    'c128/binary_sub': 8.39e-17,
    'c128/binary_truediv': 4.73e-16,
    'c128/bindown': 3.83e-16,
    'c128/component_abs': 1.48e-16,
    'c128/component_angle': 1.46e-16,
    'c128/conv': 4.10e-15,
    'c128/dot': 4.53e-17,
    'c128/dot_w': 6.78e-17,
    'c128/ee_adjoint': 9.49e-16,
    'c128/ee_adjoint_seed': 2.82e-15,
    'c128/encircled_energy': 8.52e-14,
    'c128/field_adjoint_0': 1.48e-16,
    'c128/field_adjoint_1': 2.38e-16,
    'c128/field_adjoint_2': 1.59e-16,
    'c128/intensity': 1.95e-16,
    'c128/mask_multiply': 2.79e-16,
    'c128/mask_multiply_shapes': 1.93e-16,
    'c128/mode_projection': 1.11e-17,
    'c128/mode_projection_c': 8.77e-18,
    'c128/moments': 1.00e-16,
    'c128/mul_outer': 1.99e-16,
    'c128/otf_normalize_mtf': 2.69e-16,
    'c128/otf_normalize_otf': 1.73e-16,
    'c128/otf_normalize_ptf': 1.74e-16,
    'c128/otf_seed_1': 2.86e-16,
    'c128/otf_seed_1_centre': 6.59e-17,
    'c128/otf_seed_2': 1.81e-16,
    'c128/otf_seed_2_centre': 4.32e-18,
    'c128/otf_seed_4': 2.22e-16,
    'c128/otf_seed_4_centre': 1.10e-16,
    'c128/pack': 8.23e-17,
    'c128/packed_product': 1.13e-16,
    'c128/phase_screen': 1.50e-16,
    'c128/psf_adjoint_1': 7.62e-16,
    'c128/psf_adjoint_2': 1.20e-15,
    'c128/psf_adjoint_4': 8.46e-16,
    'c128/radial_window': 1.06e-15,
    'c128/resample': 2.85e-16,
    'c128/separable_tf_0': 2.84e-16,
    'c128/separable_tf_1': 1.74e-16,
    'c128/truediv_huge': 4.31e-16,
    'c128/truediv_tiny': 4.17e-16,
    'c128/vortex': 4.90e-15,
    'c128/weighted_sum': 5.46e-16,
    'c64/balance_scale': 8.69e-17,
    'c64/binary_add': 4.54e-08,
    'c64/binary_mul': 7.23e-08,
    'c64/binary_sub': 4.40e-08,
    'c64/binary_truediv': 5.94e-08,
    'c64/bindown': 9.90e-08,
    'c64/component_abs': 6.74e-08,
    'c64/component_angle': 8.80e-08,
    'c64/conv': 4.42e-07,
    'c64/dot': 8.10e-18,
    'c64/dot_w': 3.78e-17,
    'c64/ee_adjoint': 3.04e-07,
    'c64/ee_adjoint_seed': 2.58e-08,
    'c64/encircled_energy': 8.52e-14,
    'c64/field_adjoint_0': 7.95e-08,
    'c64/field_adjoint_1': 1.21e-07,
    'c64/field_adjoint_2': 1.17e-07,
    'c64/intensity': 9.91e-08,
    'c64/mask_multiply': 1.25e-07,
    'c64/mask_multiply_shapes': 8.99e-08,
    'c64/mode_projection': 8.64e-18,
    'c64/mode_projection_c': 5.52e-18,
    'c64/moments': 1.25e-16,
    'c64/mul_outer': 1.26e-07,
    'c64/otf_normalize_mtf': 8.79e-08,
    'c64/otf_normalize_otf': 4.52e-08,
    'c64/otf_normalize_ptf': 9.78e-08,
    'c64/otf_scale_1_mtf': 4.83e-08,
    'c64/otf_scale_1_otf': 2.82e-08,
    'c64/otf_scale_1_ptf': 8.61e-08,
    'c64/otf_scale_1e+21_mtf': 6.09e-08,
    'c64/otf_scale_1e+21_otf': 2.71e-08,
    'c64/otf_scale_1e+21_ptf': 8.81e-08,
    'c64/otf_scale_1e-22_mtf': 3.93e-08,
    'c64/otf_scale_1e-22_otf': 2.60e-08,
    'c64/otf_scale_1e-22_ptf': 8.55e-08,
    'c64/otf_seed_1': 4.44e-08,
    'c64/otf_seed_1_centre': 3.66e-10,
    'c64/otf_seed_2': 3.21e-08,
    'c64/otf_seed_2_centre': 4.28e-10,
    'c64/otf_seed_4': 4.41e-08,
    'c64/otf_seed_4_centre': 1.32e-09,
    'c64/pack': 3.96e-08,
    'c64/packed_product': 9.06e-08,
    'c64/phase_screen': 1.46e-07,
    'c64/psf_adjoint_1': 2.77e-07,
    'c64/psf_adjoint_2': 3.46e-07,
    'c64/psf_adjoint_4': 3.06e-07,
    'c64/radial_window': 2.98e-08,
    'c64/resample': 3.70e-08,
    'c64/separable_tf_0': 2.98e-08,
    'c64/separable_tf_1': 2.98e-08,
    'c64/truediv_huge': 5.95e-08,
    'c64/truediv_tiny': 5.90e-08,
    'c64/vortex': 1.37e-07,
    'c64/weighted_sum': 2.75e-07,
}

REDUCTIONS = {'dot', 'dot_w', 'mode_projection', 'mode_projection_c', 'moments', 'balance_scale'}


def ceiling(name):
    dn, fig = name.split('/', 1)
    if fig == 'encircled_energy':
        return CEIL_EE
    return CEIL_RED if fig in REDUCTIONS else CEIL_ELEM[PB_C64 if dn == DN[PB_C64] else PB_C128]


# the largest figure of each name over the whole file, against 1.5x its MEASURED value, never above the ceiling
LEDGER = Ledger(MEASURED, ceiling)
check = LEDGER.check


# ---- helpers ----------------------------------------------------------------------------------------------------------
def shape_of(name):
    return S.shapes(sm_count())[name]


def crand(shape, seed, dt, scale=1.0):
    return _crand(shape, seed, S.CDT[dt], scale)


def rand(shape, seed, dt, scale=1.0):
    return (np.random.default_rng(seed).standard_normal(shape) * scale).astype(S.RDT[dt])


def wrap(a):
    """an angle difference folded into [-pi, pi]"""
    return a - 2 * np.pi * np.round(a / (2 * np.pi))


# ---- reductions -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('weighted', (False, True))
@pytest.mark.parametrize('shape', S.SHAPE_NAMES)
@pytest.mark.parametrize('dt', DTS)
def test_dot(pb, dt, shape, weighted):
    sh = shape_of(shape)
    a, b = crand(sh, 1, dt), crand(sh, 2, dt)
    w = rand(sh, 3, dt) if weighted else None
    got, n = launches(pb, lambda: pb._ops.dot(dev(a), dev(b), None if w is None else dev(w)))
    ref, cond = S.dot_ref(a, b, w)
    assert n == 1
    check(f'{DN[dt]}/dot{"_w" if weighted else ""}', S.red_fig(got, ref, cond))


@pytest.mark.parametrize('cplx', (False, True))
@pytest.mark.parametrize('k', ('1', '64', '65', 'sm*4+1'))
@pytest.mark.parametrize('dt', DTS)
def test_mode_projection(pb, dt, k, cplx):
    """k = 1 and 64 take many blocks per mode; sm*4+1 modes leave one block to read a whole mode"""
    k = sm_count() * 4 + 1 if k == 'sm*4+1' else int(k)
    sh = (255, 383)
    modes = rand((k,) + sh, 4, dt)
    bar = crand(sh, 5, dt) if cplx else rand(sh, 5, dt)
    got, n = launches(pb, lambda: pb._ops.mode_projection(dev(modes), dev(bar)))
    ref, cond = S.mode_projection_ref(modes, bar)
    assert n == 1 and got.shape == (k,)
    if k == sm_count() * 4 + 1:
        assert S.mode_projection_gx(sh[0] * sh[1], k, sm_count()) == 1
    check(f'{DN[dt]}/mode_projection{"_c" if cplx else ""}', S.red_fig(got, ref, cond))


@pytest.mark.parametrize('shape', S.SHAPE_NAMES)
@pytest.mark.parametrize('dt', DTS)
def test_moments(pb, dt, shape):
    sh = shape_of(shape)
    d = rand(sh, 6, dt) + S.RDT[dt](0.5)
    got, n = launches(pb, lambda: pb._ops.moments(dev(d)))
    ref, cond = S.moments_ref(d)
    assert n == 1
    check(f'{DN[dt]}/moments', S.red_fig(np.array(got), ref, cond))


@pytest.mark.parametrize('nr', (1, 40))
@pytest.mark.parametrize('shape', ('1x1', '31x33', '1023x769', 'red+1', 'elem+1'))
@pytest.mark.parametrize('dt', DTS)
def test_encircled_energy(pb, dt, shape, nr):
    sh = shape_of(shape)
    mtf = np.abs(rand(sh, 7, dt))
    df = 0.37
    radii = np.linspace(0.05, 40.0, nr) / df
    got, n = launches(pb, lambda: pb._ops.encircled_energy(dev(mtf), df, radii))
    ref, cond = S.ee_ref(mtf, df, radii)
    assert n == 1
    check(f'{DN[dt]}/encircled_energy', S.red_fig(got, ref, cond))


@pytest.mark.parametrize('shape', SMALL + ('red+1', 'elem+1', '2048sq'))
@pytest.mark.parametrize('dt', DTS)
def test_balance_scale_one_launch(pb, dt, shape):
    """the folded reduction and its sqrt epilogue run in one launch, no finalize kernel after it"""
    sh = shape_of(shape)
    a, b = rand(sh, 8, dt, 1e3), rand(sh, 9, dt)
    got, n = launches(pb, lambda: pb._ops.balance_scale(dev(a), dev(b)))
    ref, (sa, sb) = S.balance_ref(a, b)
    assert n == 1
    # s = sqrt(sa / sb): its relative error is half the sum of the two sums' relative errors
    check(f'{DN[dt]}/balance_scale', abs(float(host(got)[0]) - ref) / ref)


@pytest.mark.parametrize('dt', DTS)
def test_balance_scale_fallback(pb, dt):
    a, b = rand((31, 33), 10, dt), rand((31, 33), 11, dt)
    z = np.zeros_like(b)
    bad = a.copy()
    bad[3, 4] = np.inf
    nan = a.copy()
    nan[0, 0] = np.nan
    for x, y in ((a, z), (z, b), (bad, b), (a, bad), (nan, b)):
        assert float(host(pb._ops.balance_scale(dev(x), dev(y)))[0]) == 1.0


# ---- OTF path -------------------------------------------------------------------------------------------------------
def otf_figures(got, ref, which):
    """figures of (mtf, ptf, otf) outputs of which; the phase is compared as a wrapped angle over pi"""
    out = {}
    if which & 1:
        out['mtf'] = S.rel_linf(host(got[0]), ref[0])
    if which & 2:
        g = host(got[1])
        out['ptf'] = math.inf if not np.all(np.isfinite(g)) else \
            float(np.abs(wrap((S.ld(g) - ref[1]).astype(np.float64))).max()) / np.pi
    if which & 4:
        out['otf'] = S.rel_linf(host(got[2]), ref[2])
    return out


@pytest.mark.parametrize('shape', ('1x1', '1xn', 'nx1', '31x33', '1023x769', '2048sq', 'elem+1'))
@pytest.mark.parametrize('which', (1, 2, 4, 7))
@pytest.mark.parametrize('dt', DTS)
def test_otf_normalize(pb, dt, which, shape):
    sh = shape_of(shape)
    D = crand(sh, 12, dt)
    got, n = launches(pb, lambda: pb._ops.otf_normalize(dev(D), which))
    assert n == 1
    assert [g is not None for g in got] == [bool(which & 1), bool(which & 2), bool(which & 4)]
    for k, v in otf_figures(got, S.otf_normalize_ref(D), which).items():
        check(f'{DN[dt]}/otf_normalize_{k}', v)


@pytest.mark.parametrize('scale', (1e-22, 1.0, 1e21))
def test_otf_float32_psf_scale(pb, scale):
    """a float32 PSF in absolute units: the centre sample (the PSF's sum) is far from 1, and the normalisation divides
    by it.  Formed in float32, |c|^2 overflows above ~1.8e19 (NaN) and loses bits below ~1e-19."""
    sh = (256, 256)
    y, x = np.indices(sh) - 128
    psf = ((np.exp(-(x * x + y * y) / 200.0) + 0.01 * np.random.default_rng(13).random(sh)) * scale).astype(np.float32)
    pb.config.precision = 32
    try:
        mtf, ptf, otf, data = pb.otf.mtf_ptf_otf_from_psf(psf, 1.0, return_more=True)
    finally:
        pb.config.precision = 64
    D = host(data)
    assert np.all(np.isfinite(D))
    ref = S.otf_normalize_ref(D)
    for k, v in otf_figures((mtf.data, ptf.data, otf.data), ref, 7).items():
        check(f'c64/otf_scale_{scale:g}_{k}', v)


@pytest.mark.parametrize('shape', ('1x1', '1xn', 'nx1', '31x33', '1023x769', '2048sq', 'red+1', 'elem+1'))
@pytest.mark.parametrize('which', (1, 2, 4))
@pytest.mark.parametrize('dt', DTS)
def test_otf_adjoint_seed(pb, dt, which, shape):
    sh = shape_of(shape)
    D = crand(sh, 14, dt)
    bar = crand(sh, 15, dt) if which == 4 else rand(sh, 15, dt)
    got, n = launches(pb, lambda: pb._ops.otf_adjoint_seed(which, dev(bar), dev(D)))
    assert n == 2
    got = host(got)
    ref = S.otf_adjoint_seed_ref(which, bar, D)[0]
    _, Sref, Scond = S.otf_adjoint_seed_ref(which, bar, D)
    main = S.otf_adjoint_seed_ref(which, bar, D, defect='no_centre')[0]
    c = S.centre_index(sh)
    corr = main[c] - ref[c]
    err = np.abs(S.ld(got) - ref)
    # off the centre: relative to the largest term (the reduction does not enter)
    off = err.copy()
    off[c] = 0
    check(f'{DN[dt]}/otf_seed_{which}', float(off.max() / np.abs(main).max()))
    # the centre, relative to its first term and to its correction at the reduction's scale sum|terms| (the
    # correction is linear in S, so its error is S's error at that scale); for a 1 x 1
    # plane the two terms cancel exactly (zero gradient)
    scale = abs(main[c]) + abs(corr) * Scond / max(abs(Sref), np.finfo(np.float64).tiny)
    check(f'{DN[dt]}/otf_seed_{which}_centre', float(err[c] / scale))


@pytest.mark.parametrize('shape', ('1x1', '31x33', '1023x769', 'elem+1'))
@pytest.mark.parametrize('dt', DTS)
def test_encircled_energy_adjoint_seed(pb, dt, shape):
    sh = shape_of(shape)
    df = 0.37
    radii = np.linspace(0.05, 40.0, 40) / df
    ee_bar = np.random.default_rng(16).standard_normal(40)
    got, n = launches(pb, lambda: pb._ops.encircled_energy_adjoint_seed(sh, df, radii, ee_bar, TR[dt], 'cuda'))
    assert n == 1
    check(f'{DN[dt]}/ee_adjoint_seed', S.rel_linf(host(got), S.ee_adjoint_seed_ref(sh, df, radii, ee_bar)))


# ---- elementwise ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('with_w', (False, True))
@pytest.mark.parametrize('with_b', (False, True))
@pytest.mark.parametrize('mcplx', (False, True))
@pytest.mark.parametrize('flags', range(16))
@pytest.mark.parametrize('dt', DTS)
def test_mask_multiply_flags(pb, dt, flags, mcplx, with_b, with_w):
    conj, one_minus, real_out, acc = (bool(flags & f) for f in (1, 2, 4, 8))
    sh = (31, 33)
    a = crand(sh, 17, dt)
    m = crand(sh, 18, dt) if mcplx else rand(sh, 18, dt)
    b = crand(sh, 19, dt) if with_b else None
    w = rand(sh, 20, dt) if with_w else None
    out0 = (rand(sh, 21, dt) if real_out else crand(sh, 21, dt)) if acc else None
    o = None if out0 is None else dev(out0)
    got, n = launches(pb, lambda: pb._ops.mask_multiply(dev(a), dev(m), b=None if b is None else dev(b),
                                                       w=None if w is None else dev(w), conj=conj,
                                                       one_minus=one_minus, real_out=real_out, scale=0.7, out=o))
    assert n == 1 and got.is_complex() != real_out
    ref = S.mask_multiply_ref(a, m, b, w, conj, one_minus, real_out, 0.7, out0, rdt=S.RDT[dt])
    check(f'{DN[dt]}/mask_multiply', S.rel_linf(host(got), ref))


@pytest.mark.parametrize('shape', S.SHAPE_NAMES)
@pytest.mark.parametrize('dt', DTS)
def test_mask_multiply_shapes(pb, dt, shape):
    sh = shape_of(shape)
    a, m, w = crand(sh, 22, dt), crand(sh, 23, dt), rand(sh, 24, dt)
    got = pb._ops.mask_multiply(dev(a), dev(m), w=dev(w), conj=True, one_minus=True, scale=2.0)
    check(f'{DN[dt]}/mask_multiply_shapes',
          S.rel_linf(host(got), S.mask_multiply_ref(a, m, None, w, True, True, False, 2.0)))


@pytest.mark.parametrize('mode', (0, 1, 2))
@pytest.mark.parametrize('shape', ('1x1', '31x33', '1023x769', 'elem+1'))
@pytest.mark.parametrize('dt', DTS)
def test_field_adjoint(pb, dt, shape, mode):
    sh = shape_of(shape)
    k = 2 * np.pi / 0.6328e3
    f, bar, opd = crand(sh, 25, dt), crand(sh, 26, dt), rand(sh, 27, dt, 300.0)
    f.reshape(-1)[::7] = 0                                    # zero field: mode 1 returns 0 there
    got, n = launches(pb, lambda: pb._ops.field_adjoint(mode, dev(f) if mode < 2 else None, dev(bar),
                                                         dev(opd) if mode == 2 else None, k))
    assert n == 1
    g = host(got)
    ref = S.field_adjoint_ref(mode, f, bar, opd, k)
    if mode == 0:
        assert np.all(g.real == 0)
    if mode == 1:
        assert np.all(g.reshape(-1)[::7] == 0)
    check(f'{DN[dt]}/field_adjoint_{mode}', S.rel_linf(g, ref))


@pytest.mark.parametrize('which', ('real', 'imag', 'angle', 'abs'))
@pytest.mark.parametrize('shape', ('1x1', '31x33', '1023x769', 'elem+1'))
@pytest.mark.parametrize('dt', DTS)
def test_component(pb, dt, shape, which):
    sh = shape_of(shape)
    v = crand(sh, 28, dt)
    zeros = np.zeros(4, dtype=S.CDT[dt])
    zeros.real = np.array([0.0, 0.0, -0.0, -0.0])
    zeros.imag = np.array([0.0, -0.0, 0.0, -0.0])
    flat = v.reshape(-1)
    flat[:min(4, flat.size)] = zeros[:min(4, flat.size)]
    got, n = launches(pb, lambda: pb._ops.component(which, dev(v)))
    assert n == 1
    g = host(got)
    if which in ('real', 'imag'):
        assert np.array_equal(g.view(np.uint8), getattr(v, which).copy().view(np.uint8))
        return
    if which == 'angle':     # atan2 of signed zeros: +-0 and +-pi with numpy's signs
        z = flat[:min(4, flat.size)]
        np.testing.assert_array_equal(g.reshape(-1)[:z.size], np.arctan2(z.imag, z.real))
        assert np.array_equal(np.signbit(g.reshape(-1)[:z.size]), np.signbit(np.arctan2(z.imag, z.real)))
    check(f'{DN[dt]}/component_{which}', S.rel_linf(g, S.component_ref(which, v)))


@pytest.mark.parametrize('scalar', (False, True))
@pytest.mark.parametrize('reverse', (False, True))
@pytest.mark.parametrize('op', ('mul', 'truediv', 'add', 'sub'))
@pytest.mark.parametrize('shape', ('1x1', '31x33', '1023x769', 'elem+1'))
@pytest.mark.parametrize('dt', DTS)
def test_binary(pb, dt, shape, op, reverse, scalar):
    sh = shape_of(shape)
    a, b = crand(sh, 29, dt), crand(sh, 30, dt)
    bb = complex(b.reshape(-1)[0]) if scalar else b
    got, n = launches(pb, lambda: pb._ops.binary(op, dev(a), bb if scalar else dev(b), reverse))
    assert n == 1
    ref = S.binary_ref(op, a, np.full(sh, bb, dtype=S.CDT[dt]) if scalar else b, reverse)
    # division: relative to each quotient (|a/b| spans decades), everything else: to max|ref|
    g = host(got)
    fig = float(np.max(np.abs(S.ld(g) - ref) / np.abs(ref))) if op == 'truediv' else S.rel_linf(g, ref)
    check(f'{DN[dt]}/binary_{op}', fig)


@pytest.mark.parametrize('scale', ('tiny', 'huge'))
@pytest.mark.parametrize('dt', DTS)
def test_truediv_range(pb, dt, scale):
    """a / b with both far from 1: float32 1e-21 and 1e20 (past the float32 |b|^2 range), float64 1e-150 and 1e150"""
    s = {PB_C64: {'tiny': 1e-21, 'huge': 1e20}, PB_C128: {'tiny': 1e-150, 'huge': 1e150}}[dt][scale]
    sh = (1023, 769)
    a, b = crand(sh, 31, dt, s), crand(sh, 32, dt, s)
    g = host(pb._ops.binary('truediv', dev(a), dev(b)))
    ref = S.binary_ref('truediv', a, b)
    fig = math.inf if not np.all(np.isfinite(g)) else float(np.max(np.abs(S.ld(g) - ref) / np.abs(ref)))
    check(f'{DN[dt]}/truediv_{scale}', fig)


@pytest.mark.parametrize('dt', DTS)
def test_mul_outer_strided(pb, dt):
    big = crand((300, 400), 33, dt)
    vy, vx = crand(200, 34, dt), crand(311, 35, dt)
    a = dev(big)[50:250, 20:331]                              # row stride 400
    out_big = torch.zeros((210, 350), dtype=TC[dt], device='cuda')
    out = out_big[5:205, 7:318]
    for cy, cx in ((False, False), (True, False), (False, True), (True, True)):
        got, n = launches(pb, lambda: pb._ops.mul_outer(a, dev(vy), dev(vx), cy, cx, 0.3, out=out))
        assert n == 1 and got.data_ptr() == out.data_ptr()
        ref = S.mul_outer_ref(big[50:250, 20:331], vy, vx, cy, cx, 0.3, rdt=S.RDT[dt])
        check(f'{DN[dt]}/mul_outer', S.rel_linf(host(out), ref))
        ob = host(out_big)
        assert not ob[:5].any() and not ob[205:].any() and not ob[:, :7].any() and not ob[:, 318:].any()


@pytest.mark.parametrize('k', (64, 65, 129))
@pytest.mark.parametrize('dt', DTS)
def test_weighted_sum(pb, dt, k):
    sh = (255, 383)
    modes = rand((k,) + sh, 36, dt)
    w = np.random.default_rng(37).standard_normal(k)
    got, n = launches(pb, lambda: pb._ops.weighted_sum(dev(modes), w))
    assert n == -(-k // S.PB_MAX_MODES)
    ref = S.weighted_sum_ref(modes, w, S.RDT[dt])
    # a k-term sum in R: relative to the sum of the terms' magnitudes at each sample
    cond = np.tensordot(np.abs(S.ld(np.asarray(w).astype(S.RDT[dt]))), np.abs(S.ld(modes)), axes=1)
    check(f'{DN[dt]}/weighted_sum', float(np.max(np.abs(S.ld(host(got)) - ref) / cond)))


@pytest.mark.parametrize('charge', (1, 6))
@pytest.mark.parametrize('dt', DTS)
def test_vortex_phase(pb, dt, charge):
    sh = (255, 383)
    xf, yf = S.radial_axes_ref(sh, 0.013, 0.0, S.RDT[dt])
    got, n = launches(pb, lambda: pb._ops.vortex_phase(charge, dev(xf), dev(yf)))
    assert n == 1
    check(f'{DN[dt]}/vortex', S.rel_linf(host(got), S.vortex_ref(charge, xf, yf)))


@pytest.mark.parametrize('levels', ('outer', 'middle', 'inner'))
@pytest.mark.parametrize('shape', ('1x1', '31x33', '1023x769', 'elem+1'))
@pytest.mark.parametrize('dt', DTS)
def test_radial_window(pb, dt, shape, levels):
    sh = shape_of(shape)
    fdx, shift = 0.0137, 0.5 * 0.0137 * (sh[1] % 2 == 0)
    here, nxt = {'outer': (None, (2.0, 3.5)), 'middle': ((4.0, 6.0), (1.0, 1.7)), 'inner': ((0.5, 3.0), None)}[levels]
    (win, xf, yf), n = launches(pb, lambda: pb._ops.radial_window(sh, fdx, shift, here, nxt, TR[dt], 'cuda'))
    assert n == 1
    xr, yr = S.radial_axes_ref(sh, fdx, shift, S.RDT[dt])
    assert np.array_equal(host(xf), xr) and np.array_equal(host(yf), yr)
    check(f'{DN[dt]}/radial_window', S.rel_linf(host(win), S.radial_window_ref(xr, yr, here, nxt)))


@pytest.mark.parametrize('dt', DTS)
def test_resample_bilinear_edges(pb, dt):
    R = S.RDT[dt]
    ny, nx = 48, 65
    hy, hx = ny // 2, nx // 2
    cmap = crand((ny, nx), 38, dt)
    rng = np.random.default_rng(39)
    # in R, the coordinates are the rows / columns minus n//2: nodes, the last row and column exactly, -0.0, one ulp
    # (of the row / column) outside each edge, NaN, and interior points
    edge_x = [-hx, nx - 1 - hx, -0.0, 0.0, R(nx - 1 - hx) + np.spacing(R(nx - 1)), R(-hx) - np.spacing(R(hx)),
              np.nan, 0.0, 3.25]
    edge_y = [ny - 1 - hy, -hy, -0.0, R(ny - 1 - hy) + np.spacing(R(ny - 1)), 0.0, 0.0, 0.0, np.nan,
              R(-hy) - np.spacing(R(hy))]
    xf = np.concatenate([np.array(edge_x, R), rng.uniform(-hx - 2, nx - hx + 1, 5000).astype(R)])
    yf = np.concatenate([np.array(edge_y, R), rng.uniform(-hy - 2, ny - hy + 1, 5000).astype(R)])
    for fill in (0.25 - 0.5j, 'tensor'):
        ft = crand(xf.shape, 40, dt) if fill == 'tensor' else None
        got, n = launches(pb, lambda: pb._ops.resample_bilinear(dev(cmap), dev(xf), dev(yf), 0.0, 0.0, 1.0,
                                                                 dev(ft) if ft is not None else fill))
        assert n == 1
        g = host(got)
        ref = S.resample_ref(cmap, xf, yf, 0.0, 0.0, 1.0, ft if ft is not None else fill)
        assert g[0] == cmap[ny - 1, 0] and g[1] == cmap[0, nx - 1] and g[2] == cmap[hy, hx]
        assert np.array_equal(g[3:9], ref[3:9].astype(g.dtype))           # outside / NaN: the fill, exactly
        check(f'{DN[dt]}/resample', S.rel_linf(g, ref))


@pytest.mark.parametrize('amp', ('none', 'real', 'u8'))
@pytest.mark.parametrize('shape', ('1x1', '31x33', '1023x769', 'elem+1'))
@pytest.mark.parametrize('dt', DTS)
def test_phase_screen(pb, dt, shape, amp):
    sh = shape_of(shape)
    k = 2 * np.pi / 0.6328e3
    opd = rand(sh, 41, dt, 500.0)
    a = {'none': None, 'real': np.abs(rand(sh, 42, dt)), 'u8': (rand(sh, 42, dt) > 0).astype(np.uint8)}[amp]
    got, n = launches(pb, lambda: pb._ops.phase_screen(None if a is None else dev(a), dev(opd), k))
    assert n == 1
    check(f'{DN[dt]}/phase_screen', S.rel_linf(host(got), S.phase_field_ld(opd, k, a)))


@pytest.mark.parametrize('accumulate', (False, True))
@pytest.mark.parametrize('shape', S.SHAPE_NAMES)
@pytest.mark.parametrize('dt', DTS)
def test_intensity(pb, dt, shape, accumulate):
    sh = shape_of(shape)
    v = crand(sh, 43, dt)
    out0 = np.abs(rand(sh, 44, dt)) if accumulate else None
    o = None if out0 is None else dev(out0)
    got, n = launches(pb, lambda: pb._ops.intensity(dev(v), 0.75, out=o))
    assert n == 1
    check(f'{DN[dt]}/intensity', S.rel_linf(host(got), S.intensity_ref(v, 0.75, out0, S.RDT[dt])))


# ---- image chain ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('shape', ((1, 9), (8, 1), (15, 17), (16, 16), (255, 383), (256, 256)))
@pytest.mark.parametrize('dt', DTS)
def test_pack_and_packed_product_one_launch_each(pb, dt, shape):
    """pack o + i s h on the device, transform it in long double on the host, and form O H from that Z on the device"""
    rng = np.random.default_rng(45)
    o = (rng.random(shape) * 1e5).astype(S.RDT[dt])
    h = rng.random(shape).astype(S.RDT[dt])
    s, n0 = launches(pb, lambda: pb._ops.balance_scale(dev(o), dev(h)))
    zp, n1 = launches(pb, lambda: pb._ops.pack_complex(dev(o), dev(h), s))
    assert n0 == 1 and n1 == 1
    sv = float(host(s)[0])
    zh = host(zp)
    assert np.array_equal(zh.real, o)
    check(f'{DN[dt]}/pack', S.rel_linf(zh.imag, S.ld(h) * S.ld(S.RDT[dt](sv))))
    Z = np.asarray(S.ft2_ld(zh), S.CDT[dt])
    got, n = launches(pb, lambda: pb._ops.packed_spectrum_product(dev(Z), 0.5, s))
    assert n == 1
    check(f'{DN[dt]}/packed_product', S.rel_linf(host(got), S.packed_product_ref(Z, 0.5, sv)))


@pytest.mark.parametrize('dt', DTS)
def test_conv_end_to_end(pb, dt):
    """an object of sum 1e5 convolved with a unit-sum PSF against a long-double circular convolution"""
    sh = (256, 255)
    rng = np.random.default_rng(46)
    o = rng.random(sh)
    o = (o * (1e5 / o.sum())).astype(S.RDT[dt])
    y, x = np.indices(sh) - np.array(sh)[:, None, None] // 2
    h = np.exp(-(x * x + y * y) / 30.0)
    h = (h / h.sum()).astype(S.RDT[dt])
    got = host(pb.convolution.conv(dev(o), dev(h)))
    import scipy.fft as sfft
    ref = sfft.fftshift(S.conv_ref(sfft.ifftshift(S.ld(o)), sfft.ifftshift(S.ld(h))))
    check(f'{DN[dt]}/conv', S.rel_linf(got, ref))


@pytest.mark.parametrize('f', ((1, 7), (7, 1), (3, 5)))
@pytest.mark.parametrize('dt', DTS)
def test_bindown_and_tile(pb, dt, f):
    fy, fx = f
    a = rand((fy * 131, fx * 97), 47, dt)
    for mean in (False, True):
        got, n = launches(pb, lambda: pb._ops.bindown(dev(a), fy, fx, mean))
        assert n == 1
        check(f'{DN[dt]}/bindown', S.red_fig(host(got).ravel(), S.bindown_ref(a, fy, fx, mean).ravel(),
                                             S.bindown_ref(np.abs(a), fy, fx, mean).ravel()))
    small = rand((131, 97), 48, dt)
    got, n = launches(pb, lambda: pb._ops.tile(dev(small), fy, fx, 0.5))
    assert n == 1
    assert np.array_equal(host(got), np.asarray(S.tile_ref(small, fy, fx, 0.5, S.RDT[dt]), S.RDT[dt]))


@pytest.mark.parametrize('kind', (0, 1))
@pytest.mark.parametrize('dt', DTS)
def test_separable_tf(pb, dt, kind):
    fx = np.concatenate([np.arange(-8, 9) * 0.5, np.linspace(-37.3, 41.1, 300)]).astype(S.RDT[dt])
    fy = np.concatenate([np.arange(-4, 5) * 0.25, np.linspace(-13.0, 9.7, 200)]).astype(S.RDT[dt])
    for wx, wy in ((2.0, 4.0), (0.0, 0.0), (0.013, 0.0)):
        got, n = launches(pb, lambda: pb._ops.separable_tf(kind, dev(fx), dev(fy), wx, wy))
        assert n == 1
        ref = S.separable_tf_ref(kind, fx, fy, wx, wy)
        g = host(got)
        if wx == 0 and wy == 0:
            assert np.all(g == 1)
        # sinc zeros: absolute error against the largest value
        check(f'{DN[dt]}/separable_tf_{kind}', S.rel_linf(g, ref))


# ---- reverse pass through the public functions ----------------------------------------------------------------------
def psf_for(shape, seed):
    rng = np.random.default_rng(seed)
    y, x = np.indices(shape) - np.array(shape)[:, None, None] // 2
    return np.exp(-(x * x + y * y) / (0.02 * shape[0] * shape[1])) + 0.05 * rng.random(shape)


@pytest.mark.parametrize('which', (1, 2, 4))
@pytest.mark.parametrize('shape', ((256, 256), (255, 383)))
@pytest.mark.parametrize('dt', DTS)
def test_otf_from_psf_adjoint(pb, dt, shape, which):
    """mtf / ptf / otf _from_psf_adjoint (seed kernel and adjoint transform) on the device's own forward transform,
    against the long-double composite whose adjoint identity tests/test_host_streaming_reference.py checks.  The
    forward transform is held to its reference by the transform tests; feeding its output to both sides keeps the
    figure free of the 1/|D| amplification of its rounding."""
    psf = psf_for(shape, 49).astype(S.RDT[dt])
    bar = crand(shape, 50, dt) if which == 4 else rand(shape, 50, dt)
    data, _ = pb.otf.transform_psf(dev(psf), 1.0)
    fn = {1: pb.otf.mtf_from_psf_adjoint, 2: pb.otf.ptf_from_psf_adjoint, 4: pb.otf.otf_from_psf_adjoint}[which]
    got = host(fn(dev(bar), data=data))
    ref = S.transform_psf_adjoint_ld(S.otf_adjoint_seed_ref(which, bar, host(data))[0]).real
    check(f'{DN[dt]}/psf_adjoint_{which}', S.rel_linf(got, ref))


@pytest.mark.parametrize('shape', ((256, 256), (255, 383)))
@pytest.mark.parametrize('dt', DTS)
def test_encircled_energy_adjoint(pb, dt, shape):
    psf = psf_for(shape, 51).astype(S.RDT[dt])
    radii = np.array([2.0, 5.0, 11.0, 30.0])
    ee_bar = np.array([0.3, -1.2, 2.0, 0.7])
    dx = 0.5
    data, _ = pb.otf.transform_psf(dev(psf), dx)
    got = host(pb.otf.encircled_energy_adjoint(ee_bar, dx=dx, radius=radii, data=data))
    # the MTF-plane gradient is the device's own (test_encircled_energy_adjoint_seed holds it to its reference): the
    # seed and the adjoint transform of a smooth gradient cancel strongly, which would amplify its rounding here
    mtf_bar = host(pb._ops.encircled_energy_adjoint_seed(shape, 1000 / (shape[0] * dx), radii / 1e3, ee_bar, TR[dt],
                                                         'cuda'))
    ref = S.transform_psf_adjoint_ld(S.otf_adjoint_seed_ref(1, mtf_bar, host(data))[0]).real
    check(f'{DN[dt]}/ee_adjoint', S.rel_linf(got, ref))


# ---- beyond int32 ---------------------------------------------------------------------------------------------------
def test_moments_beyond_int32(pb):
    """46341^2 > 2^31 float32 ones (8.6 GB): the sums are integers below 2^53, so fp64 accumulation is exact"""
    ny = nx = 46341
    need = ny * nx * 4
    if torch.cuda.mem_get_info()[0] < 2 * need:
        pytest.skip('needs twice 8.6 GB free on the device')
    d = torch.ones((ny, nx), dtype=torch.float32, device='cuda')
    try:
        s0, sy, sx = pb._ops.moments(d)
    finally:
        del d
        torch.cuda.empty_cache()
    assert s0 == ny * nx
    assert sy == nx * (ny * (ny - 1) // 2)
    assert sx == ny * (nx * (nx - 1) // 2)


# ---- bookkeeping ----------------------------------------------------------------------------------------------------
def test_zz_every_figure_has_a_measurement():
    """a figure this session reached that has no MEASURED entry is held to the bare ceiling, a bound nobody measured"""
    if os.environ.get('PB_TEST_MEASUREMENTS'):
        pytest.skip('recording figures')
    assert not LEDGER.missing(), f'no MEASURED entry (record them with PB_TEST_MEASUREMENTS): {LEDGER.missing()}'
