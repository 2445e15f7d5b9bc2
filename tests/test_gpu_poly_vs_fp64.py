"""GPU: the polynomial kernels of csrc/orthopoly.cu, csrc/synthesis.cu (Zernike) and csrc/qpoly.cu held to the
long-double references of tests/poly_reference.py at every order, plan split and grid sweep, at both storage dtypes.

- pb_poly_seq: every family in all three kinds at every order 0-120, Jacobi at eight (alpha, beta) pairs, points
  outside the orthogonality interval; S - 1, S, S + 1, 2S + 1 and 2048^2 samples (S = one grid sweep); 520 float32
  planes at 2048^2, past 2^31 output elements.
- pb_jacobi_clenshaw: lengths 1, 2 and 121, j = 0-8, with and without the table; pb_jacobi_radial_sum with R != 1
  and points past R.
- Zernike: sequences, polar and Cartesian derivatives and sums over every mode with n <= 20 plus modes at the
  (n - |m|)/2 = 71 step limit, sums with x3 duplicates and with two plans' partial sums cancelling, the launch count
  of the plan rule.
- Forbes: Q-bfs and Q-con to n = 64, 2D-Q at |m| up to 64 in all three kinds and sums, 256-step plans.
- XY monomials to order 32767 near +-1, separable and elementwise; tensor sums at 1024 coefficients.
- Every limit plus one is refused before anything launches.

Every output is prefilled with NaN.  A figure is the smallest c with |got - ref| <= c (n + 1) 2^-53 M, plus 2^-24 |ref|
for float32 storage (the fp64 result rounded once), M the recurrence's majorant (poly_reference.c_figure).  Bounds are
1.5x the figures measured on an H100 (`MEASURED`, recorded with PB_TEST_MEASUREMENTS) and never above
poly_reference.CEIL, which tests/test_host_poly_reference.py shows every modelled defect exceeds by 10x or more.
"""
import contextlib
import os

import numpy as np
import pytest
import torch

import poly_reference as R
from accuracy import Ledger
from gpu_fixtures import pb, sm_count  # noqa: F401

pytestmark = pytest.mark.gpu

PRECS = (32, 64)
NPR = {32: np.float32, 64: np.float64}
KINDS = ('value', 'der', 'value_der')

# ---- measured fp64 figures (H100 80GB HBM3, 700 W power limit, 1980 MHz SM clock); bounds are 1.5x these, capped at
# R.CEIL, for both storage dtypes --------------------------------------------------------------------------------------
MEASURED = {
    'cheby1/der': 1.56,
    'cheby1/value': 1.64,
    'cheby1/value_der': 1.64,
    'cheby2/der': 1.72,
    'cheby2/value': 2.49,
    'cheby2/value_der': 2.49,
    'cheby3/der': 1.65,
    'cheby3/value': 4.17,
    'cheby3/value_der': 4.17,
    'cheby4/der': 1.65,
    'cheby4/value': 2.84,
    'cheby4/value_der': 2.84,
    'clenshaw_sum': 15,
    'clenshaw_table': 31.3,
    'dickson1/der': 0.411,
    'dickson1/value': 0.393,
    'dickson1/value_der': 0.411,
    'dickson2/der': 0.341,
    'dickson2/value': 0.385,
    'dickson2/value_der': 0.385,
    'hermite_h/der': 3.69,
    'hermite_h/value': 3.76,
    'hermite_h/value_der': 3.76,
    'hermite_he/der': 2.48,
    'hermite_he/value': 2.5,
    'hermite_he/value_der': 2.5,
    'jacobi/der': 20.5,
    'jacobi/value': 24.4,
    'jacobi/value_der': 24.4,
    'laguerre/der': 11.1,
    'laguerre/value': 13.6,
    'laguerre/value_der': 13.6,
    'legendre/der': 2.7,
    'legendre/value': 6.51,
    'legendre/value_der': 6.51,
    'q2d_der': 141,
    'q2d_der_xy': 209,
    'q2d_value': 9.42,
    'qbfs_der': 1.24,
    'qbfs_value': 2,
    'qcon_der': 2.5,
    'qcon_value': 5.41,
    'qsum_2d': 0.275,
    'qsum_2d_der': 0.151,
    'qsum_bfs': 0.163,
    'qsum_bfs_der': 0.215,
    'qsum_con': 0.672,
    'qsum_con_der': 0.562,
    'radial_sum': 3.02,
    'radial_sum_der': 1.46,
    'sweep': 23,
    'tsum_cheby1': 0.176,
    'tsum_monomial': 0.122,
    'xy': 0.131,
    'zernike_der': 3.41,
    'zernike_seq': 73.3,
    'zernike_sum/cancel': 0.0663,
    'zernike_sum/dup3': 0.234,
    'zernike_sum/high': 4.53,
    'zernike_sum/noll20': 0.321,
    'zernike_sum_der_xy/cancel': 0.0259,
    'zernike_sum_der_xy/dup3': 0.082,
    'zernike_sum_der_xy/high': 0.537,
    'zernike_sum_der_xy/noll20': 0.178,
}

# the worst figure of each name over the whole file.  A float32 figure is the error beyond the one rounding of the fp64
# result, so it is held to the fp64 figure of the same name: the kernels run the same fp64 arithmetic at both storage
# dtypes.
LEDGER = Ledger(MEASURED, R.CEIL, key=lambda name: name.split('/', 1)[1])
check = LEDGER.check


class _NanTorch:
    """torch with empty / empty_like returning NaN-filled tensors, so that an element a kernel leaves unwritten
    cannot pass for a result"""
    def __getattr__(self, k):
        return getattr(torch, k)

    @staticmethod
    def empty(*shape, **kw):
        shape = tuple(shape[0]) if len(shape) == 1 and isinstance(shape[0], (tuple, list, torch.Size)) else shape
        return torch.full(shape, float('nan'), **kw)

    @staticmethod
    def empty_like(t, **kw):
        return torch.full_like(t, float('nan'), **kw)


@contextlib.contextmanager
def nan_outputs(pb):
    saved = pb._ops.torch
    pb._ops.torch = _NanTorch()
    try:
        yield
    finally:
        pb._ops.torch = saved


def call(pb, fn):
    """fn()'s result with NaN-prefilled outputs, and the number of kernels it launched"""
    with nan_outputs(pb):
        torch.cuda.synchronize()
        c0 = pb._ops.launch_count()
        res = fn()
        torch.cuda.synchronize()
        return res, pb._ops.launch_count() - c0


def refused(pb, fn):
    """fn() raises and launches nothing"""
    torch.cuda.synchronize()
    c0 = pb._ops.launch_count()
    with pytest.raises(Exception):
        fn()
    torch.cuda.synchronize()
    assert pb._ops.launch_count() == c0


def dev(a, prec):
    return torch.from_numpy(np.ascontiguousarray(np.asarray(a, np.float64).astype(NPR[prec]))).cuda()


def host(t):
    return t.detach().cpu().numpy().astype(np.float64)


def family_params(fam):
    if fam == 'jacobi':
        return R.JACOBI_AB
    if fam == 'laguerre':
        return ((0.0, 0.0), (0.7, 0.0), (-0.5, 0.0), (12.0, 0.0))
    if fam.startswith('dickson'):
        return ((0.0, 0.0), (0.7, 0.0), (-1.0, 0.0))
    return ((0.0, 0.0),)


def family_refs(fam, x, ns, kind, a, b):
    """[(planes, majorants)] of the outputs of one pb_poly_seq call"""
    P, dP, M, dM = R.rec1d(fam, x, max(ns), a, b)
    val = (P[ns], M[ns])
    if kind == 'value':
        return [val]
    if fam in R.SHIFTED and kind == 'der':
        return [R.shifted_der(fam, x, ns, a, b)]
    der = (dP[ns], dM[ns])
    return [der] if kind == 'der' else [val, der]


# ---- 1-D families --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('fam', R.FAMILIES)
@pytest.mark.parametrize('prec', PRECS)
def test_family_every_order(pb, prec, fam, kind):
    x = R.family_points(fam)
    ns = list(range(R.JAC_MAX + 1))
    kc = KINDS.index(kind)
    steps = np.array(ns)[:, None]
    for a, b in family_params(fam):
        out, k = call(pb, lambda: pb._ops.poly_seq(R.FAMILIES.index(fam), kc, ns, dev(x, prec), a, b))
        assert k == 1
        outs = out if kind == 'value_der' else (out,)
        for got, (ref, maj) in zip(outs, family_refs(fam, x, ns, kind, a, b)):
            check(f'{prec}/{fam}/{kind}', R.c_figure(host(got), ref, maj, steps, prec == 32))


@pytest.mark.parametrize('prec', PRECS)
def test_family_limits_refused(pb, prec):
    x = dev(R.family_points('legendre'), prec)
    leg = R.FAMILIES.index('legendre')
    assert R.poly_refused([121], False) and R.poly_refused([0] * 513, True) and not R.poly_refused([120] * 512, True)
    refused(pb, lambda: pb._ops.poly_seq(leg, 0, [121], x))
    refused(pb, lambda: pb._ops.poly_seq(leg, 2, [q % 121 for q in range(513)], x))
    refused(pb, lambda: pb._ops.poly_seq(leg, 0, [0] * 1025, x))
    refused(pb, lambda: pb._ops.jacobi_seq([121], 0.0, 0.0, x))
    (out, k) = call(pb, lambda: pb._ops.poly_seq(leg, 2, [q % 121 for q in range(512)], x))
    assert k == 1 and not any(torch.isnan(o).any().item() for o in out)
    out, k = call(pb, lambda: pb._ops.poly_seq(leg, 0, [120] * 1024, x))
    assert k == 1 and not torch.isnan(out).any().item()


def tiled_figure(got, P, ref, maj, steps, f32):
    """got (k, count) of inputs tiled with period P: every copy must equal the first bit for bit (the kernel is a
    function of the sample), and the first copy is held to the reference"""
    k, count = got.shape
    full = count // P * P
    first = got[:, :P]
    if full:
        assert torch.equal(got[:, :full].reshape(k, -1, P), first[:, None, :].expand(k, full // P, P))
    if count > full:
        assert torch.equal(got[:, full:], first[:, :count - full])
    return R.c_figure(host(first), ref, maj, steps, f32)


@pytest.mark.parametrize('prec', PRECS)
def test_family_grid_sweeps(pb, prec):
    """Legendre and Jacobi value and derivative planes at S - 1, S, S + 1, 2S + 1 and 2048^2 samples"""
    x = R.family_points('jacobi')
    P = x.size
    ns = [0, 1, 2, 7, 64, 120]
    for count in R.sweep_counts(sm_count()) + (2048 ** 2,):
        xt = dev(np.resize(x, count), prec)
        for fam, (a, b) in (('legendre', (0.0, 0.0)), ('jacobi', (0.7, 2.0))):
            (v, d), k = call(pb, lambda: pb._ops.poly_seq(R.FAMILIES.index(fam), 2, ns, xt, a, b))
            assert k == 1
            (rv, mv), (rd, md) = family_refs(fam, x, ns, 'value_der', a, b)
            steps = np.array(ns)[:, None]
            check(f'{prec}/sweep', tiled_figure(v, P, rv, mv, steps, prec == 32))
            check(f'{prec}/sweep', tiled_figure(d, P, rd, md, steps, prec == 32))


def test_float32_past_2_31(pb):
    """520 float32 Legendre planes at 2048^2: 2.18e9 output elements, so the plane offsets need 64 bits"""
    x = R.family_points('legendre')
    P = x.size
    ns = [q % 121 for q in range(520)]
    xt = dev(np.resize(x, 2048 ** 2), 32)
    out, k = call(pb, lambda: pb._ops.poly_seq(R.FAMILIES.index('legendre'), 0, ns, xt))
    assert k == 1 and out.numel() > 2 ** 31
    Pr, _, M, _ = R.rec1d('legendre', x, 120)
    for p0 in range(0, 520, 40):
        sl = slice(p0, min(p0 + 40, 520))
        idx = ns[sl]
        check('32/legendre/value', tiled_figure(out[sl], P, Pr[idx], M[idx], np.array(idx)[:, None], True))
    del out
    torch.cuda.empty_cache()


# ---- Clenshaw and radial sums --------------------------------------------------------------------------------------
@pytest.mark.parametrize('L', (1, 2, 121))
@pytest.mark.parametrize('prec', PRECS)
def test_clenshaw(pb, prec, L):
    rng = np.random.default_rng(L)
    x = R.interval_points(-1.0, 1.0, (-1.5, 1.5), n=24)
    for a, b in R.JACOBI_AB[::2] + ((0.0, -1.0 + 2.0 ** -10),):
        s = rng.standard_normal(L)
        T, TM = R.clenshaw_ref(s, x, R.CLEN_J, a, b)
        for j in range(R.CLEN_J + 1):
            tab, k = call(pb, lambda: pb._ops.jacobi_clenshaw(s, a, b, dev(x, prec), j, True))
            assert k == 1
            check(f'{prec}/clenshaw_table', R.c_figure(host(tab), T[:j + 1], TM[:j + 1], max(L, 2), prec == 32))
            z, k = call(pb, lambda: pb._ops.jacobi_clenshaw(s, a, b, dev(x, prec), j, False))
            assert k == 1
            check(f'{prec}/clenshaw_sum', R.c_figure(host(z), T[0, 0], TM[0, 0], max(L, 2), prec == 32))
    xd = dev(x, prec)
    refused(pb, lambda: pb._ops.jacobi_clenshaw(np.ones(122), 0.0, 0.0, xd, 0, False))
    refused(pb, lambda: pb._ops.jacobi_clenshaw(np.ones(4), 0.0, 0.0, xd, 9, True))


@pytest.mark.parametrize('prec', PRECS)
def test_radial_sum(pb, prec):
    rng = np.random.default_rng(7)
    x, y = R.zernike_xy_points(60)
    x, y = R.f32(x * 1.5), R.f32(y * 1.5)
    ns = list(range(121))
    coefs = rng.standard_normal(121)
    coefs[::5] = 0.0
    for (a, b), radius in (((0.0, 0.0), 1.3), ((0.7, 2.0), 0.9), ((-0.5, -0.5), 1.0)):
        (z, dx, dy), (mz, mx, my) = R.radial_sum_ref(coefs, ns, x, y, radius, a, b)
        for der in (False, True):
            (gz, gx, gy), k = call(pb, lambda: pb._ops.jacobi_radial_sum(coefs, ns, a, b, dev(x, prec), dev(y, prec),
                                                                         radius, der))
            assert k == 1
            check(f'{prec}/radial_sum', R.c_figure(host(gz), z, mz, 120, prec == 32))
            if der:
                check(f'{prec}/radial_sum_der', R.c_figure(host(gx), dx, mx, 120, prec == 32))
                check(f'{prec}/radial_sum_der', R.c_figure(host(gy), dy, my, 120, prec == 32))
    refused(pb, lambda: pb._ops.jacobi_radial_sum([1.0], [121], 0.0, 0.0, dev(x, prec), dev(y, prec), 1.0, False))


# ---- Zernike -------------------------------------------------------------------------------------------------------
ZERN_HIGH = [(142, 0), (143, -1), (146, 4), (160, -18), (200, 60), (201, -61)]
ZERN_MODES = [(n, m) for n in range(21) for m in range(-n, n + 1, 2)] + ZERN_HIGH


def zpoints(cartesian):
    return R.zernike_xy_points() if cartesian else R.zernike_points()


@pytest.mark.parametrize('cartesian', (False, True))
@pytest.mark.parametrize('prec', PRECS)
def test_zernike_seq(pb, prec, cartesian):
    a, b = zpoints(cartesian)
    out, k = call(pb, lambda: pb._ops.zernike_seq(ZERN_MODES, dev(a, prec), dev(b, prec), True, not cartesian))
    assert k == R.zernike_plans(R.zernike_terms(ZERN_MODES))
    got = host(out)
    for q, (n, m) in enumerate(ZERN_MODES):
        ref, maj = R.zernike_ref(n, m, a, b, not cartesian)
        check(f'{prec}/zernike_seq', R.c_figure(got[q], ref, maj, n, prec == 32))


@pytest.mark.parametrize('cartesian', (False, True))
@pytest.mark.parametrize('prec', PRECS)
def test_zernike_der(pb, prec, cartesian):
    a, b = zpoints(cartesian)
    out, k = call(pb, lambda: pb._ops.zernike_der(ZERN_MODES, dev(a, prec), dev(b, prec), True, cartesian))
    assert k == R.zernike_plans(R.zernike_terms(ZERN_MODES))
    got = host(out)
    for q, (n, m) in enumerate(ZERN_MODES):
        (d0, d1), (m0, m1) = R.zernike_der_ref(n, m, a, b, cartesian)
        check(f'{prec}/zernike_der', R.c_figure(got[q, 0], d0, m0, n, prec == 32))
        check(f'{prec}/zernike_der', R.c_figure(got[q, 1], d1, m1, n, prec == 32))


def zernike_sum_cases():
    rng = np.random.default_rng(11)
    noll = [(n, m) for n in range(21) for m in range(-n, n + 1, 2)]
    dup = noll[:40] * 3
    return {'noll20': (noll, rng.standard_normal(len(noll))),
            'high': (ZERN_MODES, rng.standard_normal(len(ZERN_MODES)) * (rng.uniform(size=len(ZERN_MODES)) > 0.2)),
            'dup3': (dup, rng.standard_normal(len(dup))),
            'cancel': ([(8, 2), (8, 2), (3, -1), (3, -1)], np.array([1.0, -1.0 + 1e-3, -2.0, 2.0 - 1e-4]))}


@pytest.mark.parametrize('case', ('noll20', 'high', 'dup3', 'cancel'))
@pytest.mark.parametrize('cartesian', (False, True))
@pytest.mark.parametrize('prec', PRECS)
def test_zernike_sum(pb, prec, cartesian, case):
    nms, coefs = zernike_sum_cases()[case]
    a, b = zpoints(cartesian)
    nmax = max(n for n, _ in nms)
    out, k = call(pb, lambda: pb._ops.zernike_sum(coefs, nms, dev(a, prec), dev(b, prec), True, not cartesian))
    assert k == R.zernike_plans(R.zernike_terms(nms, coefs))
    (ref,), (maj,) = R.zernike_sum_ref(coefs, nms, a, b, not cartesian)
    check(f'{prec}/zernike_sum/{case}', R.c_figure(host(out), ref, maj, nmax, prec == 32))


@pytest.mark.parametrize('case', ('noll20', 'high', 'dup3', 'cancel'))
@pytest.mark.parametrize('prec', PRECS)
def test_zernike_sum_der_xy(pb, prec, case):
    nms, coefs = zernike_sum_cases()[case]
    x, y = R.zernike_xy_points()
    nmax = max(n for n, _ in nms)
    out, k = call(pb, lambda: pb._ops.zernike_sum_der_xy(coefs, nms, dev(x, prec), dev(y, prec), True))
    assert k == R.zernike_plans(R.zernike_terms(nms, coefs, merge=True))
    refs, majs = R.zernike_sum_ref(coefs, nms, x, y, False, der=True)
    got = host(out)
    for p in range(3):
        check(f'{prec}/zernike_sum_der_xy/{case}', R.c_figure(got[p], refs[p], majs[p], nmax, prec == 32))


@pytest.mark.parametrize('prec', PRECS)
def test_zernike_limits_refused(pb, prec):
    a, b = (dev(v, prec) for v in R.zernike_points(8))
    out, k = call(pb, lambda: pb._ops.zernike_seq([(143, 1), (0, 0)], a, b, True, True))
    assert k == R.zernike_plans(R.zernike_terms([(143, 1), (0, 0)])) == 2 and not torch.isnan(out).any().item()
    for fn in (lambda: pb._ops.zernike_seq([(0, 0), (145, 1)], a, b, True, True),
               lambda: pb._ops.zernike_sum([1.0, 1.0], [(0, 0), (144, 0)], a, b, True, True),
               lambda: pb._ops.zernike_der([(0, 0), (144, 0)], a, b, True, True),
               lambda: pb._ops.zernike_sum_der_xy([1.0, 1.0], [(0, 0), (144, 0)], a, b, True),
               lambda: pb._ops.zernike_seq([(0, 0)] * (R.ZERN_SEQ_K + 1), a, b, True, True),
               lambda: pb._ops.zernike_der([(0, 0)] * (R.ZERN_DER_K + 1), a, b, True, True)):
        refused(pb, fn)


# ---- Forbes polynomials --------------------------------------------------------------------------------------------
QKIND = {'value': 0, 'der': 1, 'der_xy': 2}


@pytest.mark.parametrize('kind', ('value', 'der'))
@pytest.mark.parametrize('family', ('bfs', 'con'))
@pytest.mark.parametrize('prec', PRECS)
def test_qbfs_qcon_seq(pb, prec, family, kind):
    r, _ = R.q_points()
    ns = list(range(R.Q_NMAX + 1))
    fc = {'bfs': 0, 'con': 1}[family]
    out, k = call(pb, lambda: pb._ops.qpoly_seq(fc, QKIND[kind], ns, None, dev(r, prec)))
    assert k == 1
    got = host(out)
    for n in ns:
        (ref,), (maj,) = R.qpoly_ref(family, n, 0, r, None, kind)
        check(f'{prec}/q{family}_{kind}', R.c_figure(got[n], ref, maj, n, prec == 32))


Q2D_GROUPS = ((0, 1, 2), (3, 20, 63), (64,))


@pytest.mark.parametrize('kind', ('value', 'der', 'der_xy'))
@pytest.mark.parametrize('prec', PRECS)
def test_q2d_seq(pb, prec, kind):
    """every n <= 64 at |m| = 0-3, 20, 63 and 64, both signs: three calls of 195 and 65 steps"""
    r, t = R.q_points()
    a, b = (R.zernike_xy_points(20) if kind == 'der_xy' else (r, t))
    for ams in Q2D_GROUPS:
        nms = [(n, s * am) for am in ams for s in ((1, -1) if am else (1,)) for n in range(R.Q_NMAX + 1)]
        ns, ms = [n for n, _ in nms], [m for _, m in nms]
        out, k = call(pb, lambda: pb._ops.qpoly_seq(2, QKIND[kind], ns, ms, dev(a, prec), dev(b, prec)))
        assert k == 1
        outs = [host(o) for o in (out if isinstance(out, tuple) else (out,))]
        for q, (n, m) in enumerate(nms):
            refs, majs = R.qpoly_ref('2d', n, m, a, b, kind)
            for o, ref, maj in zip(outs, refs, majs):
                check(f'{prec}/q2d_{kind}', R.c_figure(o[q], ref, maj, n, prec == 32))


@pytest.mark.parametrize('family', ('bfs', 'con', '2d'))
@pytest.mark.parametrize('prec', PRECS)
def test_qpoly_sum(pb, prec, family):
    rng = np.random.default_rng(3)
    r, t = R.q_points()
    if family == '2d':
        nms = [(n, s * am) for am in (0, 1, 5, 64) for s in ((1, -1) if am else (1,)) for n in range(0, 64, 3)]
    else:
        nms = [(n, 0) for n in range(R.Q_NMAX + 1)]
    ns, ms = [n for n, _ in nms], [m for _, m in nms]
    coefs = rng.standard_normal(len(nms))
    coefs[::7] = 0.0
    fc = {'bfs': 0, 'con': 1, '2d': 2}[family]
    tt = dev(t, prec) if family == '2d' else None
    (z, dr, dt), k = call(pb, lambda: pb._ops.qpoly_sum(fc, ns, ms if family == '2d' else None, coefs, dev(r, prec),
                                                        tt, True))
    assert k == 1
    refs, majs = R.qpoly_sum_ref(family, ns, ms, coefs, r, t, der=True)
    check(f'{prec}/qsum_{family}', R.c_figure(host(z), refs[0], majs[0], 64, prec == 32))
    check(f'{prec}/qsum_{family}_der', R.c_figure(host(dr), refs[1], majs[1], 64, prec == 32))
    if family == '2d':
        check(f'{prec}/qsum_{family}_der', R.c_figure(host(dt), refs[2], majs[2], 64, prec == 32))


@pytest.mark.parametrize('prec', PRECS)
def test_qpoly_limits(pb, prec):
    """256 steps launch once, 257 are refused; n or |m| of 65 and 1025 modes are refused"""
    r, t = (dev(v, prec) for v in R.q_points(4))
    nms = [(63, am) for am in (1, 2, 3, 4)]                         # 4 x 64 = 256 steps
    assert R.q_steps(R.q_groups('2d', [n for n, _ in nms], [m for _, m in nms])) == R.Q_STEPS
    out, k = call(pb, lambda: pb._ops.qpoly_seq(2, 0, [n for n, _ in nms], [m for _, m in nms], r, t))
    assert k == 1 and not torch.isnan(out).any().item()
    over = nms + [(0, 5)]
    assert R.q_steps(R.q_groups('2d', [n for n, _ in over], [m for _, m in over])) == R.Q_STEPS + 1
    refused(pb, lambda: pb._ops.qpoly_seq(2, 0, [n for n, _ in over], [m for _, m in over], r, t))
    refused(pb, lambda: pb._ops.qpoly_sum(2, [n for n, _ in over], [m for _, m in over], [1.0] * 5, r, t))
    refused(pb, lambda: pb._ops.qpoly_seq(0, 0, [65], None, r))
    refused(pb, lambda: pb._ops.qpoly_seq(2, 0, [0], [65], r, t))
    refused(pb, lambda: pb._ops.qpoly_seq(0, 0, [0] * 1025, None, r))


# ---- XY monomials and tensor sums ----------------------------------------------------------------------------------
XY_ORDERS = (0, 1, 2, 3, 100, 4097, R.XY_ORDER)


@pytest.mark.parametrize('separable', (False, True))
@pytest.mark.parametrize('prec', PRECS)
def test_xy_high_orders(pb, prec, separable):
    k = np.arange(1, 6)
    xs = R.f32(np.concatenate([1 - k * 2.0 ** -24, -(1 - k * 2.0 ** -24), [1.0, -1.0, 0.5, 0.0, 1 + 2.0 ** -23]]))
    ys = R.f32(np.concatenate([-(1 - k * 2.0 ** -24), [0.999, 1.0, -1.0]]))
    planes = [(m, n, kd) for m in XY_ORDERS for n in (0, 1, R.XY_ORDER) for kd in range(4)]
    ms, ns, kinds = ([p[i] for p in planes] for i in range(3))
    if separable:
        shape = (ys.size, xs.size)
        xe, ye = np.meshgrid(xs, ys)
        xd, yd = dev(xs, prec), dev(ys, prec)
    else:
        xe, ye = np.meshgrid(xs, ys)
        shape = (xe.size,)
        xd, yd = dev(xe.ravel(), prec), dev(ye.ravel(), prec)
    out, kk = call(pb, lambda: pb._ops.xy_seq(ms, ns, kinds, xd, yd, shape, separable))
    assert kk == 1
    got = host(out).reshape(len(planes), -1)
    for q, (m, n, kd) in enumerate(planes):
        ref, maj = R.xy_ref(m, n, kd, xe.ravel(), ye.ravel())
        check(f'{prec}/xy', R.c_figure(got[q], ref, maj, m + n, prec == 32))
    refused(pb, lambda: pb._ops.xy_seq([R.XY_ORDER + 1], [0], [0], xd, yd, shape, separable))
    refused(pb, lambda: pb._ops.xy_seq([0] * 1025, [0] * 1025, [0] * 1025, xd, yd, shape, separable))


@pytest.mark.parametrize('basis', ('monomial', 'cheby1'))
@pytest.mark.parametrize('separable', (False, True))
@pytest.mark.parametrize('prec', PRECS)
def test_tensor_sum(pb, prec, separable, basis):
    rng = np.random.default_rng(5)
    xs = R.interval_points(-1.0, 1.0, (1.0625,), n=20)
    ys = R.interval_points(-1.0, 1.0, (-1.0625,), n=12, seed=1)
    bc = {'monomial': 0, 'cheby1': 1}[basis]
    for mx, nx in ((31, 31), (1023, 0), (0, 1023), (15, 63)):
        mn = [(m, n) for m in range(mx + 1) for n in range(nx + 1)]
        assert not R.tsum_refused([m for m, _ in mn], [n for _, n in mn])
        ms, ns = [m for m, _ in mn], [n for _, n in mn]
        coefs = rng.standard_normal(len(mn)) / (1 + np.array(ms) + np.array(ns)) ** 2
        xe, ye = np.meshgrid(xs, ys)
        if separable:
            shape, xd, yd = (ys.size, xs.size), dev(xs, prec), dev(ys, prec)
        else:
            shape, xd, yd = (xe.size,), dev(xe.ravel(), prec), dev(ye.ravel(), prec)
        (z, dx, dy), k = call(pb, lambda: pb._ops.tensor_sum(bc, coefs, ms, ns, xd, yd, shape, separable, True,
                                                             0.7, 1.3))
        assert k == 1
        refs, majs = R.tensor_ref(basis, coefs, ms, ns, xe.ravel(), ye.ravel(), 0.7, 1.3)
        for got, ref, maj in zip((z, dx, dy), refs, majs):
            check(f'{prec}/tsum_{basis}', R.c_figure(host(got).ravel(), ref, maj, mx + nx, prec == 32))
    over = [(40, 0), (0, 24)]                              # 41 x 25 = 1025
    assert R.tsum_refused([m for m, _ in over], [n for _, n in over])
    xd, yd = dev(xs, prec), dev(xs, prec)
    refused(pb, lambda: pb._ops.tensor_sum(bc, [1.0, 1.0], [40, 0], [0, 24], xd, yd, (xs.size,), False, False))


def test_zz_every_figure_has_a_measurement():
    """a figure this session reached that has no MEASURED entry is held to the bare ceiling, a bound nobody measured"""
    if os.environ.get('PB_TEST_MEASUREMENTS'):
        pytest.skip('recording figures')
    assert not LEDGER.missing(), f'no MEASURED entry (record them with PB_TEST_MEASUREMENTS): {LEDGER.missing()}'
