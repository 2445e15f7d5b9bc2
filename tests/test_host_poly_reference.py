"""CPU: the long-double polynomial references of tests/poly_reference.py against mpmath, the host Forbes tables against
mp tables, and the defect models against the GPU test's ceiling."""
import mpmath as mp
import numpy as np
import pytest

import poly_reference as R

LD = R.LDBL
ORDERS = (0, 1, 2, 3, 7, 17, 60, 119, 120)


def mpld(v):
    """a long double as an mp number (its shortest round-trip decimal, so also outside the double range)"""
    return mp.mpf(np.format_float_scientific(LD(v), unique=True))


def mp_jacobi(n, a, b, x):
    """P_n^(a, b)(x) by the explicit sum DLMF 18.5.8"""
    a, b = mp.mpf(a), mp.mpf(b)
    return mp.fsum(mp.binomial(n + a, n - s) * mp.binomial(n + b, s) * ((x - 1) / 2) ** s * ((x + 1) / 2) ** (n - s)
                   for s in range(n + 1))


def mp_family(fam, n, x, a, b):
    x, a, b = mp.mpf(x), mp.mpf(a), mp.mpf(b)
    if fam == 'jacobi':
        return mp_jacobi(n, a, b, x)
    if fam == 'cheby1':
        return mp.chebyt(n, x)
    if fam == 'cheby2':
        return mp.chebyu(n, x)
    if fam == 'cheby3':      # V_n = (U_n - U_{n-1}), W_n = (U_n + U_{n-1})
        return mp.chebyu(n, x) - (mp.chebyu(n - 1, x) if n else 0)
    if fam == 'cheby4':
        return mp.chebyu(n, x) + (mp.chebyu(n - 1, x) if n else 0)
    if fam == 'legendre':
        return mp.legendre(n, x)
    if fam == 'hermite_h':
        return mp.hermite(n, x)
    if fam == 'hermite_he':
        return mp.hermite(n, x / mp.sqrt(2)) / mp.mpf(2) ** (mp.mpf(n) / 2)
    if fam == 'laguerre':
        return mp.laguerre(n, a, x)
    # Dickson with parameter a: D_n = sum n/(n-k) C(n-k, k) (-a)^k x^(n-2k), E_n = sum C(n-k, k) (-a)^k x^(n-2k)
    if n == 0:
        return mp.mpf(2 if fam == 'dickson1' else 1)
    if fam == 'dickson1':
        return mp.fsum(mp.mpf(n) / (n - k) * mp.binomial(n - k, k) * (-a) ** k * x ** (n - 2 * k)
                       for k in range(n // 2 + 1))
    return mp.fsum(mp.binomial(n - k, k) * (-a) ** k * x ** (n - 2 * k) for k in range(n // 2 + 1))


def params(fam):
    if fam == 'jacobi':
        return R.JACOBI_AB
    if fam == 'laguerre':
        return ((0.0, 0.0), (0.7, 0.0), (-0.5, 0.0), (12.0, 0.0))
    if fam.startswith('dickson'):
        return ((0.0, 0.0), (0.7, 0.0), (-1.0, 0.0))
    return ((0.0, 0.0),)


@pytest.mark.parametrize('fam', R.FAMILIES)
def test_families_vs_mpmath(fam):
    """every family, every parameter set, orders to 120, on a subset of the sample points: within 2^-60 (n + 1) M"""
    mp.mp.dps = 120          # the explicit Jacobi sum cancels to 1e-71 at n = 120
    worst = 0.0
    for a, b in params(fam):
        x = R.family_points(fam)[::7]
        P, dP, M, dM = R.rec1d(fam, x, 120, a, b)
        for n in ORDERS:
            for i, xv in enumerate(x):
                ref = mp_family(fam, n, float(xv), a, b)
                err = abs(mpld(P[n, i]) - ref)
                worst = max(worst, float(err / ((n + 1) * M[n, i])) if err else 0.0)
    assert worst < 2.0 ** -60, worst


@pytest.mark.parametrize('fam', R.FAMILIES)
def test_derivative_tracks(fam):
    """the differentiated recurrence against a central difference in mp, and the shifted-order derivative of
    Jacobi / Hermite / Laguerre against the differentiated recurrence"""
    mp.mp.dps = 50
    a, b = params(fam)[-1]
    x = R.family_points(fam)[::11]
    P, dP, M, dM = R.rec1d(fam, x, 40, a, b)
    for n in (1, 2, 9, 40):
        for i in range(0, len(x), 3):
            d = mp.diff(lambda t: mp_family(fam, n, t, a, b), mp.mpf(float(x[i])))
            assert abs(mpld(dP[n, i]) - d) <= 2.0 ** -50 * (n + 1) * float(dM[n, i]) + 1e-300
    if fam in R.SHIFTED:
        ns = list(range(0, 121, 7)) + [120]
        P, dP, M, dM = R.rec1d(fam, x, 120, a, b)
        sh, msh = R.shifted_der(fam, x, ns, a, b)
        for q, n in enumerate(ns):
            assert np.all(abs(sh[q] - dP[n]) <= LD(2.0 ** -56) * (n + 1) * (dM[n] + msh[q]))


def mp_zernike_radial(n, m, r):
    m = abs(m)
    return mp.fsum((-1) ** k * mp.factorial(n - k) / (mp.factorial(k) * mp.factorial((n + m) // 2 - k)
                   * mp.factorial((n - m) // 2 - k)) * mp.mpf(r) ** (n - 2 * k) for k in range((n - m) // 2 + 1))


def test_zernike_vs_factorial_sum():
    mp.mp.dps = 80
    r, t = R.zernike_points(12)
    for n, m in ((0, 0), (1, 1), (4, -2), (11, 5), (20, 0), (40, 8), (61, -3), (143, 1), (150, 8)):
        if (n - abs(m)) // 2 > 71:
            continue
        z, mz = R.zernike_ref(n, abs(m), r, np.zeros_like(r), True, norm=False)
        for i in range(len(r)):
            ref = mp_zernike_radial(n, m, float(r[i]))
            assert abs(mpld(z[i]) - ref) <= 2.0 ** -60 * (n + 1) * float(mz[i])


def test_zernike_cartesian_matches_polar():
    x, y = R.zernike_xy_points(20)
    r, t = np.hypot(x.astype(LD), y.astype(LD)), np.arctan2(y.astype(LD), x.astype(LD))
    for n, m in ((3, 1), (6, -4), (9, 3), (30, -10)):
        zc, mc = R.zernike_ref(n, m, x, y, False)
        zp, _ = R.zernike_ref(n, m, r, t, True)
        assert np.all(abs(zc - zp) <= LD(2.0 ** -58) * (n + 1) * mc)
        (dx, dy), (mx, my) = R.zernike_der_ref(n, m, x, y, True)
        (dr, dt), _ = R.zernike_der_ref(n, m, r, t, False)
        ok = r > 0
        c, s = np.cos(t), np.sin(t)
        assert np.all(abs(dx - (c * dr - s * dt / np.where(ok, r, 1)))[ok] <= LD(2.0 ** -50) * (n + 1) * (mx + my)[ok])


def test_clenshaw_planes_are_derivatives():
    """alpha_jj[0] is the jj-th x derivative of sum s_n P_n^(a, b) (mp differentiation at 50 digits)"""
    mp.mp.dps = 50
    rng = np.random.default_rng(1)
    for a, b in ((0.0, 0.0), (0.5, -0.5), (0.0, -1.0 + 2.0 ** -10), (0.7, 2.0)):
        s = rng.standard_normal(9)
        x = np.array([-0.75, 0.0, 0.3, 1.0])
        T, TM = R.clenshaw_ref(s, x, 3, a, b)
        for i, xv in enumerate(x):
            f = lambda t: mp.fsum(mp.mpf(float(sn)) * mp_jacobi(n, a, b, t) for n, sn in enumerate(s))  # noqa: E731
            for jj in range(4):
                d = mp.diff(f, mp.mpf(xv), jj)
                assert abs(mpld(T[jj, 0, i]) - d) <= 2.0 ** -60 * 10 * float(TM[jj, 0, i]) + 1e-40


def test_qcon_is_jacobi_04():
    mp.mp.dps = 50
    r, _ = R.q_points(8)
    for n in (0, 1, 5, 30, 64):
        (v,), (mv,) = R.qpoly_ref('con', n, 0, r)
        for i in range(len(r)):
            u = mp.mpf(float(r[i])) ** 2
            ref = u * u * mp_jacobi(n, 0, 4, 2 * u - 1)
            assert abs(mpld(v[i]) - ref) <= 2.0 ** -60 * (n + 1) * float(mv[i]) + 1e-300


def test_forbes_tables_vs_mp():
    """the long-double tables, and pb_qpoly_tables (fp64, host C++) at every m <= 64 and n <= 64, against the same
    definitions evaluated at 60 digits"""
    from prysm_b200 import _capi
    from prysm_b200 import _ops
    mp.mp.dps = 60
    f, g, h = R.qbfs_tables(64, mp.mpf, mp.sqrt)
    fl, gl, hl = R.qbfs_tables(64)
    tab = _ops.qpoly_tables(_capi.QPOLY_BFS, 0, 64)
    worst_ld, worst_64 = 0.0, 0.0
    for n in range(65):
        for ref, ld, col in ((f[n], fl[n], 0), (g[n], gl[n], 1), (h[n], hl[n], 2)):
            if ref == 0:
                assert ld == 0 and tab[n, col] == 0
                continue
            worst_ld = max(worst_ld, float(abs((mpld(ld) - ref) / ref)))
            worst_64 = max(worst_64, float(abs((tab[n, col] - ref) / ref)))
    for m in range(1, 65):
        f, g = R.q2d_fg(64, m, mp.mpf, mp.sqrt)
        tab = _ops.qpoly_tables(_capi.QPOLY_2D, m, 64)
        for n in range(65):
            for ref, col in ((f[n], 6), (g[n], 5)):
                if ref != 0:
                    worst_64 = max(worst_64, float(abs((tab[n, col] - ref) / ref)))
            if n == 0 or (m == 1 and n == 1):      # A.3 is used from n = 1 (m = 1: n = 3); D = 0 at these
                continue
            for k, ref in enumerate(R.q2d_abc(n, m, mp.mpf)):
                if ref != 0:
                    worst_64 = max(worst_64, float(abs((tab[n, k] - ref) / ref)))
    assert worst_ld < 2.0 ** -58, worst_ld
    assert worst_64 < 4e-15, worst_64


def test_qbfs_recurrence_vs_mp():
    """the fp64-table Q-bfs forward recurrence to n = 64 stays within 2e-15 of the largest |Q_n| on [0, 1]"""
    mp.mp.dps = 60
    u = np.linspace(0, 1, 33)
    Q, _, MQ, _ = R._qseries('bfs', 0, u, 64)
    f, g, h = R.qbfs_tables(64, mp.mpf, mp.sqrt)
    for i in range(0, 33, 4):
        uu = mp.mpf(float(u[i]))
        P = [mp.mpf(2), 6 - 8 * uu]
        Qm = [mp.mpf(1), (P[1] - g[0]) / f[1]]
        for n in range(2, 65):
            P.append((2 - 4 * uu) * P[-1] - P[-2])
            Qm.append((P[n] - g[n - 1] * Qm[n - 1] - h[n - 2] * Qm[n - 2]) / f[n])
        for n in range(65):
            assert abs(mpld(Q[n, i]) - Qm[n]) <= 2.0 ** -60 * (n + 1) * float(MQ[n, i])


# ---- defect models against the ceiling ---------------------------------------------------------------------------
def test_defects_land_above_ceiling():
    figs = {}
    for fam in ('legendre', 'jacobi', 'cheby1', 'laguerre', 'hermite_h'):
        a, b = params(fam)[-1]
        x = R.family_points(fam)
        P, _, M, _ = R.rec1d(fam, x, 120, a, b)
        steps = np.arange(121)[:, None]
        for dt, f32 in ((np.float64, False), (np.float32, True)):
            figs[f'faithful/{fam}/{f32}'] = R.c_figure(R.model_1d(fam, x, 120, a, b, None, dt), P, M, steps, f32)
            for d in ('f32_step',) + (() if fam == 'cheby1' else ('order_off',)):   # Chebyshev steps do not vary
                figs[f'{d}/{fam}/{f32}'] = R.c_figure(R.model_1d(fam, x, 120, a, b, d, dt), P, M, steps, f32)
        if fam == 'cheby1':
            figs['jacobi_seed/cheby1'] = R.c_figure(R.model_1d(fam, x, 120, a, b, 'jacobi_seed'), P, M, steps, False)
    nms = [(n, m) for n in range(21) for m in range(-n, n + 1, 2)]
    coefs = np.random.default_rng(2).standard_normal(len(nms))
    r, t = R.zernike_points()
    terms = R.zernike_terms(nms)
    split = sum(1 for q, (n, m) in enumerate(nms) if abs(m) <= 7)
    order = sorted(range(len(nms)), key=lambda q: abs(nms[q][1]))
    nms_o, c_o = [nms[q] for q in order], coefs[order]
    assert R.zernike_plans(terms) == 2
    (ref,), (maj,) = R.zernike_sum_ref(c_o, nms_o, r, t, True)
    for d in (None, 'partial_f32', 'r_f32'):
        figs[f'zsum/{d}'] = R.c_figure(R.model_zernike_sum(c_o, nms_o, r, t, d, split), ref, maj, 20, True)
    # a duplicated mode: the two plans' partial sums cancel to 1e-3 of either
    dup = [(8, 2), (8, 2)]
    cd = [1.0, -1.0 + 1e-3]
    (ref,), (maj,) = R.zernike_sum_ref(cd, dup, r, t, True)
    assert R.zernike_plans(R.zernike_terms(dup)) == 2
    for d in (None, 'partial_f32'):
        figs[f'zdup/{d}'] = R.c_figure(R.model_zernike_sum(cd, dup, r, t, d, 1), ref, maj, 8, True)
    # faults that start at order 40, judged on the planes n >= 40 alone: the bounds must hold high orders as well
    hi = slice(40, None)
    for fam in ('legendre', 'jacobi', 'hermite_h'):
        a, b = params(fam)[-1]
        x = R.family_points(fam)
        P, _, M, _ = R.rec1d(fam, x, 121, a, b)
        steps = np.arange(121)[:, None]
        figs[f'f32_step40/{fam}'] = R.c_figure(R.model_1d(fam, x, 120, a, b, 'f32_step', start=40)[hi], P[:121][hi],
                                               M[:121][hi], steps[hi], False)
        figs[f'plane_off40/{fam}'] = R.c_figure(P[41:122].astype(np.float64), P[40:121], M[40:121], steps[hi], False)
    r, _ = R.q_points()
    u = r * r
    Q, _, MQ, _ = R._qseries('bfs', 0, u, 65)
    steps = np.arange(65)[:, None]
    figs['faithful/qbfs'] = R.c_figure(R.model_qbfs(u, 64), Q[:65], MQ[:65], steps, False)
    for d in ('plane_off', 'h_index', 'f32_step'):
        figs[f'{d}40/qbfs'] = R.c_figure(R.model_qbfs(u, 64, d)[hi], Q[40:65], MQ[40:65], steps[hi], False)
    for am in (1, 2, 20):
        Q2, _, M2, _ = R._qseries('2d', am, u, 65)
        figs[f'plane_off40/q2d_m{am}'] = R.c_figure(Q2[41:66].astype(np.float64), Q2[40:65], M2[40:65], steps[hi],
                                                    False)
    sm = 132
    vals = np.arange(2 * R.sweep(sm) + 1, dtype=np.float64)
    for d in (None, 'drop_sweep'):
        figs[f'sweep/{d}'] = R.c_figure(R.model_sweep(vals, vals.size, sm, d), vals, vals, 0, False)
    for k, v in figs.items():
        if k.startswith(('faithful', 'zsum/None', 'zdup/None', 'sweep/None')):
            assert v < R.CEIL, (k, v)
        else:
            assert v >= 10 * R.CEIL, (k, v)


def test_plan_rules():
    """the mirrored limits: Noll up to n = 20 takes two Zernike plans, |m| = 0-7 in the first; 25 groups or a 73-step
    group do not fit one plan"""
    nms = [R.noll_to_nm(j) for j in range(1, 232)]
    assert R.zernike_plans(R.zernike_terms(nms)) == 2
    assert R.zernike_plans(R.zernike_terms([(m, m) for m in range(24)])) == 1
    assert R.zernike_plans(R.zernike_terms([(m, m) for m in range(25)])) == 2
    assert R.zernike_plans(R.zernike_terms([(142, 0)])) == 1
    assert R.zernike_plans(R.zernike_terms([(144, 0)])) is None
    assert R.zernike_plans(R.zernike_terms([(4, 0)] * 3)) == 3
    assert R.zernike_plans(R.zernike_terms([(4, 0)] * 3, merge=True)) == 1
    assert R.grid_for(R.sweep(132) + 1, 132) * R.THREADS == R.sweep(132)
