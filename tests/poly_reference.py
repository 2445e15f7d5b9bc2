"""Plain extended-precision references, plan rules and defect models of the polynomial kernels: the 1-D recurrence
families, Clenshaw and radial sums, XY monomials and tensor sums of csrc/orthopoly.cu, the Zernike kernel of
csrc/synthesis.cu and the Forbes Q-bfs, Q-con and 2D-Q kernel of csrc/qpoly.cu.

Every reference runs its recurrence in long double (80-bit on x86-64) from the exact values the device receives (float32
inputs are rounded first; alpha and beta are the doubles the host gets) and returns, beside each value, the majorant M
of the same recurrence run on absolute values, M_k = (|A_k x| + |B_k|) M_{k-1} + |C_k| M_{k-2}, capped by the running
maximum of the values made so far (`tighten`), and sum |w| M for sums.  An fp64 recurrence of n steps lands within a
small multiple of (n + 1) 2^-53 M of the exact value, so the GPU test states every bound as c (n + 1) 2^-53 M, plus
2^-24 |ref| for float32 storage (the fp64 result rounded once).  Without the cap the majorant of a recurrence that is
stable but not positive (Legendre, Q-bfs and 2D-Q inside their intervals) grows like (1 + sqrt 2)^n while the values
stay bounded, and a bound on it would pass a wrong plane above n = 40.

The recurrence coefficients are written from DLMF 18.9 and the Forbes papers (oe-18-19-19700, oe-18-13-13851,
oe-20-3-2483), not from the engine's host code.  The plan and limit rules are mirrored from the C++ so that the GPU
test can put every call on both sides of each limit and count its launches.  The `defect` models are numpy versions of
a kernel with one deliberate fault; tests/test_host_poly_reference.py shows the GPU test's ceilings would catch each.
"""
import numpy as np

from accuracy import LDBL, THREADS, grid_for, sweep  # noqa: F401
U53 = 2.0 ** -53
U24 = 2.0 ** -24

# ceilings of the GPU test's figures c (see c_figure), shown by tests/test_host_poly_reference.py to sit 10x or more
# below every modelled defect; the GPU test's bounds are 1.5x the H100 figures and never above these
CEIL = 1e4

# ---- launch and plan rules (mirrors of csrc/common.cuh, orthopoly.cu, synthesis.cu and qpoly.cu) --------------------
JAC_MAX = 120                   # PB_POLY_NMAX: highest order of a 1-D recurrence
POLY_PLANES = 1024              # PB_POLY_PLANES: output planes per 1-D call (VALUE_DER counts 2 per order)
CLEN_J = 8                      # PB_CLENSHAW_JMAX: highest Clenshaw derivative order
CLEN_LEN = JAC_MAX + 1          # Clenshaw coefficients
XY_PLANES = 1024                # PB_XY_PLANES
XY_ORDER = 32767                # highest XY order (a short)
TSUM_COEFS = 1024               # PB_TSUM_COEFS: (max m + 1)(max n + 1) of a tensor sum
ZERN_GROUPS = 24                # PB_ZERN_GROUPS: |m| groups per plan
ZERN_STEPS = 72                 # PB_ZERN_STEPS: Jacobi steps per plan, so (n - |m|)/2 <= 71
ZERN_SEQ_K = 32767              # modes of pb_zernike_seq
ZERN_DER_K = 16383              # modes of pb_zernike_der
Q_NMAX = 64                     # PB_QPOLY_NMAX: n and |m|
Q_STEPS = 256                   # PB_QPOLY_STEPS
Q_ENTRIES = 1024                # PB_QPOLY_ENTRIES

FAMILIES = ('jacobi', 'cheby1', 'cheby2', 'cheby3', 'cheby4', 'legendre', 'hermite_he', 'hermite_h', 'laguerre',
            'dickson1', 'dickson2')      # the order of capi.POLY_*
SHIFTED = ('jacobi', 'hermite_he', 'hermite_h', 'laguerre')   # POLY_DER by a shifted order, as the reference forms it


def sweep_counts(sm_count):
    """S - 1, S, S + 1 and 2S + 1 samples: both sides of the first sweep and into a third"""
    S = sweep(sm_count)
    return (S - 1, S, S + 1, 2 * S + 1)


def poly_planes(k, kind_value_der):
    return k * (2 if kind_value_der else 1)


def poly_refused(ns, value_der):
    """pb_poly_seq refuses more than 1024 planes or an order above 120"""
    return poly_planes(len(ns), value_der) > POLY_PLANES or max(ns) > JAC_MAX


def tsum_refused(ms, ns):
    return (max(ms) + 1) * (max(ns) + 1) > TSUM_COEFS


def q_steps(groups):
    """steps of a qpoly plan: {(kind, |m|): highest n} -> sum of (highest n + 1)"""
    return sum(n + 1 for n in groups.values())


def q_groups(family, ns, ms=None, coefs=None):
    """the (kind, |m|) groups of a Forbes call and the highest n of each; zero coefficients are skipped"""
    out = {}
    for q, n in enumerate(ns):
        if coefs is not None and coefs[q] == 0.0:
            continue
        am = abs(ms[q]) if family == '2d' else 0
        key = ('bfs' if am == 0 else '2d', am) if family == '2d' else (family, 0)
        out[key] = max(out.get(key, 0), n)
    return out


def zernike_terms(nms, coefs=None, merge=False):
    """(|m|, j, trig) of every Zernike term the plan holds, sorted by (|m|, j) and stable as build_terms; zero weights
    skipped; merge: duplicate (n, m) pairs first add their weights (pb_zernike_sum_der_xy)"""
    terms, seen = [], set()
    for q, (n, m) in enumerate(nms):
        if coefs is not None and coefs[q] == 0.0:
            continue
        t = (abs(m), (n - abs(m)) // 2, 2 if m < 0 else 1)
        if merge and t in seen:
            continue
        seen.add(t)
        terms.append(t)
    return sorted(terms, key=lambda t: (t[0], t[1]))


def zernike_plans(terms):
    """launches of a Zernike call: next_plan's rule (whole |m| groups while 24 groups and 72 steps fit, a repeated
    (n, m) within a plan goes to a later one); None when a group needs more than 72 steps (refused)"""
    plans = 0
    while terms:
        plans += 1
        rest, ngroups, nsteps, full, pos = [], 0, 0, False, 0
        while pos < len(terms):
            end, njmax = pos, 0
            while end < len(terms) and terms[end][0] == terms[pos][0]:
                njmax = max(njmax, terms[end][1])
                end += 1
            if njmax + 1 > ZERN_STEPS:
                return None
            if full or ngroups == ZERN_GROUPS or nsteps + njmax + 1 > ZERN_STEPS:
                full = True
                rest.extend(terms[pos:end])
                pos = end
                continue
            ngroups += 1
            used = set()
            for t in terms[pos:end]:
                if (t[1], t[2]) in used:
                    rest.append(t)
                else:
                    used.add((t[1], t[2]))
            nsteps += njmax + 1
            pos = end
        terms = rest
    return plans


def noll_to_nm(j):
    """Noll index j >= 1 -> (n, m)"""
    n = 0
    while (n + 1) * (n + 2) // 2 < j:
        n += 1
    k = j - n * (n + 1) // 2 - 1
    ms = [m for m in range(-n, n + 1, 2)]
    ams = sorted({abs(m) for m in ms})
    order = []
    for am in ams:
        if am == 0:
            order.append(0)
        else:
            first = n * (n + 1) // 2 + 1 + len(order)
            order.extend([am, -am] if first % 2 == 0 else [-am, am])
    return n, order[k]


# ---- sample points ---------------------------------------------------------------------------------------------------
def f32(v):
    return np.asarray(v, np.float64).astype(np.float32).astype(np.float64)


def interval_points(lo=-1.0, hi=1.0, out=(), seed=0, n=64):
    """points exact in float32 on [lo, hi]: the ends, 0 and +-2^-30, clusters within a few float32 ulps of the ends,
    a uniform spread, and the points `out` outside the interval"""
    rng = np.random.default_rng(seed)
    k = np.arange(1, 9)
    ends = [lo, hi, 0.0, 2.0 ** -30, -2.0 ** -30, 2.0 ** -30 * (1 + 2.0 ** -23), -1.2345e-9, 7.654e-8]
    clus = list(hi - k * 2.0 ** -23 * abs(hi))
    if lo != 0:
        clus += list(lo + k * 2.0 ** -23 * abs(lo))
    v = np.concatenate([ends, clus, rng.uniform(lo, hi, n), list(out)])
    return np.unique(f32(v))


def family_points(fam, n=120):
    if fam in ('hermite_he', 'hermite_h'):
        return interval_points(-16.0, 16.0, (-16.0, 16.0))
    if fam == 'laguerre':
        return interval_points(0.0, 4.0 * max(n, 1), (-0.5, -2.0 ** -30))
    return interval_points(-1.0, 1.0, (-1.5, 1.5, -1.25, 1.0 + 2.0 ** -20))


JACOBI_AB = ((0.0, 0.0), (0.5, -0.5), (-0.5, -0.5), (0.0, -1.0 + 2.0 ** -10), (7.5, 12.0), (-0.5, -0.75),
             (0.7, 0.0), (2.0, 3.0))
"""alpha + beta = 0 and (near) -1 (the n = 0 branch of jacobi_abc), large, negative and a non-dyadic 0.7"""


# ---- 1-D families ------------------------------------------------------------------------------------------------
def family_abc(fam, k, alpha=0.0, beta=0.0):
    """(A, B, C) in long double with P_k = (A x + B) P_{k-1} - C P_{k-2}, k >= 1 (DLMF 18.9.1-2, 18.9.7, 18.9.21-22,
    18.9.13; Dickson D_k = x D_{k-1} - a D_{k-2})"""
    a, b, n = LDBL(alpha), LDBL(beta), LDBL(k - 1)
    if fam == 'jacobi':
        s = a + b
        if k == 1:
            return (s + 2) / 2, (a - b) / 2, LDBL(0)
        A = (2 * n + s + 1) * (2 * n + s + 2) / (2 * (n + 1) * (n + s + 1))
        B = (a * a - b * b) * (2 * n + s + 1) / (2 * (n + 1) * (n + s + 1) * (2 * n + s))
        C = (n + a) * (n + b) * (2 * n + s + 2) / ((n + 1) * (n + s + 1) * (2 * n + s))
        return A, B, C
    kk = LDBL(k)
    if fam.startswith('cheby'):
        if k == 1:
            return {'cheby1': (LDBL(1), LDBL(0)), 'cheby2': (LDBL(2), LDBL(0)), 'cheby3': (LDBL(2), LDBL(-1)),
                    'cheby4': (LDBL(2), LDBL(1))}[fam] + (LDBL(0),)
        return LDBL(2), LDBL(0), LDBL(1)
    if fam == 'legendre':
        return (2 * kk - 1) / kk, LDBL(0), (kk - 1) / kk
    if fam == 'hermite_he':
        return LDBL(1), LDBL(0), kk - 1
    if fam == 'hermite_h':
        return LDBL(2), LDBL(0), 2 * (kk - 1)
    if fam == 'laguerre':
        return -1 / kk, (2 * kk - 1 + a) / kk, (kk - 1 + a) / kk
    return LDBL(1), LDBL(0), a                               # dickson1, dickson2


def family_p0(fam):
    return LDBL(2) if fam == 'dickson1' else LDBL(1)


def rec1d(fam, x, nmax, alpha=0.0, beta=0.0):
    """(P, dP, M, dM), each (nmax + 1, len(x)) long double: the values, their x derivatives (the differentiated
    recurrence) and their error scales (`tighten`).  The Dickson-1 P_1 = x (D_1 = x D_0 / 2)."""
    x = np.asarray(x, LDBL)
    P = np.zeros((nmax + 1, x.size), LDBL)
    dP, M, dM = np.zeros_like(P), np.zeros_like(P), np.zeros_like(P)
    P[0] = family_p0(fam)
    M[0] = abs(P[0])
    for k in range(1, nmax + 1):
        A, B, C = family_abc(fam, k, alpha, beta)
        if fam == 'dickson1' and k == 1:
            A, B = LDBL(0.5), LDBL(0)
        lin, mlin = A * x + B, abs(A * x) + abs(B)
        p2, m2, dp2, dm2 = (P[k - 2], M[k - 2], dP[k - 2], dM[k - 2]) if k >= 2 else (0, 0, 0, 0)
        P[k] = lin * P[k - 1] - C * p2
        M[k] = mlin * M[k - 1] + abs(C) * m2
        if fam == 'jacobi' and k == 1:
            # the kernels (and the reference package) form P_1 as (a + 1) + (a + b + 2)(x - 1)/2, whose rounding is
            # relative to these terms: with a = b it keeps only the bits of x that 1 - x keeps
            M[1] = abs(LDBL(alpha) + 1) + abs(A) * abs(x - 1)
        dP[k] = A * P[k - 1] + lin * dP[k - 1] - C * dp2
        dM[k] = abs(A) * M[k - 1] + mlin * dM[k - 1] + abs(C) * dm2
    return P, dP, *tighten(P, dP, M, dM)


def tighten(P, dP, M, dM):
    """the error scales of a forward recurrence: the majorants M, dM capped by the running maxima over the orders
    made so far, max_{k' <= k} |P_k'| (and |dP_k'| + |P_k'| for the derivative).  Where the recurrence is stable but
    not positive (|A x| + |B| above |A x + B|, as inside the orthogonality interval) the majorant grows like
    (1 + sqrt 2)^k while the values and the rounding errors stay bounded; the cap keeps the bound tight at every
    order.  Where the majorant is the smaller (a seed such as Chebyshev-1's P_1 = x near 0), it stays."""
    R = np.maximum.accumulate(abs(P), axis=0)
    dR = np.maximum.accumulate(abs(dP), axis=0) + R
    return np.minimum(M, R), np.minimum(dM, dR)


def shifted_der(fam, x, ns, alpha=0.0, beta=0.0):
    """(value, majorant) of POLY_DER of the shifted families: 0.5 (n + a + b + 1) P_{n-1}^(a+1, b+1), n He_{n-1},
    2n H_{n-1} and -L_{n-1}^(a+1); (len(ns), len(x))"""
    a, b = (alpha + 1, beta + 1) if fam == 'jacobi' else ((alpha + 1, beta) if fam == 'laguerre' else (alpha, beta))
    nm = max(max(ns) - 1, 0)
    P, _, M, _ = rec1d(fam, x, nm, a, b)
    out, maj = np.zeros((len(ns), len(x)), LDBL), np.zeros((len(ns), len(x)), LDBL)
    for q, n in enumerate(ns):
        if n == 0:
            continue
        sc = {'jacobi': (n + LDBL(alpha) + LDBL(beta) + 1) / 2, 'laguerre': LDBL(-1), 'hermite_he': LDBL(n),
              'hermite_h': LDBL(2 * n)}[fam]
        out[q], maj[q] = sc * P[n - 1], abs(sc) * M[n - 1]
    return out, maj


def clenshaw_ref(s, x, j, alpha=0.0, beta=0.0):
    """(table, majorant), each (j + 1, max(len(s), 2), len(x)): Clenshaw's alpha_jj[n] =
    (jj A_n alpha_{jj-1}[n+1] or s_n) + (A_n x + B_n) alpha_jj[n+1] - C_{n+1} alpha_jj[n+2], 0 for n > M - jj, with
    (A_n, B_n, C_n) the DLMF 18.9.2 step from P_n to P_{n+1}.  alpha_jj[0] is the jj-th x derivative of sum s_n P_n.
    The majorant of the backward recurrence is capped as `tighten` caps a forward one: by the running maxima (n
    descending) of the planes jj' <= jj and of |s|."""
    x = np.asarray(x, LDBL)
    L = len(s)
    N, Mx = max(L, 2), L - 1
    T, TM = np.zeros((j + 1, N + 2, x.size), LDBL), np.zeros((j + 1, N + 2, x.size), LDBL)
    for n in range(N - 1, -1, -1):
        A, B, _ = family_abc('jacobi', n + 1, alpha, beta)
        C1 = family_abc('jacobi', n + 2, alpha, beta)[2]
        for jj in range(j, -1, -1):
            if n > Mx - jj:
                continue
            head = LDBL(s[n]) if jj == 0 else jj * A * T[jj - 1, n + 1]
            mhead = abs(LDBL(s[n])) if jj == 0 else jj * abs(A) * TM[jj - 1, n + 1]
            T[jj, n] = head + (A * x + B) * T[jj, n + 1] - C1 * T[jj, n + 2]
            TM[jj, n] = mhead + (abs(A * x) + abs(B)) * TM[jj, n + 1] + abs(C1) * TM[jj, n + 2]
    T, TM = T[:, :N], TM[:, :N]
    run = np.maximum.accumulate(abs(T)[:, ::-1], axis=1)[:, ::-1]               # max over n' >= n
    srun = np.maximum.accumulate(abs(np.asarray(list(s) + [0.0] * (N - L), LDBL))[::-1])[::-1]
    R = np.cumsum(run, axis=0) + srun[None, :, None]
    return T, np.minimum(TM, R)


def radial_sum_ref(coefs, ns, x, y, radius, alpha=0.0, beta=0.0):
    """(z, dz/dx, dz/dy) and their majorants of sum c P_n^(a,b)(u), u = 2 (x^2 + y^2) / R^2 - 1"""
    x, y = np.asarray(x, LDBL), np.asarray(y, LDBL)
    R2 = LDBL(radius) * LDBL(radius)
    u = 2 * (x * x + y * y) / R2 - 1
    P, dP, M, dM = rec1d('jacobi', u, max(ns), alpha, beta)
    z, dz, mz, mdz = (np.zeros(x.size, LDBL) for _ in range(4))
    for c, n in zip(coefs, ns):
        z += LDBL(c) * P[n]
        dz += LDBL(c) * dP[n]
        mz += abs(LDBL(c)) * M[n]
        mdz += abs(LDBL(c)) * dM[n]
    gx, gy = 4 * x / R2, 4 * y / R2
    return (z, dz * gx, dz * gy), (mz, mdz * abs(gx) + mz * U53, mdz * abs(gy) + mz * U53)


# ---- Zernike -----------------------------------------------------------------------------------------------------
def zernike_norm(n, m):
    return np.sqrt(LDBL(2 * (n + 1)) / (2 if m == 0 else 1))


def _zern_parts(n, m, r2):
    """(P, dP/dx2, M, dM) of P_j^(0,|m|)(2 r^2 - 1), j = (n - |m|)/2"""
    am = abs(m)
    j = (n - am) // 2
    P, dP, M, dM = rec1d('jacobi', 2 * r2 - 1, j, 0.0, float(am))
    return P[j], dP[j], M[j], dM[j]


def _powc(x, y, k):
    """Re, Im (x + iy)^k by repeated multiplication in long double"""
    c, s = np.ones_like(x), np.zeros_like(x)
    for _ in range(k):
        c, s = c * x - s * y, c * y + s * x
    return c, s


def zernike_ref(n, m, a, b, polar, norm=True):
    """(Z, majorant) at (r, t) when polar, else at (x, y)"""
    a, b = np.asarray(a, LDBL), np.asarray(b, LDBL)
    am = abs(m)
    if polar:
        r, t = a, b
        H = (r ** am) * (np.sin(am * t) if m < 0 else np.cos(am * t))
        Hm = r ** am
    else:
        r = np.sqrt(a * a + b * b)
        c, s = _powc(a, b, am)
        H, Hm = (s if m < 0 else c), r ** am
    P, _, M, _ = _zern_parts(n, m, r * r)
    w = zernike_norm(n, m) if norm else LDBL(1)
    return w * P * H, w * M * Hm


def zernike_der_ref(n, m, a, b, cartesian, norm=True):
    """((d0, d1), (M0, M1)): (dZ/dr, dZ/dt) at (r, t), or (dZ/dx, dZ/dy) at (x, y)"""
    a, b = np.asarray(a, LDBL), np.asarray(b, LDBL)
    am = abs(m)
    w = zernike_norm(n, m) if norm else LDBL(1)
    if not cartesian:
        r, t = a, b
        P, dP, M, dM = _zern_parts(n, m, r * r)
        cs, sn = np.cos(am * t), np.sin(am * t)
        rm, rm1 = r ** am, (r ** (am - 1) if am > 0 else np.zeros_like(r))
        radial = am * rm1 * P + rm * 4 * r * dP
        mrad = am * abs(rm1) * M + abs(rm) * 4 * abs(r) * dM
        if m < 0:
            return (w * radial * sn, w * am * cs * rm * P), (w * mrad, w * am * abs(rm) * M)
        return (w * radial * cs, -w * am * sn * rm * P), (w * mrad, w * am * abs(rm) * M)
    x, y = a, b
    r2 = x * x + y * y
    P, dP, M, dM = _zern_parts(n, m, r2)
    hc, hs = _powc(x, y, am)
    gc, gs = _powc(x, y, am - 1) if am > 0 else (np.zeros_like(x), np.zeros_like(x))
    rm, rm1 = np.sqrt(r2) ** am, (np.sqrt(r2) ** (am - 1) if am > 0 else np.zeros_like(x))
    if m < 0:
        dx, dy = 4 * x * dP * hs + am * P * gs, 4 * y * dP * hs + am * P * gc
    else:
        dx, dy = 4 * x * dP * hc + am * P * gc, 4 * y * dP * hc - am * P * gs
    mx = 4 * abs(x) * dM * rm + am * M * rm1
    my = 4 * abs(y) * dM * rm + am * M * rm1
    return (w * dx, w * dy), (w * mx, w * my)


def zernike_sum_ref(coefs, nms, a, b, polar, norm=True, der=False):
    """sum c Z (and with der, the Cartesian slopes) with duplicate (n, m) pairs each counted; (values, majorants)"""
    out = [np.zeros(np.size(a), LDBL) for _ in range(3 if der else 1)]
    maj = [np.zeros(np.size(a), LDBL) for _ in range(3 if der else 1)]
    for c, (n, m) in zip(coefs, nms):
        if c == 0.0:
            continue
        v, mv = zernike_ref(n, m, a, b, polar, norm)
        out[0] += LDBL(c) * v
        maj[0] += abs(LDBL(c)) * mv
        if der:
            (dx, dy), (mx, my) = zernike_der_ref(n, m, a, b, True, norm)
            out[1] += LDBL(c) * dx
            out[2] += LDBL(c) * dy
            maj[1] += abs(LDBL(c)) * mx
            maj[2] += abs(LDBL(c)) * my
    return out, maj


def zernike_points(n=48, seed=3):
    """(r, t) exact in float32: r = 0, 1, 1 + 2^-20 and a spread, t up to +-1e3 rad"""
    rng = np.random.default_rng(seed)
    r = f32(np.concatenate([[0.0, 1.0, 1.0 + 2.0 ** -20, 2.0 ** -30, 1.0 - 2.0 ** -24, 0.5], rng.uniform(0, 1, n)]))
    t = f32(np.concatenate([[0.0, 1e3, -1e3, np.pi, 0.5, -2.0], rng.uniform(-np.pi, np.pi, n)]))
    return r, t


def zernike_xy_points(n=48, seed=4):
    """(x, y) exact in float32: the origin, points on and just past the unit circle and a spread"""
    rng = np.random.default_rng(seed)
    x = f32(np.concatenate([[0.0, 1.0, 0.0, 0.6, -1.0 - 2.0 ** -20, 2.0 ** -30], rng.uniform(-0.71, 0.71, n)]))
    y = f32(np.concatenate([[0.0, 0.0, -1.0, 0.8, 0.0, -2.0 ** -30], rng.uniform(-0.71, 0.71, n)]))
    return x, y


# ---- Forbes polynomials ------------------------------------------------------------------------------------------
def qbfs_tables(nmax, one=LDBL, sqrt=np.sqrt):
    """f, g, h of the Q-bfs recurrence (oe-18-19-19700 A.14-A.16)"""
    f, g, h = [one(0)] * (nmax + 1), [one(0)] * (nmax + 1), [one(0)] * (nmax + 1)
    for k in range(nmax + 1):
        if k == 0:
            f[k] = one(2)
        elif k == 1:
            f[k] = sqrt(one(19)) / 2
        else:
            f[k] = sqrt(one(k * (k + 1) + 3) - g[k - 1] ** 2 - h[k - 2] ** 2)
        h[k] = -one((k + 2) * (k + 1)) / (2 * f[k])
        g[k] = -one(1) / 2 if k == 0 else -(1 + g[k - 1] * h[k - 1]) / f[k]
    return f, g, h


def q2d_gamma(n, m, one=LDBL):
    v = one(3) / 8
    for mm in range(3, m + 1):
        v *= one(2 * (mm - 1) + 1) / (2 * (mm - 2))
    for k in range(2, n + 1):
        v *= one(k) * (2 * m + 2 * (k - 1) - 1) / ((m + (k - 1) - 2) * one(2 * (k - 1) + 1))
    return v


def q2d_F(n, m, one=LDBL):
    """F(n, m) of oe-20-3-2483 A.13 (m >= 1)"""
    nn, mm = one(n), one(m)
    if n == 0:
        if m == 1:
            return one(1) / 4
        v = one(1) / 8
        for k in range(3, m + 1):
            v *= one(2 * k - 3) / (2 * (k - 1))
        return mm * mm * v
    if m == 1:
        return (4 * (nn - 1) ** 2 * nn * nn + 1) / (8 * (2 * nn - 1) ** 2) + (one(11) / 32 if n == 1 else 0)
    chi = mm + nn - 2
    num = 2 * nn * chi * (3 - 5 * mm + 4 * nn * chi) + mm * mm * (3 - mm + 4 * nn * chi)
    den = (mm + 2 * nn - 3) * (mm + 2 * nn - 2) * (mm + 2 * nn - 1) * (2 * nn - 1)
    return num / den * q2d_gamma(n, m, one)


def q2d_G(n, m, one=LDBL):
    """G(n, m) of oe-20-3-2483 A.13 (m >= 1)"""
    nn, mm = one(n), one(m)
    if n == 0:
        v = one(1) / 4
        for k in range(2, m + 1):
            v *= one(2 * k - 1) / (2 * (k - 1))
        return v
    if m == 1:
        return -((2 * nn * nn - 1) * (nn * nn - 1)) / (8 * (4 * nn * nn - 1)) - (one(1) / 24 if n == 1 else 0)
    num = (2 * nn * (mm + nn - 1) - mm) * ((nn + 1) * (2 * mm + 2 * nn - 1))
    den = (mm + 2 * nn - 2) * (mm + 2 * nn - 1) * (mm + 2 * nn) * (2 * nn + 1)
    return -num / den * q2d_gamma(n, m, one)


def q2d_fg(nmax, m, one=LDBL, sqrt=np.sqrt):
    f, g = [], []
    for k in range(nmax + 1):
        f.append(sqrt(q2d_F(0, m, one)) if k == 0 else sqrt(q2d_F(k, m, one) - g[k - 1] ** 2))
        g.append(q2d_G(k, m, one) / f[k])
    return f, g


def q2d_abc(n, m, one=LDBL):
    """A, B, C of P_{n+1}^m = (A + B u) P_n^m - C P_{n-1}^m (oe-20-3-2483 A.3)"""
    nn, mm = one(n), one(m)
    D = (4 * nn * nn - 1) * (mm + nn - 2) * (mm + 2 * nn - 3)
    A = (2 * nn - 1) * (mm + 2 * nn - 2) * (4 * nn * (mm + nn - 2) + (mm - 3) * (2 * mm - 1)) / D
    B = -2 * (2 * nn - 1) * (mm + 2 * nn - 3) * (mm + 2 * nn - 2) * (mm + 2 * nn - 1) / D
    C = nn * (2 * nn - 3) * (mm + 2 * nn - 1) * (2 * mm + 2 * nn - 3) / D
    return A, B, C


def _qseries(kind, am, u, nmax):
    """(Q, dQ/dv, MQ, dMQ) of one Forbes recurrence, (nmax + 1, len(u)), v = u (Q-bfs, 2D-Q) or 2u - 1 (Q-con)"""
    u = np.asarray(u, LDBL)
    Z = np.zeros((nmax + 1, u.size), LDBL)
    P, dP, MP, dMP, Q, dQ, MQ, dMQ = (Z.copy() for _ in range(8))
    if kind == 'con':
        Pj, dPj, Mj, dMj = rec1d('jacobi', 2 * u - 1, nmax, 0.0, 4.0)
        return Pj, dPj, Mj, dMj
    if kind == 'bfs':
        f, g, h = qbfs_tables(max(nmax, 1))
        for j in range(nmax + 1):
            if j == 0:
                P[0], MP[0] = 2, 2
            elif j == 1:
                P[1], dP[1], MP[1], dMP[1] = 6 - 8 * u, -8, 6 + 8 * abs(u), 8
            else:
                lin, ml = 2 - 4 * u, 2 + 4 * abs(u)
                P[j] = lin * P[j - 1] - P[j - 2]
                dP[j] = -4 * P[j - 1] + lin * dP[j - 1] - dP[j - 2]
                MP[j] = ml * MP[j - 1] + MP[j - 2]
                dMP[j] = 4 * MP[j - 1] + ml * dMP[j - 1] + dMP[j - 2]
            gq = g[j - 1] if j >= 1 else 0
            hq = h[j - 2] if j >= 2 else 0
            q1, q2 = (Q[j - 1], Q[j - 2]) if j >= 2 else ((Q[0], 0) if j == 1 else (0, 0))
            d1, d2 = (dQ[j - 1], dQ[j - 2]) if j >= 2 else ((dQ[0], 0) if j == 1 else (0, 0))
            m1, m2 = (MQ[j - 1], MQ[j - 2]) if j >= 2 else ((MQ[0], 0) if j == 1 else (0, 0))
            e1, e2 = (dMQ[j - 1], dMQ[j - 2]) if j >= 2 else ((dMQ[0], 0) if j == 1 else (0, 0))
            Q[j] = (P[j] - gq * q1 - hq * q2) / f[j]
            dQ[j] = (dP[j] - gq * d1 - hq * d2) / f[j]
            MQ[j] = (MP[j] + abs(gq) * m1 + abs(hq) * m2) / f[j]
            dMQ[j] = (dMP[j] + abs(gq) * e1 + abs(hq) * e2) / f[j]
        return (Q, dQ) + tighten(Q, dQ, MQ, dMQ)
    f, g = q2d_fg(nmax, am)
    for j in range(nmax + 1):
        if j == 0:
            P[0], MP[0] = LDBL(1) / 2, LDBL(1) / 2
        elif j == 1:
            a0, a1 = (LDBL(1), LDBL(-1) / 2) if am == 1 else (LDBL(am) - LDBL(1) / 2, LDBL(1 - am))
            P[1], dP[1], MP[1], dMP[1] = a0 + a1 * u, a1, abs(a0) + abs(a1 * u), abs(a1)
        elif am == 1 and j in (2, 3):
            cf = [LDBL(3), LDBL(-12), LDBL(8)] if j == 2 else [LDBL(5), LDBL(-60), LDBL(120), LDBL(-64)]
            den = LDBL(6 if j == 2 else 10)
            P[j] = sum(c * u ** k for k, c in enumerate(cf)) / den
            dP[j] = sum(k * c * u ** (k - 1) for k, c in enumerate(cf) if k) / den
            MP[j] = sum(abs(c) * abs(u) ** k for k, c in enumerate(cf)) / den
            dMP[j] = sum(k * abs(c) * abs(u) ** (k - 1) for k, c in enumerate(cf) if k) / den
        else:
            A, B, C = q2d_abc(j - 1, am)
            lin, ml = A + B * u, abs(A) + abs(B * u)
            P[j] = lin * P[j - 1] - C * P[j - 2]
            dP[j] = B * P[j - 1] + lin * dP[j - 1] - C * dP[j - 2]
            MP[j] = ml * MP[j - 1] + abs(C) * MP[j - 2]
            dMP[j] = abs(B) * MP[j - 1] + ml * dMP[j - 1] + abs(C) * dMP[j - 2]
        if j == 0:
            Q[0], MQ[0] = P[0] / f[0], MP[0] / f[0]
        else:
            Q[j] = (P[j] - g[j - 1] * Q[j - 1]) / f[j]
            dQ[j] = (dP[j] - g[j - 1] * dQ[j - 1]) / f[j]
            MQ[j] = (MP[j] + abs(g[j - 1]) * MQ[j - 1]) / f[j]
            dMQ[j] = (dMP[j] + abs(g[j - 1]) * dMQ[j - 1]) / f[j]
    return (Q, dQ) + tighten(Q, dQ, MQ, dMQ)


def qpoly_ref(family, n, m, a, b=None, kind='value'):
    """(planes, majorants) of one Forbes mode: kind 'value' -> (v,), 'der' -> (d/dr,) or for 2D-Q (d/dr, d/dt),
    'der_xy' -> (d/dx, d/dy) (2D-Q).  a = r (or x), b = t (or y)."""
    a = np.asarray(a, LDBL)
    b = np.zeros_like(a) if b is None else np.asarray(b, LDBL)
    am = abs(m) if family == '2d' else 0
    if kind == 'der_xy':
        u = a * a + b * b
        r = np.sqrt(u)
    else:
        r = a
        u = r * r
    gk = family if family != '2d' else ('bfs' if am == 0 else '2d')
    Q, dQ, MQ, dMQ = (s[n] for s in _qseries(gk, am, u, n))
    if gk == 'bfs':
        env, denv = u * (1 - u), 1 - 2 * u
        menv = abs(u) * (1 + abs(u))
        if kind == 'value':
            return (env * Q,), (menv * MQ,)
        if kind == 'der':
            return ((2 * r * denv * Q + env * 2 * r * dQ),), (2 * abs(r) * ((1 + 2 * abs(u)) * MQ + menv * dMQ),)
        com, mcom = denv * Q + env * dQ, (1 + 2 * abs(u)) * MQ + menv * dMQ
        return (2 * a * com, 2 * b * com), (2 * abs(a) * mcom, 2 * abs(b) * mcom)
    if gk == 'con':
        if kind == 'value':
            return (u * u * Q,), (u * u * MQ,)
        return ((4 * r ** 3 * Q + 4 * r ** 5 * dQ),), (4 * abs(r) ** 3 * MQ + 4 * abs(r) ** 5 * dMQ,)
    if kind == 'der_xy':
        hc, hs = _powc(a, b, am)
        gc, gs = _powc(a, b, am - 1)
        H, dHx, dHy = (hs, am * gs, am * gc) if m < 0 else (hc, am * gc, -am * gs)
        rm, rm1 = r ** am, r ** (am - 1)
        return ((2 * a * dQ * H + Q * dHx, 2 * b * dQ * H + Q * dHy),
                (2 * abs(a) * dMQ * rm + MQ * am * rm1, 2 * abs(b) * dMQ * rm + MQ * am * rm1))
    t = b
    cs, sn = np.cos(am * t), np.sin(am * t)
    trig, dtrig = (sn, am * cs) if m < 0 else (cs, -am * sn)
    rm, rm1 = r ** am, r ** (am - 1)
    if kind == 'value':
        return (Q * trig * rm,), (MQ * rm,)
    return ((trig * (am * rm1 * Q + 2 * rm * r * dQ), dtrig * rm * Q),
            (am * rm1 * MQ + 2 * rm * abs(r) * dMQ, am * rm * MQ))


def qpoly_sum_ref(family, ns, ms, coefs, r, t=None, der=False):
    """(z, dz/dr, dz/dt) and majorants of sum c Q_n^m: the sums of the modes' values and majorants"""
    outs, majs = None, None
    for q, (n, c) in enumerate(zip(ns, coefs)):
        if c == 0.0:
            continue
        m = ms[q] if family == '2d' else 0
        v, mv = qpoly_ref(family, n, m, r, t, 'value')
        vals, maj = list(v), list(mv)
        if der:
            d, md = qpoly_ref(family, n, m, r, t, 'der')
            if family == '2d' and len(d) == 1:          # an m = 0 (Q-bfs) term adds nothing to dz/dt
                d, md = d + (np.zeros(np.size(r), LDBL),), md + (np.zeros(np.size(r), LDBL),)
            vals += list(d)
            maj += list(md)
        if outs is None:
            outs = [np.zeros(np.size(r), LDBL) for _ in vals]
            majs = [np.zeros(np.size(r), LDBL) for _ in vals]
        for k in range(len(vals)):
            outs[k] += LDBL(c) * vals[k]
            majs[k] += abs(LDBL(c)) * maj[k]
    return outs, majs


def q_points(seed=5, n=40):
    """(r, t) exact in float32: r = 0, 1, clusters at 1, a spread on [0, 1] and 1 + 2^-20; t up to +-1e3"""
    rng = np.random.default_rng(seed)
    r = f32(np.concatenate([[0.0, 1.0, 1.0 - 2.0 ** -24, 1.0 + 2.0 ** -20, 2.0 ** -30, 0.5], rng.uniform(0, 1, n)]))
    t = f32(np.concatenate([[0.0, 1e3, -1e3, 0.25, 3.0, -1.0], rng.uniform(-np.pi, np.pi, n)]))
    return r, t


# ---- XY monomials and tensor sums ----------------------------------------------------------------------------------
def mono(z, k, der):
    """(value, majorant) of z^k or d/dz z^k in long double"""
    z = np.asarray(z, LDBL)
    if der:
        v = np.zeros_like(z) if k == 0 else k * z ** (k - 1)
    else:
        v = z ** k
    return v, abs(v)


def xy_ref(m, n, kind, x, y):
    vx, mx = mono(x, m, kind & 1)
    vy, my = mono(y, n, kind & 2)
    return vx * vy, mx * my


def tensor_ref(basis, coefs, ms, ns, x, y, sx=1.0, sy=1.0):
    """((z, dz/dx / sx, dz/dy / sy), majorants) of sum c P_m(x) P_n(y), P monomials or Chebyshev-1; x, y elementwise"""
    fam = 'cheby1'
    x, y = np.asarray(x, LDBL), np.asarray(y, LDBL)
    Mx, My = max(ms), max(ns)
    if basis == 'cheby1':
        Px, dPx, MPx, dMPx = rec1d(fam, x, Mx)
        Py, dPy, MPy, dMPy = rec1d(fam, y, My)
    else:
        Px = np.array([x ** k for k in range(Mx + 1)])
        dPx = np.array([k * x ** (k - 1) if k else np.zeros_like(x) for k in range(Mx + 1)])
        Py = np.array([y ** k for k in range(My + 1)])
        dPy = np.array([k * y ** (k - 1) if k else np.zeros_like(y) for k in range(My + 1)])
        MPx, dMPx, MPy, dMPy = abs(Px), abs(dPx), abs(Py), abs(dPy)
    z, zx, zy, mz, mzx, mzy = (np.zeros(x.size, LDBL) for _ in range(6))
    for c, m, n in zip(coefs, ms, ns):
        c = LDBL(c)
        z += c * Px[m] * Py[n]
        zx += c * dPx[m] * Py[n]
        zy += c * Px[m] * dPy[n]
        mz += abs(c) * MPx[m] * MPy[n]
        mzx += abs(c) * dMPx[m] * MPy[n]
        mzy += abs(c) * MPx[m] * dMPy[n]
    return (z, zx / LDBL(sx), zy / LDBL(sy)), (mz, mzx / abs(LDBL(sx)), mzy / abs(LDBL(sy)))


# ---- figures -------------------------------------------------------------------------------------------------------
def c_figure(got, ref, maj, steps, f32_storage):
    """the smallest c with |got - ref| <= c (steps + 1) 2^-53 M + 4 (steps + 1) 2^-1074 (+ 2^-24 |ref| + 2^-150 for
    float32 storage) at every element; inf where got is NaN, or non-finite where ref is finite.  Elements whose
    reference overflows float32 must be inf of the right sign and are left out."""
    got = np.asarray(got, np.float64)
    ref = np.asarray(ref, LDBL)
    maj = np.asarray(maj, LDBL)
    steps = np.asarray(steps, np.float64)
    if f32_storage:
        over = abs(ref) > LDBL(np.finfo(np.float32).max) * (1 + LDBL(U24) / 2)
        if np.any(over):
            if not np.all(np.isinf(got[over]) & (np.sign(got[over]) == np.sign(ref[over].astype(np.float64)))):
                return float('inf')
            got, ref, maj = got[~over], ref[~over], maj[~over]
            steps = np.broadcast_to(steps, over.shape)[~over] if steps.ndim else steps
    if not np.all(np.isfinite(got)):
        return float('inf')
    # values below the normal range (x^k at x = 2^-30, r^|m| at r = 2^-30) lose bits to gradual underflow: up to a
    # few units of the smallest subnormal per step
    err = np.maximum(abs(got.astype(LDBL) - ref) - 4 * (LDBL(steps) + 1) * LDBL(2.0 ** -1074), 0)
    if f32_storage:
        err = np.maximum(err - LDBL(U24) * abs(ref) - LDBL(2.0 ** -150), 0)
    den = (LDBL(steps) + 1) * LDBL(U53) * maj
    with np.errstate(divide='ignore', invalid='ignore'):
        c = np.where(err == 0, LDBL(0), err / np.where(den > 0, den, LDBL(np.finfo(np.float64).tiny)))
    return float(c.max()) if c.size else 0.0


# ---- defect models -------------------------------------------------------------------------------------------------
def model_1d(fam, x, nmax, alpha=0.0, beta=0.0, defect=None, dtype=np.float64, start=2):
    """numpy restatement of poly1d_kernel's value track, in fp64 with one optional fault:
    'f32_step' rounds each new P_k to float32; 'order_off' uses the coefficients of order k + 1 for the step that
    makes P_k; 'jacobi_seed' forms Chebyshev-1's P_1 in the Jacobi form 1 + 2 (x - 1)/2.  'f32_step' starts at order
    `start`.  Rounded to dtype."""
    x = np.asarray(x, np.float64)
    P = np.zeros((nmax + 1, x.size))
    P[0] = float(family_p0(fam))
    if nmax >= 1:
        A, B, _ = (float(v) for v in family_abc(fam, 1, alpha, beta))
        if fam == 'jacobi':
            P[1] = (alpha + 1) + (alpha + beta + 2) * ((x - 1.0) / 2.0)
        elif defect == 'jacobi_seed' and fam == 'cheby1':
            P[1] = 1.0 + 2.0 * ((x - 1.0) / 2.0)
        else:
            P[1] = (0.5 if fam == 'dickson1' else A) * x + B
    with np.errstate(over='ignore', invalid='ignore'):     # a float32 defect may overflow; c_figure reports it
        for k in range(2, nmax + 1):
            A, B, C = (float(v) for v in family_abc(fam, k + 1 if defect == 'order_off' else k, alpha, beta))
            P[k] = (A * x + B) * P[k - 1] - C * P[k - 2]
            if defect == 'f32_step' and k >= start:
                P[k] = P[k].astype(np.float32)
        return P.astype(dtype)


def model_qbfs(u, nmax, defect=None, start=40):
    """numpy restatement of the Q-bfs value track (Q_n before the u (1 - u) prefix) in fp64 with fp64 tables and one
    optional fault from order `start` on: 'plane_off' writes Q_{n+1} into plane n, 'h_index' uses h[n-1] where the
    recurrence takes h[n-2], 'f32_step' rounds each Q_n to float32"""
    u = np.asarray(u, np.float64)
    f, g, h = (np.array([float(v) for v in t]) for t in qbfs_tables(nmax + 1))
    P = [np.full(u.shape, 2.0), 6.0 - 8.0 * u]
    Q = [np.ones(u.shape), (13.0 - 16.0 * u) / np.sqrt(19.0)]
    for j in range(2, nmax + 2):
        P.append((2.0 - 4.0 * u) * P[j - 1] - P[j - 2])
        hh = h[j - 1] if defect == 'h_index' and j >= start else h[j - 2]
        q = (P[j] - g[j - 1] * Q[j - 1] - hh * Q[j - 2]) / f[j]
        if defect == 'f32_step' and j >= start:
            q = q.astype(np.float32).astype(np.float64)
        Q.append(q)
    Q = np.array(Q)
    out = Q[:nmax + 1].copy()
    if defect == 'plane_off':
        out[start:] = Q[start + 1:nmax + 2]
    return out


def model_zernike_sum(coefs, nms, r, t, defect=None, split=None):
    """zernike_sum at (r, t) in fp64, stored as float32, with the terms split into two plans at index `split` (one plan
    when None); 'partial_f32' rounds the first plan's sum to float32 before the second adds to it (the kernel before
    its partial sums were staged in fp64); 'r_f32' forms r^|m| in float32."""
    r = np.asarray(r, np.float64)
    t = np.asarray(t, np.float64)
    parts = [list(range(len(nms)))] if split is None else [list(range(split)), list(range(split, len(nms)))]
    acc = np.zeros(r.size)
    for pi, idx in enumerate(parts):
        s = np.zeros(r.size)
        for q in idx:
            n, m = nms[q]
            am = abs(m)
            j = (n - am) // 2
            P = model_1d('jacobi', 2 * r * r - 1, j, 0.0, float(am))[j]
            rm = (np.float32(r) ** am).astype(np.float64) if defect == 'r_f32' else r ** am
            H = rm * (np.sin(am * t) if m < 0 else np.cos(am * t))
            s += coefs[q] * float(zernike_norm(n, m)) * P * H
        acc = acc + s
        if defect == 'partial_f32' and pi < len(parts) - 1:
            acc = acc.astype(np.float32).astype(np.float64)
    return acc.astype(np.float32)


def model_sweep(values, count, sm_count, defect=None):
    """an output of `count` samples as a kernel that 'drop_sweep' ends after one grid-stride sweep would leave it
    (the rest stays as prefilled, NaN)"""
    out = np.array(values[:count], np.float64)
    if defect == 'drop_sweep':
        out[grid_for(count, sm_count) * THREADS:] = np.nan
    return out

