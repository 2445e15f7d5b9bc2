"""Forbes polynomials on the device (reference prysm/polynomials/qpoly.py): Q-bfs, the slope-orthogonal asphere
(oe-18-19-19700); Q-con, the sag-orthogonal asphere (oe-18-13-13851); and 2D-Q, the freeform basis (oe-20-3-2483).

Every `*_seq` call and every `compute_z*` call is one kernel launch (pb_qpoly_seq / pb_qpoly_sum): each sample runs
the needed recurrences once in fp64 registers and writes only the requested planes, or the weighted sums with the
basis never stored.  Inputs are float32 or float64 and the outputs have the input's dtype.  Orders are limited to
n <= 64 and |m| <= 64 (QPOLY_NMAX).

Unlike the reference, the 1-D sequences take their orders in any order, and return plane i for ns[i] (the reference
assumes ascending ns).  The scalar table functions and Q2d_nm_c_to_a_b are host code; the tables come from the same
C++ the kernels are planned with.
"""
from collections import defaultdict
from functools import lru_cache
import math

import numpy as np
import torch

from . import _ops
from ._capi import QPOLY_BFS, QPOLY_CON, QPOLY_2D, QPOLY_VALUE, QPOLY_DER, QPOLY_DER_XY, QPOLY_NMAX


def _real(x):
    x = _ops.asdevice(x)
    if x.dtype not in (torch.float32, torch.float64):
        x = x.to(torch.float64)
    return x


def _orders(ns):
    return [int(n) for n in ns]


def _nms(nms):
    nms = [(int(n), int(m)) for n, m in nms]
    return [n for n, _ in nms], [m for _, m in nms]


# ------------------------------------------------------------------------------------------
# scalar tables (host)
# ------------------------------------------------------------------------------------------

@lru_cache(None)
def _table(family, m):
    return _ops.qpoly_tables(family, m, QPOLY_NMAX)


def _row(family, m, n):
    if not 0 <= n <= QPOLY_NMAX:
        raise ValueError(f'order {n} is outside 0..{QPOLY_NMAX}')
    if family == QPOLY_2D and not 1 <= m <= QPOLY_NMAX:
        raise ValueError(f'azimuthal order {m} is outside 1..{QPOLY_NMAX}')
    return _table(family, m if family == QPOLY_2D else 0)[n]


def g_qbfs(n_minus_1):
    """g(m-1) of oe-18-19-19700 eq. (A.15)."""
    return float(_row(QPOLY_BFS, 0, int(n_minus_1))[1])


def h_qbfs(n_minus_2):
    """h(m-2) of oe-18-19-19700 eq. (A.14)."""
    return float(_row(QPOLY_BFS, 0, int(n_minus_2))[2])


def f_qbfs(n):
    """f(m) of oe-18-19-19700 eq. (A.16)."""
    return float(_row(QPOLY_BFS, 0, int(n))[0])


def abc_q2d(n, m):
    """A, B, C of oe-20-3-2483 eq. (A.3); ZeroDivisionError where their denominator vanishes, as in the reference."""
    A, B, C = (float(v) for v in _row(QPOLY_2D, int(m), int(n))[:3])
    if math.isnan(A):
        raise ZeroDivisionError(f'abc_q2d({n}, {m}): the denominator of A.3 is zero')
    return A, B, C


def G_q2d(n, m):
    """G of oe-20-3-2483 eq. (A.15)."""
    return float(_row(QPOLY_2D, int(m), int(n))[3])


def F_q2d(n, m):
    """F of oe-20-3-2483 eq. (A.13)."""
    return float(_row(QPOLY_2D, int(m), int(n))[4])


def g_q2d(n, m):
    """g of oe-20-3-2483 eq. (A.18a) (n is the radial order less one)."""
    return float(_row(QPOLY_2D, int(m), int(n))[5])


def f_q2d(n, m):
    """f of oe-20-3-2483 eq. (A.18b)."""
    return float(_row(QPOLY_2D, int(m), int(n))[6])


# ------------------------------------------------------------------------------------------
# bases
# ------------------------------------------------------------------------------------------

def Qbfs_seq(ns, x):
    """Q-bfs polynomials of orders ns at x, shape (len(ns), *x.shape)."""
    return _ops.qpoly_seq(QPOLY_BFS, QPOLY_VALUE, _orders(ns), None, _real(x))


def Qbfs(n, x):
    return Qbfs_seq([n], x)[0]


def Qbfs_der_seq(ns, x):
    """d/dx of the Q-bfs polynomials of orders ns, shape (len(ns), *x.shape)."""
    return _ops.qpoly_seq(QPOLY_BFS, QPOLY_DER, _orders(ns), None, _real(x))


def Qbfs_der(n, x):
    return Qbfs_der_seq([n], x)[0]


def Qcon_seq(ns, x):
    """Q-con polynomials x^4 P_n^(0,4)(2x^2 - 1) of orders ns, shape (len(ns), *x.shape)."""
    return _ops.qpoly_seq(QPOLY_CON, QPOLY_VALUE, _orders(ns), None, _real(x))


def Qcon(n, x):
    return Qcon_seq([n], x)[0]


def Qcon_der_seq(ns, x):
    """d/dx of the Q-con polynomials of orders ns, shape (len(ns), *x.shape)."""
    return _ops.qpoly_seq(QPOLY_CON, QPOLY_DER, _orders(ns), None, _real(x))


def Qcon_der(n, x):
    return Qcon_der_seq([n], x)[0]


def Q2d_seq(nms, r, t):
    """2D-Q polynomials for the (n, m) pairs (m < 0: sine terms, m = 0: Q-bfs), shape (len(nms), *r.shape).  One
    recurrence per |m| up to the largest n requested for it; repeated pairs each get their plane."""
    ns, ms = _nms(nms)
    return _ops.qpoly_seq(QPOLY_2D, QPOLY_VALUE, ns, ms, _real(r), _real(t))


def Q2d(n, m, r, t):
    return Q2d_seq([(n, m)], r, t)[0]


def Q2d_der_seq(nms, r, t):
    """(d/dr, d/dt) of the 2D-Q polynomials, each (len(nms), *r.shape)."""
    ns, ms = _nms(nms)
    return _ops.qpoly_seq(QPOLY_2D, QPOLY_DER, ns, ms, _real(r), _real(t))


def Q2d_der(n, m, r, t):
    dr, dt = Q2d_der_seq([(n, m)], r, t)
    return dr[0], dt[0]


def Q2d_der_xy_seq(nms, x, y):
    """(d/dx, d/dy) of the 2D-Q polynomials, each (len(nms), *x.shape), through Re / Im (x + iy)^|m| so that the
    result is finite at the origin."""
    ns, ms = _nms(nms)
    return _ops.qpoly_seq(QPOLY_2D, QPOLY_DER_XY, ns, ms, _real(x), _real(y))


def Q2d_der_xy(n, m, x, y):
    dx, dy = Q2d_der_xy_seq([(n, m)], x, y)
    return dx[0], dy[0]


# ------------------------------------------------------------------------------------------
# sag and slope sums (usq is accepted for the reference's signature; the kernel squares u itself)
# ------------------------------------------------------------------------------------------

def _dense(coefs):
    if coefs is None:
        return []
    if isinstance(coefs, torch.Tensor):
        coefs = coefs.detach().cpu().numpy()
    return [float(c) for c in np.asarray(coefs, dtype=np.float64).ravel()]


def _radial(family, coefs, u, want_der):
    c = _dense(coefs)
    ns = list(range(len(c)))
    z, dr, _ = _ops.qpoly_sum(family, ns, None, c, _real(u), want_der=want_der)
    return z, dr


def compute_z_Qbfs(coefs, u, usq=None):
    """Sag u^2 (1 - u^2) sum_n c_n Q_n(u^2) of a Q-bfs surface, base sphere excluded (oe-18-19-19700 eq. 3.13)."""
    return _radial(QPOLY_BFS, coefs, u, False)[0]


def compute_z_zprime_Qbfs(coefs, u, usq=None):
    """(sag, d sag / du) of a Q-bfs surface (oe-18-19-19700 eqs. 3.13, 3.14)."""
    return _radial(QPOLY_BFS, coefs, u, True)


def compute_z_zprime_Qcon(coefs, u, usq=None):
    """(sag, d sag / du) of a Q-con surface u^4 sum_n c_n P_n^(0,4)(2u^2 - 1) (oe-18-13-13851 eq. 5.3)."""
    return _radial(QPOLY_CON, coefs, u, True)


def _q2d_terms(cm0, ams, bms):
    ns, ms, cs = [], [], []
    for n, c in enumerate(_dense(cm0)):
        ns.append(n); ms.append(0); cs.append(c)
    for i, (a, b) in enumerate(zip(ams, bms)):
        for sgn, co in ((1, a), (-1, b)):
            for n, c in enumerate(_dense(co)):
                ns.append(n); ms.append(sgn * (i + 1)); cs.append(c)
    return ns, ms, cs


def compute_z_Q2d(cm0, ams, bms, u, t):
    """Sag of a 2D-Q surface from its m = 0 coefficients cm0 and the cosine / sine coefficients ams[m-1], bms[m-1]
    (oe-20-3-2483 eq. 2.2), base sphere excluded, in one launch."""
    ns, ms, cs = _q2d_terms(cm0, ams, bms)
    return _ops.qpoly_sum(QPOLY_2D, ns, ms, cs, _real(u), _real(t))[0]


def compute_z_zprime_Q2d(cm0, ams, bms, u, t):
    """(sag, d sag / du, d sag / dt) of a 2D-Q surface in one launch."""
    ns, ms, cs = _q2d_terms(cm0, ams, bms)
    return _ops.qpoly_sum(QPOLY_2D, ns, ms, cs, _real(u), _real(t), want_der=True)


def Q2d_nm_c_to_a_b(nms, coefs):
    """(n, m) pairs and their coefficients -> (cms, ams, bms) for compute_z_zprime_Q2d: dense per-order lists with
    holes filled by 0 and trailing zeros trimmed; zero coefficients are skipped (a later repeat of a pair wins); ams /
    bms run m = 1..max m with an empty list for an order that has no terms."""
    cms, ac, bc = [], defaultdict(list), defaultdict(list)

    def put(lst, n, c):
        if len(lst) < n + 1:
            lst.extend([0] * (n + 1 - len(lst)))
        lst[n] = c

    for (n, m), c in zip(nms, coefs):
        if c == 0:
            continue
        put(cms if m == 0 else (ac[m] if m > 0 else bc[-m]), n, c)

    def trim(lst):
        while lst and lst[-1] == 0:
            lst.pop()
        return lst

    trim(cms)
    for d in (ac, bc):
        for k in list(d):
            if not trim(d[k]):
                del d[k]
    top = max(list(ac) + list(bc), default=0)
    return cms, [ac.get(m, []) for m in range(1, top + 1)], [bc.get(m, []) for m in range(1, top + 1)]


__all__ = ['Qbfs', 'Qbfs_seq', 'Qbfs_der', 'Qbfs_der_seq', 'Qcon', 'Qcon_seq', 'Qcon_der', 'Qcon_der_seq',
           'Q2d', 'Q2d_seq', 'Q2d_der', 'Q2d_der_seq', 'Q2d_der_xy', 'Q2d_der_xy_seq',
           'compute_z_Qbfs', 'compute_z_zprime_Qbfs', 'compute_z_zprime_Qcon', 'compute_z_Q2d', 'compute_z_zprime_Q2d',
           'Q2d_nm_c_to_a_b', 'g_qbfs', 'h_qbfs', 'f_qbfs', 'abc_q2d', 'G_q2d', 'F_q2d', 'g_q2d', 'f_q2d']
