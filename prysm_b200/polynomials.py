"""The polynomial-module functions around the propagation path: the weighted mode sum used as the incoherent
polychromatic sum and as the modal OPD synthesis, its adjoint (reference prysm/polynomials/fitting.py:7-57), and
the Jacobi / Zernike recurrences that build the modes, their derivatives and their sums (prysm/polynomials/
jacobi.py, zernike.py) evaluated on the device.  The other one-variable families and the XY / Chebyshev sums come
from .orthopoly, the Forbes polynomials from .qpoly, re-exported here as the reference's prysm.polynomials does."""
import math
import warnings

import numpy as np
import torch

from . import _ops
from ._capi import POLY_JACOBI, POLY_VALUE, POLY_DER, POLY_VALUE_DER, CLENSHAW_JMAX


def sum_of_2d_modes(modes, weights):
    """tensordot(modes(k, m, n), weights(k)) over the leading axis as one streaming kernel."""
    if isinstance(modes, (list, tuple)):
        warnings.warn('sum_of_2d_modes: modes is a list or tuple: for optimal performance, pre convert to array of shape (k, m, n)')
        modes = torch.stack([_ops.asdevice(m) for m in modes])
    modes = _ops.asdevice(modes)
    if isinstance(weights, torch.Tensor):
        weights = weights.detach().cpu().numpy()
    return _ops.weighted_sum(modes, np.asarray(weights, dtype=np.float64))


def sum_of_2d_modes_adjoint(modes, databar):
    """tensordot(modes(k, m, n), databar(m, n)) over the trailing axes: k reductions in one launch; the (k,)
    gradient comes back as a host array like the weights it pairs with (prysm/polynomials/fitting.py:40-57)."""
    if isinstance(modes, (list, tuple)):
        modes = torch.stack([_ops.asdevice(m) for m in modes])
    modes = _ops.asdevice(modes)
    if modes.dtype not in (torch.float32, torch.float64):
        modes = modes.to(torch.float64)
    return _ops.mode_projection(modes, _ops.asdevice(databar))


def lstsq(modes, data):
    """Least-squares fit of modes to data, ignoring the pixels where data is not finite (prysm/polynomials/fitting.py:
    103-126).  One launch (pb_masked_gram) reduces [A d]^T [A d] over the finite pixels in fp64 with no compaction;
    the (k, k) system is solved on the host with numpy.linalg.lstsq, whose minimum-norm answer equals pinv(A) d, so a
    rank-deficient basis gets the reference's answer.  The normal equations square the condition number of A.  modes:
    a (k, ...) array or a sequence of k arrays shaped like data, 1 <= k <= 64.  Returns the (k,) fp64 host array."""
    data = _ops.asdevice(data)
    if data.dtype not in (torch.float32, torch.float64):
        data = data.to(torch.float64)
    if isinstance(modes, torch.Tensor) or hasattr(modes, 'shape'):
        modes = _ops.asdevice(modes)
        mlist = [modes[k].reshape(-1) for k in range(modes.shape[0])]
    else:
        mlist = [None if m is None else _ops.asdevice(m).reshape(-1) for m in modes]
    return solve_gram(_ops.masked_gram(mlist, data.reshape(-1)), len(mlist))


def solve_gram(packed, k):
    """numpy.linalg.lstsq of the normal equations held in the packed triangle pb_masked_gram writes"""
    full = np.zeros((k + 1, k + 1))
    full[np.triu_indices(k + 1)] = packed
    G = np.triu(full[:k, :k]) + np.triu(full[:k, :k], 1).T
    return np.linalg.lstsq(G, full[:k, k], rcond=None)[0]


# ------------------------------------------------------------------------------------------
# Jacobi / Zernike by recurrence
# ------------------------------------------------------------------------------------------

def _real(x):
    x = _ops.asdevice(x)
    if x.dtype not in (torch.float32, torch.float64):
        x = x.to(torch.float64)
    return x


def jacobi_seq(ns, alpha, beta, x):
    """P_n^(alpha,beta)(x) for the sorted orders ns, shape (len(ns), *x.shape): the three-term recurrence runs once
    in registers and only the requested orders are stored (prysm/polynomials/jacobi.py:147-175).  Plane i is ns[i] in
    any order, repeats included."""
    return _ops.poly_seq(POLY_JACOBI, POLY_VALUE, [int(n) for n in ns], _real(x), alpha, beta)


def jacobi(n, alpha, beta, x):
    """prysm/polynomials/jacobi.py:42-79."""
    return jacobi_seq([int(n)], alpha, beta, x)[0]


def jacobi_der_seq(ns, alpha, beta, x):
    """dP_n/dx for the orders ns as 0.5 (n + alpha + beta + 1) P_{n-1}^(alpha+1, beta+1), the reference's route
    (prysm/polynomials/jacobi.py:237-276), in one launch; plane i is ns[i] in any order."""
    return _ops.poly_seq(POLY_JACOBI, POLY_DER, [int(n) for n in ns], _real(x), alpha, beta)


def jacobi_der(n, alpha, beta, x):
    """prysm/polynomials/jacobi.py:204-234."""
    return jacobi_der_seq([n], alpha, beta, x)[0]


def jacobi_seq_with_der(ns, alpha, beta, x):
    """(P_n, dP_n/dx) for the orders ns by the differentiated recurrence, both from one launch
    (prysm/polynomials/jacobi.py:178-201)."""
    return _ops.poly_seq(POLY_JACOBI, POLY_VALUE_DER, [int(n) for n in ns], _real(x), alpha, beta)


def jacobi_with_der(n, alpha, beta, x):
    """prysm/polynomials/jacobi.py:88-134."""
    P, dP = jacobi_seq_with_der([n], alpha, beta, x)
    return P[0], dP[0]


def jacobi_sum_clenshaw(s, alpha, beta, x, alphas=None):
    """sum_n s[n] P_n^(alpha,beta)(x) by Clenshaw's backward recurrence, per sample in registers, in one launch
    (prysm/polynomials/jacobi.py:279-316).  With `alphas`, a (max(len(s), 2), *x.shape) device tensor, the whole alpha
    table is written into it; alphas[0] is returned either way."""
    s = _dense_coefs(s)
    x = _real(x)
    if alphas is None:
        return _ops.jacobi_clenshaw(s, alpha, beta, x, 0, False)
    return _ops.jacobi_clenshaw(s, alpha, beta, x, 0, True, out=alphas.reshape((1,) + tuple(alphas.shape)))[0, 0]


def jacobi_sum_clenshaw_der(s, alpha, beta, x, j=1, alphas=None):
    """The reference's whole Clenshaw table (j + 1, max(len(s), 2), *x.shape) for the sum and its first j derivatives
    (prysm/polynomials/jacobi.py:319-373): alphas[jj, 0] is the jj-th derivative of the sum.  One launch; j <= 8.
    With `alphas`, a device tensor of that shape, the table is written into it."""
    j = int(j)
    if not 0 <= j <= CLENSHAW_JMAX:
        raise ValueError(f'derivative order j = {j} is outside 0..{CLENSHAW_JMAX}')
    return _ops.jacobi_clenshaw(_dense_coefs(s), alpha, beta, _real(x), j, True, out=alphas)


def _radial_pairs(coefs, ns):
    """(orders, coefficients) as the reference pairs them, enumerate(coefs) over ns: extra trailing orders are unused,
    an extra nonzero coefficient raises IndexError (prysm/polynomials/jacobi.py:385-388)."""
    ns = [int(n) for n in ns]
    on, oc = [], []
    for i, c in enumerate(_dense_coefs(coefs)):
        if c == 0.0:
            continue
        if i >= len(ns):
            raise IndexError(f'coefficient {i} has no order: only {len(ns)} orders')
        on.append(ns[i]); oc.append(c)
    return on, oc


def jacobi_radial_sum(coefs, ns, alpha, beta, x, y, normalization_radius):
    """sum_i coefs[i] P_{ns[i]}^(alpha,beta)(2 (x^2 + y^2) / R^2 - 1) in one pass (prysm/polynomials/jacobi.py:376-389)."""
    ns = tuple(ns)
    x = _real(x)
    if not ns:
        return torch.zeros_like(x)
    on, oc = _radial_pairs(coefs, ns)
    return _ops.jacobi_radial_sum(oc, on, alpha, beta, x, _real(y), float(normalization_radius), False)[0]


def jacobi_radial_sum_der_xy(coefs, ns, alpha, beta, x, y, normalization_radius):
    """(z, dz/dx, dz/dy) of a radial Jacobi sum in one pass, dz/du by the differentiated recurrence
    (prysm/polynomials/jacobi.py:392-413)."""
    ns = tuple(ns)
    x = _real(x)
    if not ns:
        z = torch.zeros_like(x)
        return z, z, torch.zeros_like(x)
    on, oc = _radial_pairs(coefs, ns)
    return _ops.jacobi_radial_sum(oc, on, alpha, beta, x, _real(y), float(normalization_radius), True)


def _dense_coefs(c):
    if isinstance(c, torch.Tensor):
        c = c.detach().cpu().numpy()
    return [float(v) for v in np.asarray(c, dtype=np.float64).ravel()]


def zernike_norm(n, m):
    """sqrt(2(n+1)/(1+delta_m0)) (prysm/polynomials/zernike.py:25-27)."""
    return math.sqrt((2 * (n + 1)) / (1 + (1 if m == 0 else 0)))


def zernike_nm_seq(nms, r, t, norm=True):
    """Zernike modes for the (n, m) pairs, shape (k, *r.shape).  One kernel evaluates every mode per sample, the
    Jacobi recurrences shared per |m| like the reference's de-duplication (prysm/polynomials/zernike.py:74-166)."""
    return _ops.zernike_seq([(int(n), int(m)) for n, m in nms], _real(r), _real(t), norm, polar=True)


def zernike_nm(n, m, r, t, norm=True):
    """prysm/polynomials/zernike.py:35-71."""
    return zernike_nm_seq([(n, m)], r, t, norm)[0]


def zernike_sum(coefs, nms, x, y, norm=True):
    """sum_k coefs[k] * Z_k on Cartesian unit-disk coordinates without materialising the basis: the OPD goes from
    coefficients to one array in one pass (prysm/polynomials/zernike.py:169-181)."""
    nms = [(int(n), int(m)) for n, m in nms]
    x = _real(x)
    if not nms:
        return torch.zeros_like(x)
    if isinstance(coefs, torch.Tensor):
        coefs = coefs.detach().cpu().numpy()
    return _ops.zernike_sum(np.asarray(coefs, dtype=np.float64), nms, x, _real(y), norm, polar=False)


def zernike_nm_der_seq(nms, r, t, norm=True):
    """(len(nms), 2, *r.shape): dZ/dr and dZ/dt of each mode, every |m| group's Jacobi recurrence run once with its
    derivative beside it (prysm/polynomials/zernike.py:273-380).  Pairs with |m| > n or odd n - |m| raise ValueError."""
    return _ops.zernike_der([(int(n), int(m)) for n, m in nms], _real(r), _real(t), norm, cartesian=False)


def zernike_nm_der(n, m, r, t, norm=True):
    """(dZ/dr, dZ/dt) (prysm/polynomials/zernike.py:184-270)."""
    out = zernike_nm_der_seq([(n, m)], r, t, norm)
    return out[0, 0], out[0, 1]


def zernike_nm_der_xy_seq(nms, x, y, norm=True):
    """(len(nms), 2, *x.shape): dZ/dx and dZ/dy through Re / Im (x + iy)^|m|, finite at the origin
    (prysm/polynomials/zernike.py:448-531)."""
    return _ops.zernike_der([(int(n), int(m)) for n, m in nms], _real(x), _real(y), norm, cartesian=True)


def zernike_nm_der_xy(n, m, x, y, norm=True):
    """(dZ/dx, dZ/dy) (prysm/polynomials/zernike.py:383-445)."""
    out = zernike_nm_der_xy_seq([(n, m)], x, y, norm)
    return out[0, 0], out[0, 1]


def zernike_sum_der_xy(coefs, nms, x, y, norm=True):
    """(W, dW/dx, dW/dy) of W = sum coefs[i] Z_i(x, y) from the coefficients in one pass, no basis stored: a forward
    recurrence per |m| with the weights applied as each order is made (prysm/polynomials/zernike.py:534-630).
    Duplicate (n, m) pairs add; zero coefficients are skipped."""
    nms = [(int(n), int(m)) for n, m in nms]
    x = _real(x)
    y = _real(y)
    if not nms:
        z = torch.zeros_like(x)
        return z, torch.zeros_like(x), torch.zeros_like(x)
    c = _dense_coefs(coefs)[:len(nms)]
    out = _ops.zernike_sum_der_xy(c, nms[:len(c)], x, y, norm)
    return out[0], out[1], out[2]


def nm_to_fringe(n, m):
    """(n, m) -> Fringe index (prysm/polynomials/zernike.py:633-638)."""
    term1 = (1 + (n + abs(m)) / 2) ** 2
    term2 = 2 * abs(m)
    term3 = (1 + (m > 0) - (m < 0)) / 2
    return int(term1 - term2 - term3) + 1


def nm_to_ansi_j(n, m):
    """(n, m) -> ANSI single index (prysm/polynomials/zernike.py:641-643)."""
    return int((n * (n + 2) + m) / 2)


def ansi_j_to_nm(idx):
    """ANSI single index -> (n, m) (prysm/polynomials/zernike.py:646-650)."""
    n = int(math.ceil((-3 + math.sqrt(9 + 8 * idx)) / 2))
    return n, 2 * idx - n * (n + 2)


def noll_to_nm(idx):
    """Noll index -> (n, m) (prysm/polynomials/zernike.py:653-681; host integer bookkeeping)."""
    n = int(math.ceil((-1 + math.sqrt(1 + 8 * idx)) / 2) - 1)
    if n == 0:
        return 0, 0
    res = idx - int((n + 1) * (n + 2) / 2) - 1
    ms = [1, 1] if n % 2 else [0]
    for _ in range(n // 2):
        ms.append(ms[-1] + 2)
        ms.append(ms[-1])
    return n, ms[res] * (-1 if idx % 2 else 1)


def fringe_to_nm(idx):
    """Fringe index -> (n, m) (prysm/polynomials/zernike.py:684-690)."""
    m_n = 2 * (math.ceil(math.sqrt(idx)) - 1)
    g_s = (m_n // 2) ** 2 + 1
    n = m_n // 2 + (idx - g_s) // 2
    m = (m_n - n) * (1 - ((idx - g_s) % 2) * 2)
    return int(n), int(m)


# Forbes Q polynomials (prysm/polynomials/__init__.py re-exports the same names from its qpoly module)
from .qpoly import (  # noqa: E402,F401
    Qbfs,
    Qbfs_seq,
    Qbfs_der,
    Qbfs_der_seq,
    Qcon,
    Qcon_seq,
    Qcon_der,
    Qcon_der_seq,
    Q2d,
    Q2d_seq,
    Q2d_der,
    Q2d_der_seq,
    Q2d_der_xy,
    Q2d_der_xy_seq,
)

# the other one-variable families, XY monomials and the two-variable sums (prysm/polynomials/__init__.py)
from .orthopoly import *  # noqa: E402,F401,F403
