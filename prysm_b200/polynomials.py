"""The polynomial-module functions around the propagation path: the weighted mode sum used as the incoherent
polychromatic sum and as the modal OPD synthesis, its adjoint (reference prysm/polynomials/fitting.py:7-57), and
the Jacobi / Zernike recurrences that build the modes (prysm/polynomials/jacobi.py:13-175, zernike.py:25-181,
633-690) evaluated on the device."""
import math
import warnings

import numpy as np
import torch

from . import _ops


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
    in registers and only the requested orders are stored (prysm/polynomials/jacobi.py:147-175)."""
    return _ops.jacobi_seq(list(ns), alpha, beta, _real(x))


def jacobi(n, alpha, beta, x):
    """prysm/polynomials/jacobi.py:42-79."""
    return _ops.jacobi_seq([int(n)], alpha, beta, _real(x))[0]


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
