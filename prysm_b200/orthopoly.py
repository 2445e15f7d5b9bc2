"""The one-variable orthogonal families and the XY / Chebyshev two-variable sums on the device (reference
prysm/polynomials/cheby.py, legendre.py, hermite.py, laguerre.py, dickson.py, xy.py).

Every 1-D family is the three-term recurrence P_k = (A_k x + B_k) P_{k-1} - C_k P_{k-2}; each `*_seq` and
`*_der_seq` call is one launch of one kernel (pb_poly_seq) that runs the recurrence once per sample in fp64 registers
and writes only the requested planes.  Derivatives follow the reference's route: the differentiated recurrence for
Chebyshev, Legendre and Dickson, n P_{n-1} (He) / 2n P_{n-1} (H) for Hermite and -L_{n-1}^(alpha+1) for Laguerre.
Inputs are float32 or float64 and the outputs have the input's dtype.  Orders are limited to 0 <= n <= 120.

Unlike the reference, whose sequences assume ascending ns, plane i is the order ns[i] in any order, repeats included;
an empty ns gives an empty (0, *x.shape) array without a launch.

The XY monomials and the sums (xy_sum, xy_sum_der_xy, cheby1_2d_sum, cheby1_2d_sum_der_xy) are one launch each, the
sums in one pass with no basis stored.  With cartesian_grid the XY functions read x[0, :] and y[:, 0] of 2-D inputs
and return (ny, nx) planes, as the reference does (prysm/coordinates.py optimize_xy_separable).
"""
import math

import numpy as np
import torch

from . import _ops
from ._capi import (POLY_CHEBY1, POLY_CHEBY2, POLY_CHEBY3, POLY_CHEBY4, POLY_LEGENDRE, POLY_HERMITE_HE, POLY_HERMITE_H,
                    POLY_LAGUERRE, POLY_DICKSON1, POLY_DICKSON2, POLY_VALUE, POLY_DER, TSUM_MONOMIAL, TSUM_CHEBY1)


def _real(x):
    x = _ops.asdevice(x)
    if x.dtype not in (torch.float32, torch.float64):
        x = x.to(torch.float64)
    return x


def _orders(ns):
    return [int(n) for n in ns]


def _seq(family, kind, ns, x, alpha=0.0):
    return _ops.poly_seq(family, kind, _orders(ns), _real(x), alpha)


def _dense(coefs):
    if isinstance(coefs, torch.Tensor):
        coefs = coefs.detach().cpu().numpy()
    return [float(c) for c in np.asarray(coefs, dtype=np.float64).ravel()]


# ------------------------------------------------------------------------------------------
# Chebyshev (first to fourth kind), Legendre, Hermite, Laguerre, Dickson
# ------------------------------------------------------------------------------------------

def cheby1_seq(ns, x):
    """Chebyshev polynomials of the first kind of orders ns, shape (len(ns), *x.shape)."""
    return _seq(POLY_CHEBY1, POLY_VALUE, ns, x)


def cheby1(n, x):
    return cheby1_seq([n], x)[0]


def cheby1_der_seq(ns, x):
    """d/dx of the Chebyshev polynomials of the first kind of orders ns."""
    return _seq(POLY_CHEBY1, POLY_DER, ns, x)


def cheby1_der(n, x):
    return cheby1_der_seq([n], x)[0]


def cheby2_seq(ns, x):
    """Chebyshev polynomials of the second kind of orders ns."""
    return _seq(POLY_CHEBY2, POLY_VALUE, ns, x)


def cheby2(n, x):
    return cheby2_seq([n], x)[0]


def cheby2_der_seq(ns, x):
    return _seq(POLY_CHEBY2, POLY_DER, ns, x)


def cheby2_der(n, x):
    return cheby2_der_seq([n], x)[0]


def cheby3_seq(ns, x):
    """Chebyshev polynomials of the third kind of orders ns."""
    return _seq(POLY_CHEBY3, POLY_VALUE, ns, x)


def cheby3(n, x):
    return cheby3_seq([n], x)[0]


def cheby3_der_seq(ns, x):
    return _seq(POLY_CHEBY3, POLY_DER, ns, x)


def cheby3_der(n, x):
    return cheby3_der_seq([n], x)[0]


def cheby4_seq(ns, x):
    """Chebyshev polynomials of the fourth kind of orders ns."""
    return _seq(POLY_CHEBY4, POLY_VALUE, ns, x)


def cheby4(n, x):
    return cheby4_seq([n], x)[0]


def cheby4_der_seq(ns, x):
    return _seq(POLY_CHEBY4, POLY_DER, ns, x)


def cheby4_der(n, x):
    return cheby4_der_seq([n], x)[0]


def legendre_seq(ns, x):
    """Legendre polynomials of orders ns, shape (len(ns), *x.shape)."""
    return _seq(POLY_LEGENDRE, POLY_VALUE, ns, x)


def legendre(n, x):
    return legendre_seq([n], x)[0]


def legendre_der_seq(ns, x):
    return _seq(POLY_LEGENDRE, POLY_DER, ns, x)


def legendre_der(n, x):
    return legendre_der_seq([n], x)[0]


def hermite_He_seq(ns, x):
    """Probabilist's Hermite polynomials He_n of orders ns."""
    return _seq(POLY_HERMITE_HE, POLY_VALUE, ns, x)


def hermite_He(n, x):
    return hermite_He_seq([n], x)[0]


def hermite_He_der_seq(ns, x):
    """d/dx He_n = n He_{n-1}."""
    return _seq(POLY_HERMITE_HE, POLY_DER, ns, x)


def hermite_He_der(n, x):
    return hermite_He_der_seq([n], x)[0]


def hermite_H_seq(ns, x):
    """Physicist's Hermite polynomials H_n of orders ns."""
    return _seq(POLY_HERMITE_H, POLY_VALUE, ns, x)


def hermite_H(n, x):
    return hermite_H_seq([n], x)[0]


def hermite_H_der_seq(ns, x):
    """d/dx H_n = 2n H_{n-1}."""
    return _seq(POLY_HERMITE_H, POLY_DER, ns, x)


def hermite_H_der(n, x):
    return hermite_H_der_seq([n], x)[0]


def laguerre_seq(ns, alpha, x):
    """Generalized Laguerre polynomials L_n^(alpha) of orders ns."""
    return _seq(POLY_LAGUERRE, POLY_VALUE, ns, x, alpha)


def laguerre(n, alpha, x):
    return laguerre_seq([n], alpha, x)[0]


def laguerre_der_seq(ns, alpha, x):
    """d/dx L_n^(alpha) = -L_{n-1}^(alpha+1)."""
    return _seq(POLY_LAGUERRE, POLY_DER, ns, x, alpha)


def laguerre_der(n, alpha, x):
    return laguerre_der_seq([n], alpha, x)[0]


def dickson1_seq(ns, alpha, x):
    """Dickson polynomials of the first kind D_n(x, alpha) of orders ns (D_0 = 2)."""
    return _seq(POLY_DICKSON1, POLY_VALUE, ns, x, alpha)


def dickson1(n, alpha, x):
    return dickson1_seq([n], alpha, x)[0]


def dickson1_der_seq(ns, alpha, x):
    return _seq(POLY_DICKSON1, POLY_DER, ns, x, alpha)


def dickson1_der(n, alpha, x):
    return dickson1_der_seq([n], alpha, x)[0]


def dickson2_seq(ns, alpha, x):
    """Dickson polynomials of the second kind E_n(x, alpha) of orders ns (E_0 = 1)."""
    return _seq(POLY_DICKSON2, POLY_VALUE, ns, x, alpha)


def dickson2(n, alpha, x):
    return dickson2_seq([n], alpha, x)[0]


def dickson2_der_seq(ns, alpha, x):
    return _seq(POLY_DICKSON2, POLY_DER, ns, x, alpha)


def dickson2_der(n, alpha, x):
    return dickson2_der_seq([n], alpha, x)[0]


# ------------------------------------------------------------------------------------------
# two-variable sums and XY monomials
# ------------------------------------------------------------------------------------------

def _pairs(coefs, mns):
    """(coefficients, ms, ns) paired by zip, as the reference pairs them."""
    cs, ms, ns = [], [], []
    for c, (m, n) in zip(_dense(coefs), mns):
        cs.append(c); ms.append(int(m)); ns.append(int(n))
    return cs, ms, ns


def _elementwise(x, y):
    x, y = _real(x), _real(y)
    dt = torch.promote_types(x.dtype, y.dtype)
    x, y = torch.broadcast_tensors(x.to(dt), y.to(dt))
    return x.contiguous(), y.contiguous(), tuple(x.shape)


def _separable(x, y):
    """x[0, :] and y[:, 0] of 2-D inputs (1-D ones as a row and a column), and the (ny, nx) shape they span."""
    x, y = _real(x), _real(y)
    dt = torch.promote_types(x.dtype, y.dtype)
    xs = x[0, :] if x.ndim == 2 else x.reshape(-1)
    ys = y[:, 0] if y.ndim == 2 else y.reshape(-1)
    return xs.to(dt).contiguous(), ys.to(dt).contiguous(), (ys.numel(), xs.numel())


def cheby1_2d_sum(coefs, mns, x, y):
    """sum c T_m(x) T_n(y) over the zip of coefs and (m, n) pairs, in one pass."""
    cs, ms, ns = _pairs(coefs, tuple(mns))
    x, y, shape = _elementwise(x, y)
    if not ms:
        return torch.zeros(shape, dtype=x.dtype, device=x.device)
    return _ops.tensor_sum(TSUM_CHEBY1, cs, ms, ns, x, y, shape, False, False)[0]


def cheby1_2d_sum_der_xy(coefs, mns, x, y, x_norm=1.0, y_norm=1.0):
    """(z, dz/dx / x_norm, dz/dy / y_norm) of a Chebyshev-T tensor sum, in one pass."""
    cs, ms, ns = _pairs(coefs, tuple(mns))
    x, y, shape = _elementwise(x, y)
    if not ms:
        z = torch.zeros(shape, dtype=x.dtype, device=x.device)
        return z, z, torch.zeros_like(z)
    return _ops.tensor_sum(TSUM_CHEBY1, cs, ms, ns, x, y, shape, False, True, x_norm, y_norm)


def xy_j_to_mn(j):
    """Mono-index j -> (m, n) powers of x and y; j = 1 is piston (prysm/polynomials/xy.py:11-27)."""
    if j < 1:
        raise ValueError('j must be >= 1')
    if j == 1:
        return 0, 0
    total_order = int(math.ceil((math.sqrt(8 * j + 1) - 3) / 2))
    first_j = total_order * (total_order + 1) // 2 + 1
    y_order = j - first_j
    return total_order - y_order, y_order


def _xy(mns, x, y, separable, kind):
    mns = [(int(m), int(n)) for m, n in mns]
    if separable:
        xs, ys, shape = _separable(x, y)
    else:
        xs, ys, shape = _elementwise(x, y)
    return _ops.xy_seq([m for m, _ in mns], [n for _, n in mns], [kind] * len(mns), xs, ys, shape, separable)


def _seq_separable(x, cartesian_grid):
    return bool(cartesian_grid) and _real(x).ndim > 1


def xy_seq(mns, x, y, cartesian_grid=True):
    """x^m y^n for the (m, n) pairs, shape (len(mns), *grid)."""
    return _xy(mns, x, y, _seq_separable(x, cartesian_grid), 0)


def xy(m, n, x, y, cartesian_grid=True):
    return _xy([(m, n)], x, y, bool(cartesian_grid), 0)[0]


def xy_der_x_seq(mns, x, y, cartesian_grid=True):
    """d/dx x^m y^n = m x^(m-1) y^n (zero for m = 0)."""
    return _xy(mns, x, y, _seq_separable(x, cartesian_grid), 1)


def xy_der_x(m, n, x, y, cartesian_grid=True):
    return _xy([(m, n)], x, y, bool(cartesian_grid), 1)[0]


def xy_der_y_seq(mns, x, y, cartesian_grid=True):
    """d/dy x^m y^n = n x^m y^(n-1) (zero for n = 0)."""
    return _xy(mns, x, y, _seq_separable(x, cartesian_grid), 2)


def xy_der_y(m, n, x, y, cartesian_grid=True):
    return _xy([(m, n)], x, y, bool(cartesian_grid), 2)[0]


def xy_der_xy_seq(mns, x, y, cartesian_grid=True):
    """d^2/dxdy x^m y^n = m n x^(m-1) y^(n-1)."""
    return _xy(mns, x, y, _seq_separable(x, cartesian_grid), 3)


def xy_der_xy(m, n, x, y, cartesian_grid=True):
    return _xy([(m, n)], x, y, bool(cartesian_grid), 3)[0]


def _xy_sum(coefs, mns, x, y, cartesian_grid, want_der):
    cs, ms, ns = _pairs(coefs, tuple(mns))
    sep = _seq_separable(x, cartesian_grid)
    xs, ys, shape = _separable(x, y) if sep else _elementwise(x, y)
    if not ms:
        z = torch.zeros(shape, dtype=xs.dtype, device=xs.device)
        return (z, z, torch.zeros_like(z)) if want_der else (z, None, None)
    return _ops.tensor_sum(TSUM_MONOMIAL, cs, ms, ns, xs, ys, shape, sep, want_der)


def xy_sum(coefs, mns, x, y, cartesian_grid=True):
    """sum c x^m y^n in one pass, no basis stored."""
    return _xy_sum(coefs, mns, x, y, cartesian_grid, False)[0]


def xy_sum_der_xy(coefs, mns, x, y, cartesian_grid=True):
    """(z, dz/dx, dz/dy) of an XY-monomial sum in one pass."""
    return _xy_sum(coefs, mns, x, y, cartesian_grid, True)


__all__ = ['cheby1', 'cheby1_seq', 'cheby1_der', 'cheby1_der_seq', 'cheby1_2d_sum', 'cheby1_2d_sum_der_xy',
           'cheby2', 'cheby2_seq', 'cheby2_der', 'cheby2_der_seq', 'cheby3', 'cheby3_seq', 'cheby3_der',
           'cheby3_der_seq', 'cheby4', 'cheby4_seq', 'cheby4_der', 'cheby4_der_seq',
           'dickson1', 'dickson1_seq', 'dickson1_der', 'dickson1_der_seq', 'dickson2', 'dickson2_seq', 'dickson2_der',
           'dickson2_der_seq', 'hermite_He', 'hermite_He_seq', 'hermite_He_der', 'hermite_He_der_seq', 'hermite_H',
           'hermite_H_seq', 'hermite_H_der', 'hermite_H_der_seq', 'laguerre', 'laguerre_seq', 'laguerre_der',
           'laguerre_der_seq', 'legendre', 'legendre_seq', 'legendre_der', 'legendre_der_seq',
           'xy_j_to_mn', 'xy', 'xy_seq', 'xy_der_x', 'xy_der_x_seq', 'xy_der_y', 'xy_der_y_seq', 'xy_der_xy',
           'xy_der_xy_seq', 'xy_sum', 'xy_sum_der_xy']
