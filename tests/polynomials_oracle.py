"""The orthogonal-polynomial, Zernike-derivative and polynomial-sum cases the engine is checked on
(prysm/polynomials), and the writer of tests/golden/polynomials*.npz.

    PYTHONDONTWRITEBYTECODE=1 python tests/polynomials_oracle.py   (needs the unmodified reference: PRYSM_REFERENCE or
                                                                    oracle/_ref)

The fixtures are the REFERENCE's own outputs at precision 64:
  - `line_<family>`: each 1-D family's *_seq and *_der_seq (and Jacobi's *_seq_with_der) at the orders NS on a line
    over its natural domain (Hermite [-6, 6], Laguerre [0, 20], the rest [-1, 1]);
  - `clen_*`: jacobi_sum_clenshaw and the whole jacobi_sum_clenshaw_der table, j = 1..3 and len(s) = 1;
  - on the qpoly grids (`odd`: 33 x 33 over [-1, 1]; `even`: 32 x 40 on fftrange / 16, both holding r = 0 and r = 1):
    the Zernike polar and Cartesian derivative sequences, zernike_sum_der_xy, the radial Jacobi sums, the XY monomial
    sequences and sums (separable and elementwise) and the Chebyshev-1 tensor sums;
  - `slope_*`: the slope map of a 36-coefficient Noll 2-37 pupil at 256^2;
  - `xypsf*`: an XY-polynomial pupil taken to focus by the reference's host pipeline.
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (ROOT, os.path.join(ROOT, 'oracle'), HERE):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import reference  # noqa: E402
from qpoly_oracle import grids  # noqa: E402  (the same two grids)

NS = [0, 1, 2, 3, 5, 8, 13, 21, 30, 34]      # ascending: the reference's 1-D sequences assume it
ALPHA, BETA = 0.5, 1.5                       # Jacobi; Laguerre takes ALPHA
DICKSON_ALPHA = 0.7
# family -> (domain, the extra positional parameters of its reference functions)
FAMILIES = {
    'cheby1': ((-1, 1), ()), 'cheby2': ((-1, 1), ()), 'cheby3': ((-1, 1), ()), 'cheby4': ((-1, 1), ()),
    'legendre': ((-1, 1), ()), 'hermite_He': ((-6, 6), ()), 'hermite_H': ((-6, 6), ()),
    'laguerre': ((0, 20), (ALPHA,)), 'dickson1': ((-1, 1), (DICKSON_ALPHA,)), 'dickson2': ((-1, 1), (-1.0,)),
    'jacobi': ((-1, 1), (ALPHA, BETA)),
}
LINE = 201
# m = 0, +-1, sine and cosine, |m| up to 12, n up to 20
ZNMS = [(0, 0), (1, 1), (1, -1), (2, 0), (2, 2), (2, -2), (3, 1), (3, -3), (4, 0), (5, -1), (6, 6), (8, -4), (12, 12),
        (13, -11), (20, 0), (20, 12), (16, -12), (7, 1)]
ZSUMS = {
    'mixed': ([0.3, -0.2, 0.1, 0.05, 0.0, -0.07, 0.02], [(2, 0), (1, 1), (3, -1), (4, 0), (6, 2), (5, 5), (12, -12)]),
    'dups': ([0.2, 0.1, -0.3, 0.3, 0.05], [(2, 2), (2, 2), (3, -1), (3, -1), (0, 0)]),      # duplicates, one cancelling
    'trailing': ([0.1, -0.05, 0.0, 0.0], [(4, 0), (3, 3), (8, 0), (7, -1)]),
    'zeros': ([0.0, 0.0], [(2, 0), (1, -1)]),
}
CLEN_S = {'dense': [0.4, -0.3, 0.2, 0.1, -0.05, 0.02], 'one': [0.7], 'trailing': [0.1, 0.2, 0.0, 0.3, 0.0, 0.0]}
CLEN_J = [1, 2, 3]         # j = 0 raises in the reference (its alphas then lack the j axis)
RADIAL = {'dense': ([0.3, -0.2, 0.1, 0.05], [0, 2, 4, 6]), 'extra_orders': ([0.2, 0.0, -0.1], [1, 3, 5, 7, 9]),
          'zeros': ([0.0, 0.0], [2, 4])}
RADIAL_R = 1.25
XY_MNS = [(0, 0), (1, 0), (0, 1), (2, 0), (1, 1), (0, 2), (3, 1), (2, 3), (5, 0), (0, 6), (4, 4)]
XY_COEFS = [0.1, -0.2, 0.3, 0.05, 0.0, -0.1, 0.02, 0.07, -0.03, 0.01, 0.004]
CHEB_MNS = [(0, 0), (1, 0), (0, 1), (2, 1), (3, 3), (5, 2), (1, 6), (2, 1)]
CHEB_COEFS = [0.2, -0.1, 0.3, 0.0, 0.05, -0.02, 0.01, 0.04]
CHEB_NORM = (2.0, 0.5)
SLOPE_N = 256
SLOPE_SEED = 20260923
# the end-to-end XY pupil: (m, n) pairs, coefficients (microns), samples, diameter (mm), wavelength, efl, Q
XYPSF_MNS = [(2, 0), (0, 2), (1, 1), (3, 0), (1, 2), (4, 0), (2, 2), (0, 4)]
XYPSF_COEFS = [0.08, 0.05, -0.04, 0.03, -0.02, 0.02, -0.03, 0.01]
XYPSF_N, XYPSF_D, XYPSF_WVL, XYPSF_EFL, XYPSF_Q = 128, 10.0, 0.6328, 100.0, 2


def line(family):
    lo, hi = FAMILIES[family][0]
    return np.linspace(lo, hi, LINE)


def slope_inputs():
    """The 256^2 unit-disk grid (x, y), Noll 2-37 (n, m) and the 36 coefficients of the slope-map case, fp64."""
    n = SLOPE_N
    v = (np.arange(n, dtype=np.float64) - n // 2) / (n // 2)
    x, y = np.meshgrid(v, v)
    coefs = np.random.default_rng(SLOPE_SEED).normal(0, 0.1, 36)
    return x, y, coefs


def xypsf_inputs():
    """Pupil amplitude, the normalised Cartesian grid and dx of the end-to-end XY case, fp64."""
    n = XYPSF_N
    dx = XYPSF_D / n
    v = (np.arange(n, dtype=np.float64) - n // 2) * dx
    x, y = np.meshgrid(v, v)
    u, w = x / (XYPSF_D / 2), y / (XYPSF_D / 2)
    amp = (np.hypot(u, w) <= 1).astype(np.float64)
    return amp, u, w, dx


def reference_modules():
    from prysm.conf import config
    from prysm import polynomials
    from prysm.propagation import Wavefront
    config.precision = 64
    return types.SimpleNamespace(p=polynomials, Wavefront=Wavefront)


def run(m):
    p = m.p
    out = {}
    for fam, (_, extra) in FAMILIES.items():
        x = line(fam)
        out[f'line_{fam}_x'] = x
        out[f'line_{fam}'] = getattr(p, f'{fam}_seq')(NS, *extra, x)
        out[f'line_{fam}_der'] = getattr(p, f'{fam}_der_seq')(NS, *extra, x)
    out['line_jacobi_wd_v'], out['line_jacobi_wd_d'] = p.jacobi_seq_with_der(NS, ALPHA, BETA, line('jacobi'))
    x = line('jacobi')
    for name, s in CLEN_S.items():
        out[f'clen_{name}'] = p.jacobi_sum_clenshaw(s, ALPHA, BETA, x)
        for j in CLEN_J:
            out[f'clen_{name}_j{j}'] = p.jacobi_sum_clenshaw_der(s, ALPHA, BETA, x, j=j)
    for g, (x, y, r, t) in grids().items():
        out.update({f'{g}_x': x, f'{g}_y': y, f'{g}_r': r, f'{g}_t': t})
        out[f'{g}_zder'] = p.zernike_nm_der_seq(ZNMS, r, t)
        out[f'{g}_zder_xy'] = p.zernike_nm_der_xy_seq(ZNMS, x, y)
        out[f'{g}_zder_raw'] = p.zernike_nm_der_seq(ZNMS, r, t, norm=False)
        for name, (c, nms) in ZSUMS.items():
            out[f'{g}_zsum_{name}'] = np.stack(p.zernike_sum_der_xy(c, nms, x, y))
        for name, (c, ns) in RADIAL.items():
            out[f'{g}_rad_{name}'] = p.jacobi_radial_sum(c, ns, ALPHA, BETA, x, y, RADIAL_R)
            out[f'{g}_rad_{name}_der'] = np.stack(p.jacobi_radial_sum_der_xy(c, ns, ALPHA, BETA, x, y, RADIAL_R))
        for kind in ('', '_der_x', '_der_y', '_der_xy'):
            fn = getattr(p, f'xy{kind}_seq')
            out[f'{g}_xy{kind}'] = fn(XY_MNS, x, y)
            out[f'{g}_xy{kind}_elem'] = fn(XY_MNS, x, y, cartesian_grid=False)
        out[f'{g}_xysum'] = p.xy_sum(XY_COEFS, XY_MNS, x, y)
        out[f'{g}_xysum_der'] = np.stack(p.xy_sum_der_xy(XY_COEFS, XY_MNS, x, y))
        out[f'{g}_xysum_elem'] = p.xy_sum(XY_COEFS, XY_MNS, x, y, cartesian_grid=False)
        out[f'{g}_chsum'] = p.cheby1_2d_sum(CHEB_COEFS, CHEB_MNS, x, y)
        out[f'{g}_chsum_der'] = np.stack(p.cheby1_2d_sum_der_xy(CHEB_COEFS, CHEB_MNS, x, y, *CHEB_NORM))
    x, y, coefs = slope_inputs()
    nms = [p.noll_to_nm(j) for j in range(2, 38)]
    out['slope_W'], out['slope_dx'], out['slope_dy'] = p.zernike_sum_der_xy(coefs, nms, x, y)   # one plane per part
    amp, u, w, dx = xypsf_inputs()
    opd = p.xy_sum(XYPSF_COEFS, XYPSF_MNS, u, w)
    wf = m.Wavefront.from_amp_and_phase(amp, opd * 1e3, XYPSF_WVL, dx)      # microns -> nm
    out['xypsf_opd'] = opd
    out['xypsf'] = np.asarray(wf.focus(XYPSF_EFL, Q=XYPSF_Q).intensity.data)
    return {k: np.asarray(v, dtype=np.float64) for k, v in out.items()}


def reference_outputs():
    import warnings
    with reference.loaded(), warnings.catch_warnings():
        m = reference_modules()
        warnings.simplefilter('ignore')
        return run(m)


def main():
    """Write tests/golden/polynomials*.npz from the unmodified reference."""
    with reference.loaded():
        from make_golden import save      # imports the reference
        save('polynomials.npz', reference_outputs())


if __name__ == '__main__':
    main()
