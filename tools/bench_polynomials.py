"""Orthogonal polynomials, Zernike derivatives and polynomial sums on the device (prysm_b200.polynomials), with the
reference's host calls in the same run.

    python tools/bench_polynomials.py [--iters 20] [--no-reference] [--out result.json]

CUDA events over `iters` calls after warm-up, at 512^2 and 2048^2 (the unit disk's bounding square), fp64 and fp32:
- legendre_seq, orders 0-40 (41 planes);
- zernike_nm_der_xy_seq, Noll 2-37 (36 modes, 72 planes);
- zernike_sum_der_xy with 36 coefficients on the same modes (x, y read; W, dW/dx, dW/dy written);
- xy_sum_der_xy over every m + n <= 10 (66 terms) on the separable grid (one row and one column read, 3 planes written).
Each with its byte floor, the planes read plus the planes written over the H100 SXM data sheet's 3.35 TB/s
(arithmetic, not a measurement).  The reference's numpy calls (oracle/_ref, fp64) are timed once at 512^2.  The card
name, power limit and current and maximum SM clocks are read in the same run.
"""
import argparse
import json
import os
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'oracle')]
import reference  # noqa: E402
from benchlib import HBM_BYTES_PER_S, card, host_time, timed  # noqa: E402

SIZES = (512, 2048)
LEG_NS = list(range(41))
XY_MNS = [(m, n) for m in range(11) for n in range(11) if m + n <= 10]
assert len(XY_MNS) == 66


def grid(N):
    v = np.linspace(-1.0, 1.0, N)
    return np.meshgrid(v, v)


def coefficients(k, seed):
    return np.random.default_rng(seed).standard_normal(k) * 0.01


def reference_times(N, nms):
    if not reference.installed():
        return None
    with reference.loaded():
        from prysm.conf import config
        from prysm import polynomials as p
        config.precision = 64
        x, y = grid(N)
        zc, xc = coefficients(len(nms), 1), coefficients(len(XY_MNS), 2)
        with warnings.catch_warnings():
            warnings.simplefilter('ignore')
            return {'legendre_seq_s': host_time(lambda: p.legendre_seq(LEG_NS, x)),
                    'zernike_nm_der_xy_seq_s': host_time(lambda: p.zernike_nm_der_xy_seq(nms, x, y)),
                    'zernike_sum_der_xy_s': host_time(lambda: p.zernike_sum_der_xy(zc, nms, x, y)),
                    'xy_sum_der_xy_s': host_time(lambda: p.xy_sum_der_xy(xc, XY_MNS, x, y))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--no-reference', action='store_true')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()

    import torch
    from prysm_b200 import polynomials as P

    nms = [P.noll_to_nm(j) for j in range(2, 38)]
    zc, xc = coefficients(len(nms), 1), coefficients(len(XY_MNS), 2)
    res = {'card': card(), 'sizes': {}}
    for N in SIZES:
        row = {}
        xh, yh = grid(N)
        for dt, name in ((torch.float64, 'fp64'), (torch.float32, 'fp32')):
            x, y = (torch.as_tensor(v).to('cuda', dt) for v in (xh, yh))
            es, px = x.element_size(), N * N
            row[f'legendre_seq_{name}_s'] = timed(lambda: P.legendre_seq(LEG_NS, x), args.iters)[0]
            row[f'legendre_seq_{name}_floor_s'] = (len(LEG_NS) + 1) * px * es / HBM_BYTES_PER_S
            row[f'zernike_nm_der_xy_seq_{name}_s'] = timed(lambda: P.zernike_nm_der_xy_seq(nms, x, y), args.iters)[0]
            row[f'zernike_nm_der_xy_seq_{name}_floor_s'] = (2 * len(nms) + 2) * px * es / HBM_BYTES_PER_S
            row[f'zernike_sum_der_xy_{name}_s'] = timed(lambda: P.zernike_sum_der_xy(zc, nms, x, y), args.iters)[0]
            row[f'zernike_sum_der_xy_{name}_floor_s'] = 5 * px * es / HBM_BYTES_PER_S
            row[f'xy_sum_der_xy_{name}_s'] = timed(lambda: P.xy_sum_der_xy(xc, XY_MNS, x, y), args.iters)[0]
            row[f'xy_sum_der_xy_{name}_floor_s'] = 3 * px * es / HBM_BYTES_PER_S
            del x, y
            torch.cuda.empty_cache()
        if not args.no_reference and N == 512:
            row['reference'] = reference_times(N, nms)
        res['sizes'][f'{N}^2'] = row
        print(json.dumps({f'{N}^2': row}), flush=True)
    if args.out:
        with open(args.out, 'w') as fh:
            json.dump(res, fh, indent=1)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
