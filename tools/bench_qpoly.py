"""Forbes polynomials on the device (prysm_b200.qpoly), with the reference's host calls in the same run.

    python tools/bench_qpoly.py [--iters 20] [--no-reference] [--out result.json]

CUDA events over `iters` calls after warm-up, at 512^2 and 2048^2 (a polar grid over the unit disk's bounding square),
fp64 and fp32, with the 117-mode 2D-Q set n <= 8, |m| <= 6 (cosine and sine terms):
- Q2d_seq (117 planes), Q2d_der_xy_seq (2 x 117 planes), each with its byte floor: the planes written plus the two
  inputs read once, over the H100 SXM data sheet's 3.35 TB/s (arithmetic, not a measurement);
- compute_z_zprime_Q2d with one coefficient per mode (three planes written).
The reference's numpy calls (oracle/_ref, fp64) are timed once at 512^2 (at 2048^2 its per-order tables and outputs
run to several GB of host memory).  The card name, power limit and current and
maximum SM clocks are read in the same run.
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
NMS = [(n, m) for m in range(-6, 7) for n in range(9)]          # 13 x 9 = 117 modes
assert len(NMS) == 117


def polar(N):
    v = np.linspace(-1.0, 1.0, N)
    x, y = np.meshgrid(v, v)
    return x, y, np.hypot(x, y), np.arctan2(y, x)


def coefficients():
    rng = np.random.default_rng(5)
    return rng.standard_normal(len(NMS)) * 0.01


def reference_times(N):
    if not reference.installed():
        return None
    with reference.loaded():
        from prysm.conf import config
        from prysm.polynomials import qpoly as q
        config.precision = 64
        x, y, r, t = polar(N)
        cm0, ams, bms = q.Q2d_nm_c_to_a_b(NMS, coefficients())
        with warnings.catch_warnings():
            warnings.simplefilter('ignore')
            return {'Q2d_seq_s': host_time(lambda: q.Q2d_seq(NMS, r, t)),
                    'Q2d_der_xy_seq_s': host_time(lambda: q.Q2d_der_xy_seq(NMS, x, y)),
                    'compute_z_zprime_Q2d_s': host_time(lambda: q.compute_z_zprime_Q2d(cm0, ams, bms, r, t))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--no-reference', action='store_true')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()

    import torch
    from prysm_b200 import qpoly as Q

    res = {'card': card(), 'sizes': {}}
    for N in SIZES:
        row = {}
        xh, yh, rh, th = polar(N)
        for dt, name in ((torch.float64, 'fp64'), (torch.float32, 'fp32')):
            x, y, r, t = (torch.as_tensor(v).to('cuda', dt) for v in (xh, yh, rh, th))
            es = x.element_size()
            cm0, ams, bms = Q.Q2d_nm_c_to_a_b(NMS, coefficients())
            row[f'Q2d_seq_{name}_s'] = timed(lambda: Q.Q2d_seq(NMS, r, t), args.iters)[0]
            row[f'Q2d_seq_{name}_floor_s'] = (len(NMS) + 2) * N * N * es / HBM_BYTES_PER_S
            row[f'Q2d_der_xy_seq_{name}_s'] = timed(lambda: Q.Q2d_der_xy_seq(NMS, x, y), args.iters)[0]
            row[f'Q2d_der_xy_seq_{name}_floor_s'] = (2 * len(NMS) + 2) * N * N * es / HBM_BYTES_PER_S
            row[f'compute_z_zprime_Q2d_{name}_s'] = timed(lambda: Q.compute_z_zprime_Q2d(cm0, ams, bms, r, t),
                                                          args.iters)[0]
            row[f'compute_z_zprime_Q2d_{name}_floor_s'] = 5 * N * N * es / HBM_BYTES_PER_S
            del x, y, r, t
            torch.cuda.empty_cache()
        if not args.no_reference and N == 512:          # at 2048^2 the reference's tables outgrow host memory
            row['reference'] = reference_times(N)
        res['sizes'][f'{N}^2'] = row
        print(json.dumps({f'{N}^2': row}), flush=True)
    if args.out:
        with open(args.out, 'w') as fh:
            json.dump(res, fh, indent=1)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
