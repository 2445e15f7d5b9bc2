"""Thin-film stacks on the device (prysm_b200.thinfilm, prysm_b200.coatings), with the reference's host calls in the
same run.

    python tools/bench_thinfilm.py [--iters 10] [--no-reference] [--out result.json]

CUDA events over `iters` calls after warm-up, results stored in fp64 (the chain is fp64 at either precision):
- `ml_pixel_2048`: multilayer_stack_rt, 4 layers with per-pixel index and thickness maps at 2048^2 (device inputs);
- `fold_mirror_2048`: a 2-layer protected-silver fold mirror (1-D layers) under a 2048^2 AOI map, s and p;
- `rta_40_<grid>`: RTA of a 40-layer stack with one lossy layer on 2001 x 61 and 8192 x 512 (wavelength x angle);
- `fwd_grad_40_<grid>`: forward_eval + thickness_gradient with a dR seed on the same grids.
Each has a byte floor (operands read and outputs written once, over the H100 SXM data sheet's 3.35 TB/s) and an fp64
floor (FP64_OPS_PER_LAYER operations per layer and sample, transcendentals counted as one, over the data sheet's
34 TFLOP/s of non-tensor FP64); both are arithmetic, not measurements.  The reference's numpy calls (oracle/_ref,
fp64) are timed once at the sizes it finishes in seconds.  The card name, power limit and SM clocks are read in the
same run.
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

FP64_FLOP_PER_S = 34e12          # H100 SXM data sheet, FP64 without tensor cores
# per layer and sample: Snell cosine (complex divide, square, square root), phase and admittance, complex sin / cos,
# and the 2 x 2 matrix-vector product; the gradient's reverse sweep about twice that
FP64_OPS_PER_LAYER = 110
GRIDS = {'2001x61': (2001, 61), '8192x512': (8192, 512)}
SILVER = ([1.46, 0.05 + 3.9j], [0.08, 0.12])


def pixel_maps(N, rng):
    idx = np.array([1.38, 2.05, 1.38, 2.05])[:, None, None] * np.ones((1, N, N))
    th = np.array([0.1, 0.07, 0.1, 0.07])[:, None, None] * (1 + 0.02 * rng.standard_normal((1, N, N)))
    return idx, th


def aoi_map(N):
    v = np.linspace(-1, 1, N)
    x, y = np.meshgrid(v, v)
    return 45.0 + 8.0 * x + 2.0 * x * y


def stack40():
    rng = np.random.default_rng(3)
    ind = [1.45 if i % 2 else 2.3 for i in range(40)]
    ind[5] = 1.5 + 0.3j
    return ind, rng.uniform(0.05, 0.15, 40), 1.52


def grid(name):
    W, A = GRIDS[name]
    return np.linspace(0.4, 0.9, W)[:, None], np.radians(np.linspace(0, 60, A))[None, :]


def floors(samples, layers, bytes_moved, grad=False):
    ops = FP64_OPS_PER_LAYER * (3 if grad else 1) * layers * samples
    return {'byte_floor_s': bytes_moved / HBM_BYTES_PER_S, 'fp64_floor_s': ops / FP64_FLOP_PER_S}


def reference_times():
    if not reference.installed():
        return None
    with reference.loaded():
        from prysm.conf import config
        from prysm import thinfilm
        from prysm.x.coatings import Stack, RTA, forward_eval, thickness_gradient
        config.precision = 64
        out = {}
        with warnings.catch_warnings():
            warnings.simplefilter('ignore')
            idx, th = pixel_maps(512, np.random.default_rng(0))
            out['ml_pixel_512_s'] = host_time(lambda: thinfilm.multilayer_stack_rt(idx, th, 0.55, 'p', 1.52, aoi=10))
            a = aoi_map(512)
            out['fold_mirror_512_s'] = host_time(lambda: [thinfilm.multilayer_stack_rt(*SILVER, 0.55, p, 1.52, aoi=a)
                                                          for p in 'sp'])
            st = Stack(*stack40())
            w, t = grid('2001x61')
            out['rta_40_2001x61_s'] = host_time(lambda: RTA(st, w, t, 's'))

            def fg():
                f = forward_eval(st, w, t, 's')
                return thickness_gradient(f, dR=np.ones_like(f.r.real))
            out['fwd_grad_40_2001x61_s'] = host_time(fg)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--no-reference', action='store_true')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()

    import torch
    from prysm_b200 import coatings as c, thinfilm as tf

    res = {'card': card(), 'workloads': {}}

    def record(name, fn, fl):
        s, launches = timed(fn, args.iters)
        row = {'s': s, 'launches': launches, **fl}
        res['workloads'][name] = row
        print(json.dumps({name: row}), flush=True)

    N = 2048
    idx, th = pixel_maps(N, np.random.default_rng(0))
    idx_d = torch.as_tensor(idx).to('cuda', torch.complex128)
    th_d = torch.as_tensor(th).to('cuda', torch.float64)
    record('ml_pixel_2048', lambda: tf.multilayer_stack_rt(idx_d, th_d, 0.55, 'p', 1.52, aoi=10),
           floors(N * N, 4, 4 * N * N * (16 + 8) + 2 * N * N * 16))
    del idx_d, th_d
    a = torch.as_tensor(aoi_map(N)).to('cuda', torch.float64)
    record('fold_mirror_2048', lambda: [tf.multilayer_stack_rt(*SILVER, 0.55, p, 1.52, aoi=a) for p in 'sp'],
           floors(2 * N * N, 2, 2 * (N * N * 8 + 2 * N * N * 16)))
    del a
    st = c.Stack(*stack40())
    for g in GRIDS:
        w, t = grid(g)
        n = w.size * t.size
        record(f'rta_40_{g}', lambda: c.RTA(st, w, t, 's'), floors(n, 40, n * (8 + 8 + 40 * 8)))

        def fg():
            f = c.forward_eval(st, w, t, 's')
            return c.thickness_gradient(f, dR=1.0)
        # forward_eval keeps r, t, E, H, R, T, A, |E|^2, eta0, eta_sub; the gradient reads E, H and the dR seed
        fwd_bytes = n * (4 * 16 + 2 * 41 * 16 + 2 * 8 + 40 * 8 + 41 * 8)
        record(f'fwd_grad_40_{g}', fg, floors(n, 40, fwd_bytes + n * (2 * 41 * 16 + 8), grad=True))
        torch.cuda.empty_cache()
    if not args.no_reference:
        res['reference'] = reference_times()
        print(json.dumps({'reference': res['reference']}), flush=True)
    if args.out:
        with open(args.out, 'w') as fh:
            json.dump(res, fh, indent=1)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
