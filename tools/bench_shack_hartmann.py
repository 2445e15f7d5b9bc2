"""Shack-Hartmann sensing on the device (prysm_b200.shack_hartmann), with the reference's host screen in the same run.

    python tools/bench_shack_hartmann.py [--iters 20] [--no-reference] [--out result.json]

CUDA events over `iters` calls after warm-up, at 512^2 with 16^2 lenslets and 2048^2 with 64^2 lenslets (dx = 10 um,
pitch = 32 samples, efl 20 mm, 0.55 um, fp64 and fp32 grids):
- shack_hartmann: the screen, one launch (rectangle lenslets, and circles with shift=True), as a whole call (which
  reads the grid spacing back from the device to find its cached plan) and as the launch alone;
- ShackHartmann.forward_model: (wave * screen).free_space(dz=efl).intensity on a cached screen;
- spot_centroids of 16 uint16 frames, against their byte bound (the frames read once over the H100 SXM data sheet's
  3.35 TB/s; the bound is arithmetic, not a measurement);
- reconstruct of 10 modes (Noll 2-11) from one slope vector and from 16.
The reference's numpy screen (oracle/_ref) is timed once per configuration.  The card name, power limit and current and
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

CONFIGS = ((512, 16), (2048, 64))
DX, PITCH_SAMPLES, EFL, WVL = 0.01, 32, 20.0, 0.55


def reference_screen_times(N, n, pitch):
    if not reference.installed():
        return None
    with reference.loaded():
        from prysm.conf import config
        from prysm.coordinates import make_xy_grid
        from prysm.geometry import circle
        from prysm.x.shack_hartmann import shack_hartmann
        config.precision = 64
        x, y = make_xy_grid(N, dx=DX)
        with warnings.catch_warnings():
            warnings.simplefilter('ignore')
            return {'rectangle': host_time(lambda: shack_hartmann(pitch, n, EFL, WVL, x, y)),
                    'circle_shift': host_time(lambda: shack_hartmann(pitch, n, EFL, WVL, x, y, aperture=circle,
                                                                     shift=True))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--no-reference', action='store_true')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()

    import torch
    import prysm_b200 as pb
    from prysm_b200 import shack_hartmann as S

    res = {'card': card(), 'configs': {}}
    for N, n in CONFIGS:
        pitch = PITCH_SAMPLES * DX
        row = {}
        for prec in (64, 32):
            pb.config.precision = prec
            x, y = pb.coordinates.make_xy_grid(N, dx=DX)
            row[f'screen_rect_fp{prec}_s'] = timed(lambda: S.shack_hartmann(pitch, n, EFL, WVL, x, y), args.iters)[0]
            plan = S._plan_for(pitch, n, x, y, False)
            row[f'screen_rect_kernel_fp{prec}_s'] = timed(lambda: S._screen(plan, pitch, EFL, WVL, x, y, S.rectangle, None),
                                                          args.iters)[0]
            row[f'screen_bytes_fp{prec}'] = x.numel() * x.element_size() * 4      # x, y read; complex written
            row[f'screen_circle_shift_fp{prec}_s'] = timed(
                lambda: S.shack_hartmann(pitch, n, EFL, WVL, x, y, aperture=pb.geometry.circle, shift=True), args.iters)[0]
            sh = S.ShackHartmann(pitch, n, EFL, WVL, x, y, shift=True)
            wave = pb.Wavefront(torch.ones_like(x).to(pb.config.complex_dtype), WVL, DX)
            row[f'forward_model_fp{prec}_s'] = timed(lambda: sh.forward_model(wave), args.iters)[0]
        pb.config.precision = 64
        x, y = pb.coordinates.make_xy_grid(N, dx=DX)
        sh = S.ShackHartmann(pitch, n, EFL, WVL, x, y, shift=True)
        I = sh.forward_model(pb.Wavefront(torch.ones_like(x).to(torch.complex128), WVL, DX)).data
        frame = np.round(I.cpu().numpy() / float(I.max()) * 60000).astype(np.uint16)
        stack = pb.asdevice(np.repeat(frame[None], 16, axis=0))
        t = timed(lambda: sh.centroids(stack, 0.0), args.iters)[0]
        row['centroids_16_u16_s'] = t
        row['centroids_16_u16_threshold_s'] = timed(lambda: sh.centroids(stack, 0.1), args.iters)[0]
        row['centroids_16_u16_bytes'] = stack.numel() * 2
        row['centroids_16_u16_bound_s'] = stack.numel() * 2 / HBM_BYTES_PER_S
        # the reconstructor of Noll 2-11 over the full grid (tilt, focus, astigmatism, coma, trefoil, spherical)
        xh, yh = x.cpu().numpy(), y.cpu().numpy()
        R0 = N * DX / 2
        r, th = np.hypot(xh, yh) / R0, np.arctan2(yh, xh)
        modes = np.stack([r * np.cos(th), r * np.sin(th), 2 * r ** 2 - 1, r ** 2 * np.sin(2 * th), r ** 2 * np.cos(2 * th),
                          (3 * r ** 3 - 2 * r) * np.sin(th), (3 * r ** 3 - 2 * r) * np.cos(th), r ** 3 * np.sin(3 * th),
                          r ** 3 * np.cos(3 * th), 6 * r ** 4 - 6 * r ** 2 + 1]) * 50.0
        sh.calibrate(modes, 1.0)
        s1 = sh.slopes(I)
        s16 = s1[None].repeat(16, 1, 1, 1).contiguous()
        row['reconstruct_1_s'] = timed(lambda: sh.reconstruct(s1), args.iters)[0]
        row['reconstruct_16_s'] = timed(lambda: sh.reconstruct(s16), args.iters)[0]
        row['valid_subapertures'] = int(sh.valid.sum())
        if not args.no_reference:
            row['reference_screen_s'] = reference_screen_times(N, n, pitch)
        res['configs'][f'{N}^2/{n}^2'] = row
        print(json.dumps({f'{N}^2/{n}^2': row}), flush=True)
    if args.out:
        with open(args.out, 'w') as fh:
            json.dump(res, fh, indent=1)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
