"""GPU timing of the deformable mirror (prysm_b200.dm.DM) and of its cubic-spline warp kernel (fp32).

    python tools/bench_dm.py [--out FILE.json]

For 512^2 (48^2 actuators, sep 8), 1024^2 (48^2, 16) and 2048^2 (64^2, 24), each flat, tilted (5, 0, 10) and tilted
with upsample 0.75: render and render_adjoint per call (CUDA events over 20 calls after warm-up) and launches per
call; a forward + inverse pb_fft2 pair of the same size as the yardstick; the warp (prefilter + interpolation) alone
with its HBM bandwidth from the bytes it must move; and the unmodified reference's render on the host cores, when
oracle/_ref holds it.  The card's name and power limit are printed with the numbers.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'oracle')]
import prysm_b200 as pb  # noqa: E402
import reference  # noqa: E402
from benchlib import card, timed  # noqa: E402
from prysm_b200 import _ops  # noqa: E402

SIZES = ((512, 48, 8), (1024, 48, 16), (2048, 64, 24))
VARIANTS = (('flat', dict()), ('tilt', dict(rot=(5, 0, 10))), ('tilt_up075', dict(rot=(5, 0, 10), upsample=0.75)))


def ifn_for(n, sep):
    y = np.arange(n) - n // 2
    return np.exp(-2 * ((y[None, :] / (1.2 * sep)) ** 2 + (y[:, None] / (1.2 * sep)) ** 2)).astype(np.float32)


def reference_render_us(n, nact, sep, kw, reps=3):
    if not reference.installed():
        return None
    with reference.loaded():
        from prysm.conf import config
        from prysm.x.dm import DM
        config.precision = 32
        dm = DM(ifn_for(n, sep), Nout=n, Nact=nact, sep=sep, **kw)
        dm.actuators[:] = np.random.default_rng(0).uniform(-1, 1, dm.actuators.shape).astype(np.float32)
        dm.render()
        t0 = time.perf_counter()
        for _ in range(reps):
            dm.render()
        return (time.perf_counter() - t0) / reps * 1e6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    pb.config.precision = 32
    rows = []
    print('card:', card())
    for n, nact, sep in SIZES:
        x = pb.asdevice(np.random.default_rng(1).standard_normal((n, n)).astype(np.float32))
        xc = _ops.fft2(x)
        pair_s, _ = timed(lambda: _ops.fft2(_ops.fft2(xc, dir=-1, shift_in=True), dir=+1, shift_out=True), 20)
        Mfwd, Mifwd = pb.dm.projection_matrices((n, n), (5, 0, 10))
        warp_s, warp_launches = timed(lambda: _ops.warp(x, matrix=Mifwd), 20)
        pair_us, warp_us = pair_s * 1e6, warp_s * 1e6
        # prefilter: read fp32 input, write + read fp64 intermediate, write + read fp64 coefficients; interpolation
        # writes fp32 (the 4 x 4 taps mostly hit L1 / L2): the least traffic of the two passes and the gather
        warp_bytes = n * n * (4 + 8 + 8 + 8 + 8 + 4)
        print(f'{n}^2: fft2 pair {pair_us:.1f} us; warp {warp_us:.1f} us ({warp_launches:.0f} launches, '
              f'{warp_bytes / warp_us / 1e3:.0f} GB/s of {warp_bytes / 2**20:.0f} MiB)')
        for vname, kw in VARIANTS:
            dm = pb.dm.DM(ifn_for(n, sep), Nout=n, Nact=nact, sep=sep, **kw)
            dm.update(np.random.default_rng(0).uniform(-1, 1, (nact, nact)).astype(np.float32))
            r_s, r_l = timed(dm.render, 20)
            g = dm.render().clone()
            a_s, a_l = timed(lambda: dm.render_adjoint(g), 20)
            r_us, a_us = r_s * 1e6, a_s * 1e6
            ref_us = reference_render_us(n, nact, sep, kw)
            row = dict(n=n, nact=nact, sep=sep, variant=vname, render_us=r_us, render_launches=r_l, adjoint_us=a_us,
                       adjoint_launches=a_l, fft2_pair_us=pair_us, warp_us=warp_us, warp_gbs=warp_bytes / warp_us / 1e3,
                       reference_render_us=ref_us)
            rows.append(row)
            ref_s = 'not measured' if ref_us is None else f'{ref_us / 1e3:.1f} ms'
            print(f'  {vname:11s} render {r_us:8.1f} us ({r_l:.0f} launches)  adjoint {a_us:8.1f} us ({a_l:.0f} launches)'
                  f'  reference render on the host {ref_s}')
    if args.out:
        with open(args.out, 'w') as fh:
            json.dump({'card': card(), 'rows': rows}, fh, indent=1)


if __name__ == '__main__':
    main()
