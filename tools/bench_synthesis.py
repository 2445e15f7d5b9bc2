"""GPU timing of the SURVEY.md 8(f) rank-3 row: pupil synthesis at the BASELINE C2 size (2048^2, fp32 storage).

    python tools/bench_synthesis.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import prysm_b200 as pb  # noqa: E402
from benchlib import timed  # noqa: E402
from prysm_b200 import coordinates as C, geometry as G, polynomials as Z, propagation as P  # noqa: E402


for prec in (32, 64):
    pb.config.precision = prec
    N = 2048
    b = 4 if prec == 32 else 8
    x, y = C.make_xy_grid(N, diameter=2.0)
    r, t = C.cart_to_polar(x, y)
    nms = [Z.noll_to_nm(j) for j in range(2, 38)]
    coefs = np.random.default_rng(1).normal(0, 30, 36)
    us = timed(lambda: C.make_xy_grid(N, diameter=2.0), 20)[0] * 1e6
    print(f'[p{prec}] make_xy_grid {N}^2: {us:.1f} us ({2 * N * N * b / us / 1e3:.0f} GB/s written)')
    us = timed(lambda: C.cart_to_polar(x, y), 20)[0] * 1e6
    print(f'[p{prec}] cart_to_polar {N}^2: {us:.1f} us ({4 * N * N * b / us / 1e3:.0f} GB/s r+w)')
    us = timed(lambda: G.circle(1.0, r), 20)[0] * 1e6
    print(f'[p{prec}] circle {N}^2: {us:.1f} us')
    us = timed(lambda: Z.zernike_nm_seq(nms, r, t), 20)[0] * 1e6
    print(f'[p{prec}] zernike_nm_seq 36 modes {N}^2: {us:.1f} us ({38 * N * N * b / us / 1e3:.0f} GB/s r+w)')
    us = timed(lambda: Z.zernike_sum(coefs, nms, x, y), 20)[0] * 1e6
    print(f'[p{prec}] zernike_sum 36 modes {N}^2 (coefficients -> OPD, no basis): {us:.1f} us ({3 * N * N * b / us / 1e3:.0f} GB/s r+w)')
    basis = Z.zernike_nm_seq(nms, r, t)
    us = timed(lambda: Z.sum_of_2d_modes(basis, coefs), 20)[0] * 1e6
    print(f'[p{prec}] sum_of_2d_modes over the stored 36-mode basis {N}^2: {us:.1f} us ({37 * N * N * b / us / 1e3:.0f} GB/s r+w)')
    amp = G.circle(1.0, r)

    def model():
        opd = Z.zernike_sum(coefs, nms, x, y)
        return P.Wavefront.from_amp_and_phase(amp, opd, 0.6328, 2.0 / N).focus(100.0, Q=2)
    if prec == 32:
        us = timed(model, 20)[0] * 1e6
        print(f'[p{prec}] coefficients -> OPD -> pupil -> focus {N}^2 -> {2 * N}^2: {us:.1f} us')
    del basis
