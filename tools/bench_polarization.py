"""Polarized propagation on the device (prysm_b200.polarization), with the reference's host path in the same run.

    python tools/bench_polarization.py [--iters 20] [--no-reference] [--out result.json]

At precision 32, with CUDA events over `iters` calls after warm-up:
- Jones focus 2048^2 -> 4096^2 (Q = 2) of an element-planar field, against 4 single-field focus calls, alternated;
- Jones focus_dft (MDFT 1024^2 -> 256^2) against 4 single-field executor calls, alternated;
- the four kernels at 4096^2: pb_jones_planar (interleaved device field -> planes), pb_jones_product (Jones @ Jones),
  pb_jones_elements (vector vortex retarder from an azimuth plane) and pb_jones_reduce (jones_to_mueller), with the
  bytes each must move (read once, written once) over its time, against the H100 SXM data sheet's 3.35 TB/s.
The reference's numpy path (oracle/_ref, fp64 as it runs by default) is timed once per call: the Jones focus and
focus_dft at the same sizes, the elementwise calls at 2048^2 (its (M, N, 4, 4) temporaries at 4096^2 take >10 GB).
The card name, power limit and current SM clock are read in the same run.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'oracle')]
import reference  # noqa: E402
from benchlib import HBM_BYTES_PER_S, card, host_time, timed  # noqa: E402


def alternate(fa, fb, iters, rounds=5):
    """Median over `rounds` of (fa, fb) timed back to back."""
    ta, tb = [], []
    for _ in range(rounds):
        ta.append(timed(fa, iters, warm=1)[0] * 1e6)
        tb.append(timed(fb, iters, warm=1)[0] * 1e6)
    return float(np.median(ta)), float(np.median(tb))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--no-reference', action='store_true')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import torch
    import prysm_b200 as pb
    from prysm_b200 import propagation as P, polarization as pol
    pb.config.precision = 32
    rng = np.random.default_rng(0)
    res = {'card (name, power limit, SM clock, max SM clock)': card(), 'precision': 32}

    def rfield(n):
        return pb.asdevice((rng.standard_normal((n, n)) + 1j * rng.standard_normal((n, n))).astype(np.complex64))

    # ---- Jones focus 2048^2 -> 4096^2
    n = 2048
    f = rfield(n)
    J = pol.apply_polarization_optic(f, pol.linear_retarder(pb.asdevice(rng.uniform(0, 1, (n, n)).astype(np.float32)),
                                                            theta=0.3, shape=(n, n)))
    planes = [J[..., i, j] for i in range(2) for j in range(2)]
    jfocus = pol.jones_adapter(P.focus)
    tj, ts = alternate(lambda: jfocus(J, 2), lambda: [P.focus(p, 2) for p in planes], args.iters)
    res['jones_focus_2048_Q2_us'] = tj
    res['4x_focus_2048_Q2_us'] = ts
    res['jones_focus_over_4x'] = tj / ts - 1

    # ---- Jones focus_dft: MDFT 1024^2 -> 256^2
    n, m = 1024, 256
    ex = P.prepare_executor(10.0 / n, (n, n), 0.55 * 100 / 10 / 2, (m, m), 0.55, 100.0, kind='mdft')
    Jd = pol.apply_polarization_optic(rfield(n), pol.pauli_spin_matrix(0))
    dplanes = [Jd[..., i, j] for i in range(2) for j in range(2)]
    jdft = pol.jones_adapter(P.focus_dft)
    tj, ts = alternate(lambda: jdft(Jd, ex), lambda: [ex(p) for p in dplanes], args.iters)
    res['jones_focus_dft_1024_256_us'] = tj
    res['4x_mdft_1024_256_us'] = ts
    res['jones_focus_dft_over_4x'] = tj / ts - 1
    del J, Jd, planes, dplanes, f

    # ---- the four kernels at 4096^2
    n = 4096
    px = n * n
    A = pol.apply_polarization_optic(rfield(n), pol.linear_retarder(0.4, theta=0.2))
    B = pol.apply_polarization_optic(rfield(n), pol.linear_retarder(1.1, theta=-0.5))
    inter = A.contiguous()                          # interleaved (n, n, 2, 2) on the device
    theta = pb.asdevice(rng.uniform(-np.pi, np.pi, (n, n)).astype(np.float32))
    kernels = {
        'pb_jones_planar (interleaved -> planes)': (lambda: pol._planes(inter), 32 + 32),
        'pb_jones_product (Jones @ Jones)': (lambda: pol.jones_matmul(A, B), 32 + 32 + 32),
        'pb_jones_elements (vector vortex retarder)': (lambda: pol.vector_vortex_retarder(2, theta), 4 + 32),
        'pb_jones_reduce (jones_to_mueller)': (lambda: pol.jones_to_mueller(A), 32 + 64),
    }
    res['kernels_4096'] = {}
    for name, (fn, bpp) in kernels.items():
        t = timed(fn, args.iters, warm=1)[0] * 1e6
        gbs = bpp * px / (t * 1e-6) / 1e9
        res['kernels_4096'][name] = {'us': t, 'bytes_per_pixel': bpp, 'GB/s': gbs,
                                     'share_of_3.35TB/s': gbs * 1e9 / HBM_BYTES_PER_S}
    del A, B, inter, theta
    torch.cuda.empty_cache()

    # ---- the reference's host path
    if not args.no_reference:
        with reference.loaded():
            from prysm.x import polarization as rpol
            from prysm import propagation as rprop
            hr = {}
            n = 2048
            Jh = (rng.standard_normal((n, n, 2, 2)) + 1j * rng.standard_normal((n, n, 2, 2)))
            hr['jones_focus_2048_Q2_us'] = 1e6 * host_time(lambda: rpol.jones_adapter(rprop.focus)(Jh, 2))
            n, m = 1024, 256
            rex = rprop.prepare_executor(10.0 / n, (n, n), 0.55 * 100 / 10 / 2, (m, m), 0.55, 100.0, kind='mdft')
            Jm = Jh[:n, :n].copy()
            hr['jones_focus_dft_1024_256_us'] = 1e6 * host_time(lambda: rpol.jones_adapter(rprop.focus_dft)(Jm, rex))
            Kh = Jh[::-1].copy()
            th = rng.uniform(-np.pi, np.pi, Jh.shape[:2])
            hr['matmul_2048_us'] = 1e6 * host_time(lambda: Jh @ Kh)
            hr['vector_vortex_retarder_2048_us'] = 1e6 * host_time(lambda: rpol.vector_vortex_retarder(2, th.copy()))
            hr['jones_to_mueller_2048_us'] = 1e6 * host_time(lambda: rpol.jones_to_mueller(Jh))
        res['reference_host_fp64'] = hr
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as fh:
            fh.write(line + '\n')


if __name__ == '__main__':
    main()
