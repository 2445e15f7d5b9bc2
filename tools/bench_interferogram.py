"""Interferogram metrology: each step of a circular NaN-masked map with tilt and power, on the engine (CUDA events)
and on the host reference (perf_counter), at 1000^2 and 2048^2.

    python tools/bench_interferogram.py [--sizes 1000 2048] [--iters 5] [--no-reference]

Prints the card (name, power limit, clocks) and one line per step and size: engine ms, kernel launches per call,
reference ms.  The reference runs from oracle/_ref (or PRYSM_REFERENCE).
"""
import argparse
import os
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'oracle'), os.path.join(ROOT, 'tools')):
    if p not in sys.path:
        sys.path.insert(0, p)

import benchlib  # noqa: E402


def make_map(n, seed=1):
    rng = np.random.default_rng(seed)
    y, x = (np.mgrid[:n, :n] - n // 2) / (n // 2)
    d = 40 * x - 25 * y + 1.5 * (x * x + y * y) + rng.standard_normal((n, n))
    d[np.hypot(x, y) > 0.95] = np.nan
    return d


def steps(I, d, dx):
    """name -> callable on a fresh object; the filter runs on the filled map (a NaN spreads through the transform)"""
    f = np.nan_to_num(d) if isinstance(d, np.ndarray) else d.nan_to_num()

    def fresh(a):
        return I(a.copy() if isinstance(a, np.ndarray) else a.clone(), dx=dx)
    return {
        'pvr': lambda: fresh(d).pvr(),
        'remove_tiptilt': lambda: fresh(d).remove_tiptilt(),
        'remove_power': lambda: fresh(d).remove_power(),
        'psd': lambda: fresh(f).psd(),
        'bandlimited_rms': lambda: fresh(f).bandlimited_rms(flow=1.0, fhigh=5.0),
        'total_integrated_scatter': lambda: fresh(f).total_integrated_scatter(10.6),
        'filter_lp': lambda: fresh(f).filter(2.0, 'lp'),
        'rms_pv_Sa_std': lambda: [getattr(fresh(d), k) for k in ('rms', 'pv', 'Sa', 'std')],
        'slope': lambda: fresh(d).slope(),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--sizes', type=int, nargs='+', default=[1000, 2048])
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--no-reference', action='store_true')
    args = ap.parse_args()
    import torch
    import prysm_b200 as pb
    import reference
    print('card:', benchlib.card())
    dx = 0.05
    for n in args.sizes:
        d = make_map(n)
        eng = steps(pb.interferogram.Interferogram, torch.from_numpy(d).cuda(), dx)
        ref = {}
        if not args.no_reference and reference.installed():
            with reference.loaded(), warnings.catch_warnings():
                warnings.simplefilter('ignore')
                from prysm import interferogram as pifg
                for k, fn in steps(pifg.Interferogram, d, dx).items():
                    fn()
                    ref[k] = min(benchlib.host_time(fn) for _ in range(2))
        for k, fn in eng.items():
            t, nl = benchlib.timed(fn, args.iters)
            r = f'{ref[k] * 1e3:10.2f} ms' if k in ref else '    (not run)'
            print(f'{n:5d}^2 {k:26s} engine {t * 1e3:9.3f} ms  {nl:5.1f} launches   reference {r}', flush=True)


if __name__ == '__main__':
    main()
