"""Optical monitoring on the device (prysm_b200.coatings simulate_run, simulate_runs, monitoring_error_sensitivity and
choose_monitor_wavelength), with the reference's host engine in the same run.

    python tools/bench_monitoring.py [--iters 10] [--no-reference] [--out result.json]

Workloads, on HL stacks of quarter waves at 0.55 um (2.35 / 1.46 on a 1.52 substrate) with thicknesses jittered by
up to 5 % (seeded), monitored at 0.6 um by level cut with the reference's defaults (600 grid points, max_factor 1.8):
- `simulate_run_<L>` (L = 20, 40): one run, end to end on the host clock (it copies the N as-built thicknesses back);
- `sensitivity_40`: monitoring_error_sensitivity read at 401 wavelengths (0.45-0.65 um), CUDA events;
- `choose_40`: choose_monitor_wavelength over 7 candidates (0.45-0.75 um) at 401 wavelengths, host clock (it copies
  the scores back);
- `simulate_runs_40_mc1000`: simulate_runs of 1000 seeded Monte-Carlo draws of the signal errors (sigma 5e-4),
  CUDA events;
- `ref_*`: the same calls on the reference's host engine (oracle/_ref, numpy fp64), one call each (the Monte-Carlo
  loop extrapolated from `ref_simulate_run_40`).
Each row gives seconds per call and kernel launches per call.  The card name, power limit and SM clocks are read in
the same run.
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
from benchlib import card, host_time, timed  # noqa: E402

SUB = 1.52
MON = 0.6
DESIGN = np.linspace(0.45, 0.65, 401)
CANDIDATES = [0.45, 0.5, 0.55, 0.6, 0.65, 0.7, 0.75]


def hl(L):
    n = [2.35 if i % 2 == 0 else 1.46 for i in range(L)]
    rng = np.random.default_rng(L)
    return n, np.array([0.55 / 4 / x for x in n]) * (1 + 0.05 * rng.uniform(-1, 1, L)), SUB


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--no-reference', action='store_true')
    ap.add_argument('--out')
    args = ap.parse_args()

    import torch
    import prysm_b200 as pb
    from prysm_b200 import coatings as c, _ops
    pb.config.precision = 64
    res = {'card': card(), 'workloads': {}}

    def put(name, s, n):
        row = {'s': s, 'launches': n}
        res['workloads'][name] = row
        print(json.dumps({name: row}), flush=True)

    def host_timed(fn):
        fn()
        n0 = _ops.launch_count()
        s = min(host_time(lambda: (fn(), torch.cuda.synchronize())) for _ in range(args.iters))
        return s, (_ops.launch_count() - n0) / args.iters

    for L in (20, 40):
        st = c.Stack(*hl(L))
        put(f'simulate_run_{L}', *host_timed(lambda: c.simulate_run(st, MON)))
    st = c.Stack(*hl(40))
    put('sensitivity_40', *timed(lambda: c.monitoring_error_sensitivity(st, MON, DESIGN), args.iters))
    put('choose_40', *host_timed(lambda: c.choose_monitor_wavelength(st, CANDIDATES, DESIGN)))
    se = 5e-4 * np.random.default_rng(1).standard_normal((1000, 40))
    se_dev = _ops.asdevice(se)
    put('simulate_runs_40_mc1000', *timed(lambda: c.simulate_runs(st, MON, signal_errors=se_dev), args.iters))

    if not args.no_reference and reference.installed():
        with reference.loaded(), warnings.catch_warnings():
            warnings.simplefilter('ignore')
            from prysm.conf import config
            from prysm.x.coatings import Stack, monitoring as mon
            config.precision = 64
            for L in (20, 40):
                rs = Stack(*hl(L))
                put(f'ref_simulate_run_{L}', host_time(lambda: mon.simulate_run(rs, MON)), 0)
            rs = Stack(*hl(40))
            put('ref_sensitivity_40', host_time(lambda: mon.monitoring_error_sensitivity(rs, MON, DESIGN)), 0)
            put('ref_choose_40', host_time(lambda: mon.choose_monitor_wavelength(rs, CANDIDATES, DESIGN)), 0)
            put('ref_simulate_runs_40_mc1000_extrapolated', 1000 * res['workloads']['ref_simulate_run_40']['s'], 0)
    if args.out:
        with open(args.out, 'w') as fh:
            json.dump(res, fh, indent=1)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
