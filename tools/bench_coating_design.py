"""Coating design on the device (prysm_b200.coatings merit terms and needle_function), with the reference's host
design loop in the same run.

    python tools/bench_coating_design.py [--iters 10] [--rounds 3] [--no-reference] [--out result.json]

Workloads, on HL stacks of 20 and 40 layers (2.35 / 1.46 quarter-waves at 0.55 um on a 1.52 substrate):
- `vg_avg_<L>`: Reflectance(target=0.5, pol='avg').value_and_grad on 2001 wavelengths (0.4-0.8 um) x 61 angles
  (0-60 deg), the fused path: two launches and one copy of the value;
- `fwd_grad_sp_<L>`: what it replaces, forward_eval + thickness_gradient for s and then p on the same grid;
  the two are timed alternately, `rounds` times each, and the median is kept;
- `needle_avg_<L>` / `needle_s2001_<L>`: needle_function over 240 depths on that grid (avg) and on the 2001-sample
  s-polarised term at normal incidence;
- `refine_<L>`: the reference's own refine(maxiter=50) on the 2001-sample s-polarised term after
  set_backend_to_b200(), end to end on the host clock, and the same call on the reference's host engine
  (oracle/_ref, fp64) in the same run.
CUDA events over `iters` calls after warm-up, the fp64 chain at fp64 storage.  The card name, power limit and SM
clocks are read in the same run.
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
LAYERS = (20, 40)


def hl(L):
    n = [2.35 if i % 2 == 0 else 1.46 for i in range(L)]
    return n, [0.55 / 4 / x for x in n], SUB


def grid():
    return np.linspace(0.4, 0.8, 2001)[:, None], np.radians(np.linspace(0, 60, 61))[None, :]


def refine_times(L, iters):
    """(device, host) seconds of the reference's refine(maxiter=50) on the 2001-sample s-polarised term."""
    if not reference.installed():
        return None
    import torch
    import prysm_b200 as pb
    with reference.loaded(), warnings.catch_warnings():
        warnings.simplefilter('ignore')
        from prysm.conf import config
        config.precision = 64
        from prysm.x import coatings as rc
        w = np.linspace(0.4, 0.8, 2001)

        def run():
            st = rc.Stack(*hl(L))
            return rc.refine(st, rc.Reflectance(w, pol='s', target=0.5), maxiter=50)
        pb.mathops.set_backend_to_b200()
        try:
            run()
            torch.cuda.synchronize()
            dev = min(host_time(lambda: (run(), torch.cuda.synchronize())) for _ in range(iters))
            nit = run().nit
        finally:
            pb.mathops.set_backend_to_defaults()
        host = host_time(run)
        return {'device_s': dev, 'host_s': host, 'nit': nit}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--no-reference', action='store_true')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()

    import torch
    from prysm_b200 import coatings as c

    res = {'card': card(), 'workloads': {}}

    def record(name, row):
        res['workloads'][name] = row
        print(json.dumps({name: row}), flush=True)

    w, t = grid()
    for L in LAYERS:
        st = c.Stack(*hl(L))
        term = c.Reflectance(w, theta=t, target=0.5, pol='avg')

        def fused():
            return term.value_and_grad(st)

        def unfused():
            for pol in 'sp':
                f = c.forward_eval(st, w, t, pol)
                c.thickness_gradient(f, dR=1.0)
        runs = {'vg_avg': [], 'fwd_grad_sp': []}
        for _ in range(args.rounds):
            runs['vg_avg'].append(timed(fused, args.iters))
            runs['fwd_grad_sp'].append(timed(unfused, args.iters))
        for k, v in runs.items():
            s = sorted(x[0] for x in v)
            record(f'{k}_{L}', {'s': s[len(s) // 2], 'all_s': s, 'launches': v[0][1]})
        torch.cuda.empty_cache()
        z = np.linspace(0.0, float(np.sum(st.thicknesses)), 240)
        s, n = timed(lambda: c.needle_function(st, term, 1.38, z), args.iters)
        record(f'needle_avg_{L}', {'s': s, 'launches': n})
        term_s = c.Reflectance(np.linspace(0.4, 0.8, 2001), pol='s', target=0.5)
        s, n = timed(lambda: c.needle_function(st, term_s, 1.38, z), args.iters)
        record(f'needle_s2001_{L}', {'s': s, 'launches': n})
        if not args.no_reference:
            record(f'refine_{L}', refine_times(L, min(args.iters, 3)))
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, 'w') as fh:
            json.dump(res, fh, indent=1)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
