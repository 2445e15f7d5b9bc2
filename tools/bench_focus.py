"""Kernel-level timing of the batched focus pipeline at the benchmark's shape, one package tree per subprocess.

    python tools/bench_focus.py [--trees DIR ...] [--alternate N] [--intensity | --screen] [--profile DIR] [--out FILE.json]

Each DIR is the root of a built checkout (default: this one); its `prysm_b200` is imported in a process of its own, so
that two builds, e.g. a change and its parent, can be compared in one session.  Each run times `propagation.focus`
(and, with --intensity, `propagation.focus_intensity`) on a (16, 2048, 2048) complex64 stack -> 4096^2 with CUDA
events over a window of at least 0.5 s, and reports microseconds per propagation, the algorithmic bandwidth (pupil read
+ field written) and the HBM bytes the pipeline moves, counted from the shapes.  --alternate N runs the tree list N
times in turn (A/B/A/B...), so that drifts of the card show as spread.  --profile DIR writes torch.profiler kernel
times of one call per tree under DIR.  --screen times the inputs the focus pair stages first instead, microseconds per
call: `propagation.psf_from_amp_and_phase` with a bool amplitude at N = 512, 1024 and 2048, as a complex field and as a
weighted |.|^2 accumulate (the per-wavelength step of `polychromatic_psf_fft`), and `propagation.focus` of a 2048^2
complex64 input whose base is 8 bytes off 16-byte alignment.  The card's name, power limit and SM clock are printed with
the numbers (read-only nvidia-smi queries).
"""
import argparse
import json
import os
import subprocess
import sys

from benchlib import card

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N, Q, BATCH = 2048, 2, 16
K = N * Q
MIB = 2 ** 20
ALG = {'complex': 8 * N * N + 8 * K * K, 'intensity': 8 * N * N + 4 * K * K}
# HBM bytes per propagation counted from the shapes: pupil reads, plane 1 of the 16 N^2-byte intermediate but for its
# first KEEP1 bytes (written and read back; plane 0 and those bytes stay in L2, kPlane1KeepBytes in csrc/fft_tuned.cu),
# output writes
KEEP1 = 2 * MIB
HBM = {'complex': 8 * N * N + 2 * (8 * N * N - KEEP1) + 8 * K * K, 'intensity': 8 * N * N + 2 * (8 * N * N - KEEP1) + 4 * K * K}

_CHILD = r'''
import json, sys, time
import torch
sys.path.insert(0, %(root)r)
import prysm_b200 as pb
from prysm_b200 import propagation as P, _ops
pb.config.precision = 32
N, Q, B = %(n)d, %(q)d, %(b)d
gen = torch.Generator(device='cuda').manual_seed(5)
stack = torch.complex(torch.randn((B, N, N), generator=gen, device='cuda'), torch.randn((B, N, N), generator=gen, device='cuda'))
res = {}
kinds = ['complex'] + (['intensity'] if %(intensity)r else [])
for kind in kinds:
    fn = (lambda: P.focus(stack, Q)) if kind == 'complex' else (lambda: P.focus_intensity(stack, Q))
    for _ in range(3):
        out = fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); out = fn(); e1.record(); torch.cuda.synchronize()
    reps = max(4, int(0.6e3 / max(e0.elapsed_time(e1), 1e-3)) + 1)   # a window of >= 0.5 s
    l0 = _ops.launch_count()
    e0.record()
    for _ in range(reps):
        out = fn()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    res[kind] = {'us_per_prop': ms * 1e3 / (reps * B), 'window_ms': ms, 'calls': reps,
                 'launches_per_call': (_ops.launch_count() - l0) / reps}
    del out
    if %(profile)r:
        from torch.profiler import profile, ProfilerActivity
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn(); torch.cuda.synchronize()
        kt = {}
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                kt.setdefault(ev.name, []).append(ev.device_time_total if hasattr(ev, 'device_time_total') else ev.cuda_time_total)
        res[kind]['kernels_us'] = {k: {'count': len(v), 'total': sum(v), 'mean': sum(v) / len(v)} for k, v in kt.items()}
print('RESULT', json.dumps(res))
'''

_SCREEN_CHILD = r'''
import json, sys
import torch
sys.path.insert(0, %(root)r)
import prysm_b200 as pb
from prysm_b200 import propagation as P, _ops
pb.config.precision = 32
gen = torch.Generator(device='cuda').manual_seed(5)
cases = {}
for n in (512, 1024, 2048):
    mask = torch.rand((n, n), generator=gen, device='cuda') > 0.3
    opd = torch.randn((n, n), generator=gen, device='cuda') * 60.0
    acc = torch.zeros((2 * n, 2 * n), device='cuda')
    cases[f'screen_field/{n}'] = lambda m=mask, o=opd: P.psf_from_amp_and_phase(m, o, 0.6328, 2, field=True)
    cases[f'screen_accumulate/{n}'] = lambda m=mask, o=opd, a=acc: P.psf_from_amp_and_phase(m, o, 0.6328, 2, weight=0.5, out=a)
flat = torch.randn(2048 * 2048 + 1, dtype=torch.complex64, generator=gen, device='cuda')
misaligned = flat[1:].view(2048, 2048)
assert misaligned.data_ptr() %% 16 == 8
cases['misaligned_focus/2048'] = lambda: P.focus(misaligned, 2)
res = {}
for name, fn in cases.items():
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); fn(); e1.record(); torch.cuda.synchronize()
    reps = max(4, int(0.6e3 / max(e0.elapsed_time(e1), 1e-3)) + 1)   # a window of >= 0.5 s
    l0 = _ops.launch_count()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    res[name] = {'us_per_call': ms * 1e3 / reps, 'window_ms': ms, 'calls': reps,
                 'launches_per_call': (_ops.launch_count() - l0) / reps}
print('RESULT', json.dumps(res))
'''


def run_child(root, src):
    r = subprocess.run([sys.executable, '-c', src], capture_output=True, text=True, timeout=900)
    if r.returncode != 0:
        raise RuntimeError(f'{root}: exit {r.returncode}\n{r.stderr[-3000:]}')
    return json.loads([ln for ln in r.stdout.splitlines() if ln.startswith('RESULT ')][-1][7:])


def run_tree(root, intensity, profile):
    res = run_child(root, _CHILD % {'root': root, 'n': N, 'q': Q, 'b': BATCH, 'intensity': intensity, 'profile': bool(profile)})
    for kind, row in res.items():
        us = row['us_per_prop']
        row['alg_gbs'] = ALG[kind] / (us * 1e-6) / 1e9
        row['hbm_mib_counted'] = HBM[kind] / MIB
        row['hbm_gbs_counted'] = HBM[kind] / (us * 1e-6) / 1e9
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--trees', nargs='+', default=[ROOT], metavar='DIR', help='roots of built checkouts to time')
    ap.add_argument('--alternate', type=int, default=1, metavar='N', help='run the tree list N times in turn')
    ap.add_argument('--intensity', action='store_true', help='time focus_intensity (the fused PSF variant) too')
    ap.add_argument('--screen', action='store_true', help='time the staged inputs (phase screen, misaligned) instead')
    ap.add_argument('--profile', default=None, metavar='DIR', help='write torch.profiler kernel times under DIR')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    trees = [os.path.abspath(t) for t in args.trees]
    print('card (name, power limit, SM clock, max SM clock):', card(), flush=True)
    if args.screen:
        return screen(trees, args)
    runs = []
    for rnd in range(args.alternate):
        for i, tree in enumerate(trees):
            res = run_tree(tree, args.intensity, args.profile)
            runs.append({'round': rnd, 'tree': tree, **res})
            line = f'[{rnd}] {tree:32s}'
            for kind, row in res.items():
                line += (f'  {kind}: {row["us_per_prop"]:7.1f} us/prop  {row["alg_gbs"]:6.0f} GB/s alg  '
                         f'HBM {row["hbm_mib_counted"]:.0f} MiB  {row["launches_per_call"]:.0f} launches/call')
            print(line, flush=True)
            if args.profile:
                os.makedirs(args.profile, exist_ok=True)
                with open(os.path.join(args.profile, f'kernels_tree{i}_{rnd}.json'), 'w') as fh:
                    json.dump({'tree': tree, **res}, fh, indent=1)
    print('card after:', card(), flush=True)
    summary = {}
    for tree in trees:
        for kind in ('complex', 'intensity'):
            xs = [r[kind]['us_per_prop'] for r in runs if r['tree'] == tree and kind in r]
            if xs:
                summary[f'{tree} {kind}'] = {'min': min(xs), 'max': max(xs), 'spread_pct': 100 * (max(xs) - min(xs)) / min(xs)}
    for k, s in summary.items():
        print(f'{k:44s} min {s["min"]:7.1f}  max {s["max"]:7.1f} us/prop  spread {s["spread_pct"]:.1f} %')
    if args.out:
        with open(args.out, 'w') as fh:
            json.dump({'card': card(), 'runs': runs, 'summary': summary}, fh, indent=1)


def screen(trees, args):
    runs = []
    for rnd in range(args.alternate):
        for tree in trees:
            res = run_child(tree, _SCREEN_CHILD % {'root': tree})
            runs.append({'round': rnd, 'tree': tree, **res})
            print(f'[{rnd}] {tree}', flush=True)
            for name, row in res.items():
                print(f'    {name:24s} {row["us_per_call"]:8.1f} us/call  {row["launches_per_call"]:.0f} launches/call', flush=True)
    print('card after:', card(), flush=True)
    summary = {}
    for tree in trees:
        for name in (k for k in runs[0] if k not in ('round', 'tree')):
            xs = [r[name]['us_per_call'] for r in runs if r['tree'] == tree and name in r]
            if xs:
                summary[f'{tree} {name}'] = {'min': min(xs), 'max': max(xs), 'spread_pct': 100 * (max(xs) - min(xs)) / min(xs)}
    for k, s in summary.items():
        print(f'{k:60s} min {s["min"]:8.1f}  max {s["max"]:8.1f} us/call  spread {s["spread_pct"]:.1f} %')
    if args.out:
        with open(args.out, 'w') as fh:
            json.dump({'card': card(), 'runs': runs, 'summary': summary}, fh, indent=1)


if __name__ == '__main__':
    main()
