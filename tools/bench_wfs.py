"""Wavefront sensing on the device (prysm_b200.fibers, .sri, .pdi, .psi), with the reference's host path in the same run.

    python tools/bench_wfs.py [--iters 20] [--no-reference] [--out result.json]

At precision 32, with CUDA events over `iters` calls after warm-up:
- SRI forward_model, 1024^2 pupil -> 256^2 fiber;
- PS/PDI forward_model at 1024^2 (sin_amp grating, default arms);
- compute_LP_modes and multimode_coupling at V = 20 on 256^2 (105 modes);
- PSI (degroot_formalism_psi) of 13 frames at 2048^2, float32 and uint16 frames, against its byte bound: the frames
  read once and the phase written once, over the H100 SXM data sheet's 3.35 TB/s.  (The bound is arithmetic, not a
  measurement.)
The reference's numpy path (oracle/_ref, fp64 as it runs by default) is timed once per call at the same sizes.  The
card name, power limit and current SM clock are read in the same run.
"""
import argparse
import json
import os
import sys
import types
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'oracle')]
import reference  # noqa: E402
from benchlib import HBM_BYTES_PER_S, card, host_time, timed  # noqa: E402


def cases(m, xp, asarray):
    """The benchmark calls for the modules of m (engine or reference), as {name: callable}."""
    n = 1024
    x = (np.arange(n) - n // 2) * (8.0 / n)
    xx, yy = np.meshgrid(x, x)
    r = np.hypot(xx, yy)
    pupil = asarray((r <= 4).astype(np.float64) * np.exp(1j * 0.3 * (xx * yy) / 16))
    gx, gy = asarray(xx), asarray(yy)
    sri = m.sri.SelfReferencedInterferometer(gx, gy, 16.0, 8.0, 0.55, fiber_a=0.96, fiber_samples=256)
    pdi = m.pdi.PSPDI(gx, gy, 80.0, 8.0, 0.55, test_arm_transmissivity=0.7)
    nf = 256
    f = (np.arange(nf) - nf // 2) * 0.09375
    fx, fy = np.meshgrid(f, f)
    rf, tf = asarray(np.hypot(fx, fy)), asarray(np.arctan2(fy, fx))
    md = m.fibers.find_all_modes(20)
    modes = m.fibers.compute_LP_modes(20, md, 6.0, rf, tf)
    E = asarray(np.exp(-(np.hypot(fx, fy) / 5) ** 2) * np.exp(1j * 0.2 * fx))
    N = 2048
    rng = np.random.default_rng(5)
    frames32 = [asarray(rng.random((N, N), dtype=np.float32)) for _ in range(13)]
    frames16 = [asarray(rng.integers(0, 4096, (N, N), dtype=np.uint16)) for _ in range(13)]
    Z = m.psi.ZYGO_THIRTEEN_FRAME
    return {
        'sri_forward_1024_to_256': lambda: sri.forward_model(pupil, phase_shift=np.pi / 2),
        'pdi_forward_1024': lambda: pdi.forward_model(pupil, phase_shift=np.pi / 3),
        'compute_LP_modes_V20_256': lambda: m.fibers.compute_LP_modes(20, md, 6.0, rf, tf),
        'multimode_coupling_V20_256': lambda: m.fibers.multimode_coupling(E, modes),
        'psi13_2048_f32': lambda: m.psi.degroot_formalism_psi(frames32, Z),
        'psi13_2048_u16': lambda: m.psi.degroot_formalism_psi(frames16, Z),
    }, sum(len(v) for v in md.values())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--no-reference', action='store_true')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import prysm_b200 as pb
    pb.config.precision = 32
    eng = types.SimpleNamespace(fibers=pb.fibers, sri=pb.sri, pdi=pb.pdi, psi=pb.psi)
    calls, nmodes = cases(eng, None, pb.asdevice)
    res = {'card': card(), 'precision': 32, 'iters': args.iters, 'modes_V20': nmodes, 'engine_us': {}, 'reference_us': {}}
    for k, fn in calls.items():
        res['engine_us'][k] = timed(fn, args.iters, warm=1)[0] * 1e6
    N = 2048
    for k, nbytes in (('psi13_2048_f32', 13 * N * N * 4 + N * N * 4), ('psi13_2048_u16', 13 * N * N * 2 + N * N * 8)):
        bound = nbytes / HBM_BYTES_PER_S * 1e6
        res[f'{k}_bytes'] = nbytes
        res[f'{k}_bound_us'] = bound
        res[f'{k}_fraction_of_bound'] = bound / res['engine_us'][k]
    res['modes_V20_fp32_bytes'] = nmodes * 256 * 256 * 4
    del calls
    if not args.no_reference:
        sys.path.insert(0, os.path.join(ROOT, 'tests'))
        import wfs_oracle as O
        with reference.loaded(also=('skimage',)), warnings.catch_warnings():
            m = O.reference_modules()
            warnings.simplefilter('ignore')
            ref_calls, _ = cases(m, np, np.asarray)
            for k, fn in ref_calls.items():
                res['reference_us'][k] = host_time(fn) * 1e6
        res['speedup'] = {k: res['reference_us'][k] / res['engine_us'][k] for k in res['reference_us']}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as fh:
            fh.write(line + '\n')


if __name__ == '__main__':
    main()
