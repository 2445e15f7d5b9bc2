"""Image sensors on the device (prysm_b200.detector, prysm_b200.bayer), with the reference's host path in the same run.

    python tools/bench_sensor.py [--iters 20] [--no-reference] [--out result.json]

CUDA events over `iters` calls after warm-up, each call against its byte bound (the bytes the call must move, computed
from the shapes below, over the H100 SXM data sheet's 3.35 TB/s; the bound is arithmetic, not a measurement):
- Detector.expose at 2048^2, float32 aerial image, 12-bit camera, float32 prnu and dcnu maps, frames 1 and 16, at a mean
  of 5 e- (the inversion branch) and 2e4 e- (PTRS), and with a float32 LUT.  Bytes: the image and both maps read once,
  every frame written once.  The call's one synchronisation (the error-flag read) is inside the timed window.
- demosaic_malvar at 3072 x 4096, float32 and uint16 mosaics: the mosaic read once, the float32 RGB written once.
- wb_prescale(safe=True) at 3072 x 4096 float32 (read for the maxima, then read and written) and composite_bayer
  (four planes read at the sites they contribute, the mosaic written).
The reference's numpy path (oracle/_ref) is timed once per call at the same sizes.  The card name, power limit and
current and maximum SM clocks are read in the same run.
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

N = 2048
M_RAW, N_RAW = 3072, 4096


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--no-reference', action='store_true')
    ap.add_argument('--out')
    args = ap.parse_args()
    if args.no_reference:
        return run(args, None)
    with reference.loaded():
        from prysm import bayer as rbayer, detector as rdet
        return run(args, (rdet, rbayer))


def run(args, ref):
    """Every case, each beside the reference modules' call (ref: detector, bayer) when ref is not None."""
    import torch
    import prysm_b200 as pb
    if not torch.cuda.is_available():
        raise SystemExit('bench_sensor needs a CUDA device')
    rng = np.random.default_rng(0)
    results = []

    def record(name, seconds, nbytes, ref_fn=None):
        row = dict(name=name, gpu_us=seconds * 1e6, bytes=nbytes, bound_us=nbytes / HBM_BYTES_PER_S * 1e6,
                   share_of_bound=(nbytes / HBM_BYTES_PER_S) / seconds)
        if ref_fn is not None:
            with warnings.catch_warnings():
                warnings.simplefilter('ignore')
                row['reference_host_s'] = host_time(ref_fn)
        results.append(row)
        print(json.dumps(row), flush=True)

    shape = (N, N)
    prnu = (1 + 0.01 * rng.standard_normal(shape)).astype(np.float32)
    dcnu = (1 + 0.05 * rng.standard_normal(shape)).astype(np.float32)
    lut = np.sqrt(np.arange(4096, dtype=np.float64) * 4096).astype(np.float32)
    prnu_d, dcnu_d, lut_d = pb.asdevice(prnu), pb.asdevice(dcnu), pb.asdevice(lut)
    for mean in (5.0, 2e4):
        aerial = (mean * (0.5 + rng.random(shape))).astype(np.float32)     # e-/s at t = 1 s
        aerial_d = pb.asdevice(aerial)
        for frames in (1, 16):
            for with_lut in (False, True):
                if with_lut and frames == 1:
                    continue
                cam = pb.detector.Detector(0.5, 3.0, 100, 60_000, 15.0, 12, 1.0, prnu=prnu_d, dcnu=dcnu_d,
                                           lut=lut_d if with_lut else None)
                t = timed(lambda: cam.expose(aerial_d, frames=frames), args.iters)[0]
                out_bytes = 4 if with_lut else 2
                nbytes = 3 * N * N * 4 + frames * N * N * out_bytes
                ref_fn = None
                if ref is not None:
                    rc = ref[0].Detector(0.5, 3.0, 100, 60_000, 15.0, 12, 1.0, prnu=prnu, dcnu=dcnu,
                                         lut=lut if with_lut else None)
                    ref_fn = (lambda rc=rc, f=frames, a=aerial: rc.expose(a, frames=f))
                record(f'expose_{N}^2_mean{mean:g}_frames{frames}{"_lut" if with_lut else ""}', t, nbytes, ref_fn)

    raw_f32 = (rng.random((M_RAW, N_RAW)) * 4000).astype(np.float32)
    raw_u16 = rng.integers(0, 4096, (M_RAW, N_RAW)).astype(np.uint16)
    pb.config.precision = 32
    for name, raw in (('float32', raw_f32), ('uint16', raw_u16)):
        d = pb.asdevice(raw)
        t = timed(lambda: pb.bayer.demosaic_malvar(d, 'rggb'), args.iters)[0]
        nbytes = raw.nbytes + M_RAW * N_RAW * 3 * 4
        ref_fn = None
        if ref is not None:
            ref_fn = (lambda raw=raw: ref[1].demosaic_malvar(raw, 'rggb'))
        record(f'demosaic_malvar_{M_RAW}x{N_RAW}_{name}', t, nbytes, ref_fn)
    d = pb.asdevice(raw_f32)
    t = timed(lambda: pb.bayer.wb_prescale(d, 1.0, 1.0, 1.0, 1.0, safe=True, saturation=1e9), args.iters)[0]
    record(f'wb_prescale_safe_{M_RAW}x{N_RAW}_float32', t, 3 * raw_f32.nbytes,
           None if ref is None else (lambda: ref[1].wb_prescale(raw_f32.copy(), 1.9, 1.0, 1.0, 1.6, safe=True,
                                                                 saturation=4000)))
    planes = [pb.asdevice((rng.random((M_RAW, N_RAW))).astype(np.float32)) for _ in range(4)]
    out = torch.empty((M_RAW, N_RAW), dtype=torch.float32, device=planes[0].device)
    t = timed(lambda: pb.bayer.composite_bayer(*planes, output=out), args.iters)[0]
    hp = [p.cpu().numpy() for p in planes]
    record(f'composite_bayer_{M_RAW}x{N_RAW}_float32', t, 2 * raw_f32.nbytes,
           None if ref is None else (lambda: ref[1].composite_bayer(*hp)))
    res = dict(card=card(), results=results)
    print(json.dumps(dict(card=res['card'])))
    if args.out:
        with open(args.out, 'w') as fh:
            json.dump(res, fh, indent=1)


if __name__ == '__main__':
    main()
