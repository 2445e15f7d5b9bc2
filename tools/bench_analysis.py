"""PSF / MTF analysis on the device (RichData slices, psf.fwhm, exact_polar), with the reference's host time for the same
call in the same run.

    python tools/bench_analysis.py [--iters 20] [--no-reference] [--out result.json]

CUDA events over `iters` calls after warm-up, at 2048^2 and 4096^2, fp32 and fp64 data (an MTF of a Gaussian PSF with 5 %
multiplicative noise):
- all azimuthal statistics (count, mean, var, min, max and median: one launch) and azavg alone (count, mean, var, min,
  max: the first-read launch);
- psf.fwhm (four launches; the call waits for the two numbers it returns);
- exact_polar at 10^4 points.
Each 2-D reduction is set against its read-once floor: the data (4 N^2 or 8 N^2 bytes) over the H100 SXM data sheet's
3.35 TB/s.  The lattice reads every sample about four times through L2 and along circles, so the floor is a bound, not
a prediction.  The card name, power limit and SM clocks are read in the same run.  The reference (oracle/_ref) is timed
once per size on the host at fp64.
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

SIZES = (2048, 4096)
NPOINTS = 10_000


def psf_of(n):
    rng = np.random.default_rng(1)
    x = np.arange(n) - n // 2
    r2 = x[None, :] ** 2 + x[:, None] ** 2
    return np.exp(-r2 / (2 * (n / 64) ** 2)) * (1 + 0.05 * rng.random((n, n)))


def polar_points(n):
    """10^4 points inside the MTF's frequency grid (df = 1000 / n cy/mm for a PSF sampled at 1 um)"""
    rng = np.random.default_rng(2)
    return rng.random(NPOINTS) * (n // 2 - 2) * (1000 / n), rng.random(NPOINTS) * 2 * np.pi


def reference_times(n, psf):
    if not reference.installed():
        return None
    with reference.loaded(), warnings.catch_warnings():
        warnings.simplefilter('ignore')
        from prysm.conf import config
        from prysm import otf, psf as ppsf
        config.precision = 64
        mtf = otf.mtf_from_psf(psf, 1.0)
        rho, phi = polar_points(n)
        out = {'azavg_s': host_time(lambda: mtf.slices().azavg)}
        sl = mtf.slices()
        sl.azavg
        out['then_azmedian_s'] = host_time(lambda: sl.azmedian)
        out['fwhm_s'] = host_time(lambda: ppsf.fwhm(psf, 1.0))
        out['exact_polar_1e4_s'] = host_time(lambda: mtf.exact_polar(rho, phi))
        return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--no-reference', action='store_true')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()

    import torch
    import prysm_b200 as pb
    from prysm_b200 import _capi, _ops

    res = {'card': card(), 'sizes': {}}
    for n in SIZES:
        psf = psf_of(n)
        row = {}
        for rdt, tag in ((torch.float32, 'fp32'), (torch.float64, 'fp64')):
            mtf = pb.otf.mtf_from_psf(pb.asdevice(psf).to(rdt), 1.0)
            sl = mtf.slices()
            xd, yd, rmax = sl._lattice()
            data = sl._source = mtf.data.contiguous()
            floor = data.numel() * data.element_size() / HBM_BYTES_PER_S
            t_all = timed(lambda: _ops.azimuthal_stats(data, xd, yd, rmax, _capi.AZ_ALL), args.iters)[0]
            stats = _capi.AZ_COUNT | _capi.AZ_MEAN | _capi.AZ_VAR | _capi.AZ_MIN | _capi.AZ_MAX
            t_avg = timed(lambda: _ops.azimuthal_stats(data, xd, yd, rmax, stats), args.iters)[0]
            t_fwhm = timed(lambda: pb.psf.fwhm(data, 1.0), args.iters)[0]
            rho, phi = polar_points(n)
            t_pol = timed(lambda: mtf.exact_polar(rho, phi), args.iters)[0]
            row[tag] = {'read_once_floor_s': floor,
                        'all_stats_s': t_all, 'all_stats_floor_fraction': floor / t_all,
                        'azavg_s': t_avg, 'azavg_floor_fraction': floor / t_avg,
                        'fwhm_s': t_fwhm, 'fwhm_floor_fraction': floor / t_fwhm,
                        'exact_polar_1e4_s': t_pol}
        if not args.no_reference:
            row['reference_host_fp64'] = reference_times(n, psf)
        res['sizes'][f'{n}^2'] = row
        print(json.dumps({f'{n}^2': row}), flush=True)
    if args.out:
        with open(args.out, 'w') as fh:
            json.dump(res, fh, indent=1)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
