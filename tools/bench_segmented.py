"""Segmented apertures on the device: constructor, prepare_opd_bases, compose_opd and compose_opd_adjoint of
prysm_b200.segmented.CompositeHexagonalAperture, with the reference on the host in the same run.

    python tools/bench_segmented.py [--iters 200] [--precision 32] [--no-reference] [--out result.json]

Cases: JWST at 512^2 (18 segments), LUVOIR-A at 2048^2 (120 segments), and a TMT-like 1024^2 aperture of 492
segments (13 rings, the 492 segments nearest the centre, centre excluded), each with an 11-term Zernike basis per
segment.  compose_opd / compose_opd_adjoint are timed with CUDA events over `iters` calls after warm-up, with the
coefficients / gradient already on the device.  Their algorithmic bytes are the OPD written (and read: it is
accumulated into), plus every segment's mask and every unique basis read once; the reference's time is one host call.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'oracle')]
import reference  # noqa: E402
from benchlib import HBM_BYTES_PER_S, card, timed  # noqa: E402

NMS = [(0, 0), (1, 1), (1, -1), (2, 0), (2, -2), (2, 2), (3, -1), (3, 1), (3, -3), (3, 3), (4, 0)]
L2_BYTES = 50 * 2 ** 20


def tmt_exclude(rings, keep):
    from prysm_b200.segmented import hex_ring, hex_to_xy
    cells = [(0, 0, 0)] + [c for k in range(1, rings + 1) for c in hex_ring(k)]
    r = np.array([np.hypot(*hex_to_xy(c, 1.0)) for c in cells])
    order = np.argsort(r, kind='stable')
    return tuple(int(i) for i in order[keep + 1:]) + (0,)


CASES = {   # name -> (n, diameter, rings, segment flat-to-flat, gap, exclude)
    'jwst512': (512, 6.6, 2, 1.32, 0.007, (0,)),
    'luvoira2048': (2048, 15.0, 6, 1.223, 0.007, (0, 91, 109, 97, 103, 115, 121)),
    'tmt1024': (1024, 30.0, 13, 1.44 / 1.1547005383792515, 0.0025, None),
}


def run_case(name, iters, precision, with_reference):
    import torch
    import prysm_b200 as pb
    n, diameter, rings, diam, gap, exclude = CASES[name]
    if exclude is None:
        exclude = tmt_exclude(rings, 492)
    pb.config.precision = precision
    x, y = pb.coordinates.make_xy_grid(n, diameter=diameter)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    cha = pb.segmented.CompositeHexagonalAperture(x, y, rings, diam, gap, exclude=exclude)
    torch.cuda.synchronize()
    t_ctor = time.perf_counter() - t0
    t0 = time.perf_counter()
    cha.prepare_opd_bases(pb.polynomials.zernike_nm_seq, NMS)
    torch.cuda.synchronize()
    t_prep = time.perf_counter() - t0
    nseg = len(cha.windows)
    c = pb.asdevice(np.random.default_rng(1).standard_normal((nseg, len(NMS))) * 1e-2)
    out = torch.zeros_like(cha.x)
    g = torch.randn_like(cha.x)
    us_fwd = timed(lambda: cha.compose_opd(c, out=out), iters, warm=5)[0] * 1e6
    us_adj = timed(lambda: cha.compose_opd_adjoint(g), iters, warm=5)[0] * 1e6
    esize = cha.x.element_size()
    nunique = len({b.data_ptr() for b in cha.opd_bases})
    base_bytes = cha._bases.numel() * esize
    mask_bytes = sum(m.numel() for m in cha.local_masks) * esize
    fwd_bytes = 2 * n * n * esize + base_bytes + mask_bytes
    adj_bytes = n * n * esize + base_bytes + mask_bytes
    res = dict(case=name, precision=precision, segments=nseg, unique_grids=nunique, window=list(cha.local_masks[0].shape),
               constructor_s=t_ctor, prepare_opd_bases_s=t_prep, compose_opd_us=us_fwd, compose_opd_adjoint_us=us_adj,
               bases_MiB=base_bytes / 2 ** 20, bases_fit_in_L2=base_bytes <= L2_BYTES,
               compose_bytes=fwd_bytes, compose_GBps=fwd_bytes / us_fwd / 1e3,
               compose_hbm_bound_us=fwd_bytes / HBM_BYTES_PER_S * 1e6, adjoint_GBps=adj_bytes / us_adj / 1e3,
               bound='memory (bytes / HBM bandwidth; under 1 flop per byte)')
    if with_reference:
        with reference.loaded():
            from prysm.conf import config
            from prysm import segmented as S, polynomials as P, coordinates as C
            config.precision = precision
            xr, yr = C.make_xy_grid(n, diameter=diameter)
            t0 = time.perf_counter()
            rc = S.CompositeHexagonalAperture(xr, yr, rings, diam, gap, exclude=exclude)
            res['reference_constructor_s'] = time.perf_counter() - t0
            t0 = time.perf_counter()
            rc.prepare_opd_bases(P.zernike_nm_seq, NMS)
            res['reference_prepare_opd_bases_s'] = time.perf_counter() - t0
            ch = c.cpu().numpy()
            rc.compose_opd(ch)
            t0 = time.perf_counter()
            for _ in range(3):
                rc.compose_opd(ch)
            res['reference_compose_opd_ms'] = (time.perf_counter() - t0) / 3 * 1e3
    pb.config.precision = 64
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=200)
    ap.add_argument('--precision', type=int, default=32)
    ap.add_argument('--no-reference', action='store_true')
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('bench_segmented needs a CUDA device')
    result = {'card': card(), 'cases': [run_case(k, a.iters, a.precision, not a.no_reference) for k in CASES]}
    for r in result['cases']:
        print(json.dumps(r))
    print(json.dumps({'card': result['card']}))
    if a.out:
        with open(a.out, 'w') as fh:
            json.dump(result, fh, indent=1)


if __name__ == '__main__':
    main()
