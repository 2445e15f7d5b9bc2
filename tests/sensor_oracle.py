"""The image-sensor cases the engine is checked on (prysm/detector.py, prysm/bayer.py) and the writer of
tests/golden/sensor*.npz.

    PYTHONDONTWRITEBYTECODE=1 python tests/sensor_oracle.py   (needs the unmodified reference: PRYSM_REFERENCE or oracle/_ref)

The fixtures are the REFERENCE's own outputs at precision 64, from the inputs `inputs()` builds with numpy.
`run(det, bayer, g, ...)` computes every deterministic case with the modules det and bayer: the reference's with numpy
arrays, or the engine's (tests/test_gpu_sensor.py).  A case that raises records the exception's class name.  The random
part of Detector.expose is not a fixture: the engine's random numbers equal the reference's in distribution only, so
tests/test_gpu_sensor.py checks it statistically.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (ROOT, os.path.join(ROOT, 'oracle')):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import reference  # noqa: E402

SHAPES = ((2, 2), (3, 5), (4, 4), (7, 9), (64, 96), (257, 130))
SMALL = SHAPES[:4]
CFAS = ('rggb', 'BGGR', 'RgGb', 'bggr')          # mixed case: every function but assemble_superresolved lower-cases
SUPERRES_SHAPES = ((8, 12), (17, 10), (32, 48))
MALVAR_LARGE = (('rggb', 'f64'), ('BGGR', 'u16'))  # the 257 x 130 demosaic cases (the others run on every shape)
WB_GAINS = (1.9, 1.05, 0.95, 1.6)


def inputs():
    """Every input array of the cases: float64 and uint16 host arrays."""
    rng = np.random.default_rng(20261016)
    g = {}
    for m, n in SHAPES:
        t = f'{m}x{n}'
        g[f'mosaic_f64_{t}'] = rng.random((m, n)) * 1000
        g[f'mosaic_u16_{t}'] = rng.integers(0, 4096, (m, n)).astype(np.uint16)
        if (m, n) in SMALL or (m, n) == (64, 96):
            for p in ('r', 'g1', 'g2', 'b'):
                g[f'plane_{p}_{t}'] = rng.random((m, n))
            g[f'rgb_{t}'] = rng.random((m, n, 3)) * 800
    for m, n in SUPERRES_SHAPES:
        for p in ('r', 'g1', 'g2', 'b'):
            g[f'sr_{p}_{m}x{n}'] = rng.random((m, n))
    x = (np.arange(-6, 7) * 0.25)[None, :]
    y = (np.arange(-5, 6) * 0.25)[:, None]
    g['pix_x'], g['pix_y'] = np.broadcast_to(x, (11, 13)).copy(), np.broadcast_to(y, (11, 13)).copy()
    g['lut_codes'] = rng.integers(0, 4096, (9, 14)).astype(np.uint16)
    g['lut_table'] = np.sqrt(np.arange(4096) * 16.0).astype(np.uint16)
    g['lut_short'] = np.arange(100, dtype=np.float64) * 0.5
    return g


def _err(fn):
    try:
        return fn()
    except Exception as exc:            # the class name is the fixture
        return np.asarray(type(exc).__name__)


def run(det, bayer, g, to_numpy=np.asarray, asarray=np.asarray):
    """Every deterministic case through the modules det (detector) and bayer."""
    out = {}

    def keep(key, fn):
        v = _err(fn)
        out[key] = v if isinstance(v, np.ndarray) and v.dtype.kind == 'U' else to_numpy(v)

    for m, n in SHAPES:
        t = f'{m}x{n}'
        for cfa in CFAS:
            for kind in ('f64', 'u16'):
                if (m, n) == (257, 130) and (cfa, kind) not in MALVAR_LARGE:
                    continue
                keep(f'malvar_{kind}_{cfa}_{t}', lambda: bayer.demosaic_malvar(asarray(g[f'mosaic_{kind}_{t}']), cfa))
            if (m, n) == (257, 130):
                continue
            for kind in ('f64', 'u16'):
                keep(f'deint_{kind}_{cfa}_{t}', lambda: bayer.demosaic_deinterlace(asarray(g[f'mosaic_{kind}_{t}']), cfa))
            planes = [asarray(g[f'plane_{p}_{t}']) for p in ('r', 'g1', 'g2', 'b')]
            keep(f'comp_{cfa}_{t}', lambda: bayer.composite_bayer(*planes, cfa=cfa))
            keep(f'recomp_{cfa}_{t}', lambda: bayer.recomposite_bayer(*planes, cfa=cfa))
            dec = bayer.decomposite_bayer(asarray(g[f'mosaic_f64_{t}']), cfa)
            for p, v in zip(('r', 'g1', 'g2', 'b'), dec):
                out[f'decomp_{p}_{cfa}_{t}'] = to_numpy(v)
            for safe in (False, True):
                def pre():
                    a = g[f'mosaic_f64_{t}'].copy()
                    bayer.wb_prescale(a, *WB_GAINS, cfa=cfa, safe=safe, saturation=(900, 1000, 1000, 800))
                    return a
                keep(f'wbpre_{int(safe)}_{cfa}_{t}', pre)
            if cfa == 'rggb':
                for safe in (False, True):
                    def post():
                        a = g[f'rgb_{t}'].copy()
                        bayer.wb_postscale(a, 1.7, 1.0, 1.4, safe=safe, saturation=(1000, 900, 1000))
                        return a
                    keep(f'wbpost_{int(safe)}_{t}', post)
    for cfa in ('grbg', 'GRBG'):
        a = g['mosaic_f64_4x4']
        pl = [g[f'plane_{p}_4x4'] for p in ('r', 'g1', 'g2', 'b')]
        keep(f'bad_malvar_{cfa}', lambda: bayer.demosaic_malvar(asarray(a), cfa))
        keep(f'bad_deint_{cfa}', lambda: bayer.demosaic_deinterlace(asarray(a), cfa))
        keep(f'bad_comp_{cfa}', lambda: bayer.composite_bayer(*[asarray(p) for p in pl], cfa=cfa))
        keep(f'bad_recomp_{cfa}', lambda: bayer.recomposite_bayer(*[asarray(p) for p in pl], cfa=cfa))
        keep(f'bad_decomp_{cfa}', lambda: bayer.decomposite_bayer(asarray(a), cfa))
        keep(f'bad_wbpre_{cfa}', lambda: bayer.wb_prescale(a.copy(), *WB_GAINS, cfa=cfa))
    for m, n in SUPERRES_SHAPES:
        t = f'{m}x{n}'
        pl = [asarray(g[f'sr_{p}_{t}']) for p in ('r', 'g1', 'g2', 'b')]
        for z in (1, 2.5):
            keep(f'superres_z{z}_{t}', lambda: bayer.assemble_superresolved(*pl, z))
    pl = [asarray(g[f'sr_{p}_8x12']) for p in ('r', 'g1', 'g2', 'b')]
    for cfa in ('bggr', 'RGGB'):
        keep(f'bad_superres_{cfa}', lambda: bayer.assemble_superresolved(*pl, 2, cfa=cfa))

    # detector: the pixel footprint (samples on its edges), lookup tables, and the reference's deterministic exposures
    for i, (wx, wy) in enumerate(((1.5, 2.0), (3.0, 0.5), (0.25, 10.0))):
        keep(f'pixel_{i}', lambda: det.pixel(asarray(g['pix_x']), asarray(g['pix_y']), wx, wy))
    keep('lut_full', lambda: det.apply_lut(asarray(g['lut_codes']), asarray(g['lut_table'])))
    keep('lut_short', lambda: det.apply_lut(asarray(g['lut_codes'] % 100), asarray(g['lut_short'])))
    keep('lut_short_overflow', lambda: det.apply_lut(asarray(g['lut_codes']), asarray(g['lut_short'])))
    keep('expose_bias', lambda: det.Detector(0, 0, 10, 60_000, 2, 12, 1).expose(asarray(np.zeros((3, 4)))))
    keep('expose_lut', lambda: det.Detector(0, 0, 3, 15, 1, 4, 1, lut=asarray(np.arange(16, dtype=np.uint8) + 10))
         .expose(asarray(np.zeros((1, 2)))))
    keep('expose_saturation', lambda: det.Detector(0, 0, 0, 1e9, 1, 8, 1).expose(asarray(np.full((2, 2), 1e6))))
    keep('expose_prnu_zero', lambda: det.Detector(0, 0, 0, 1e9, 1, 12, 1, prnu=asarray(np.zeros((2, 3))))
         .expose(asarray(np.ones((2, 3))), frames=4))
    keep('expose_bits33', lambda: det.Detector(0, 0, 0, 1e9, 1, 33, 1).expose(asarray(np.ones((2, 3)))))
    return out


def reference_modules():
    from prysm.conf import config
    from prysm import bayer, detector
    config.precision = 64
    return detector, bayer


def reference_outputs():
    import warnings
    with reference.loaded(), warnings.catch_warnings():
        det, bayer = reference_modules()
        warnings.simplefilter('ignore')
        np.random.seed(0)                  # the deterministic exposures still draw (zero-variance) noise
        return run(det, bayer, inputs())


def main():
    """Write tests/golden/sensor*.npz from the unmodified reference."""
    with reference.loaded():
        from make_golden import save      # imports the reference
        save('sensor.npz', reference_outputs())


if __name__ == '__main__':
    main()
