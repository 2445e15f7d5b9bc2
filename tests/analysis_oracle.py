"""The PSF / MTF analysis cases the engine is checked on (RichData slices, azimuthal statistics and exact sampling,
psf.estimate_size and its metrics, the Airy functions, diffraction_limited_mtf), and the writer of
tests/golden/analysis*.npz.

    PYTHONDONTWRITEBYTECODE=1 python tests/analysis_oracle.py   (needs the unmodified reference: PRYSM_REFERENCE
                                                                 or oracle/_ref)

Every fixture is the REFERENCE's own result at precision 64.  The inputs are stored beside them (`<case>_data`), so a
float32 run starts from the same data rounded once.  Keys:
  - `<case>_az<stat>` for stat in avg, median, min, max, var, std, pv, and `<case>_rho`, for every case of AZ_CASES;
  - `mtf_*`: the MTF of small.npz's wf_psf_intensity, its slices and statistics, and the PSF's size metrics;
  - `xy_*`, `polar_*`, `ex_*`, `ey_*`: exact sampling of the 96 x 128 case at the query points QUERIES names;
  - `size_<metric>_<criteria>`: estimate_size of the Gaussian `gauss_data`, and `gauss_fwhm`;
  - `difflim_*`, `airy_*`, `ee_*`: the analytic functions.
"""
import os
import sys
import types
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (ROOT, os.path.join(ROOT, 'oracle'), HERE):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import reference  # noqa: E402

DX = 0.5
STATS = ('avg', 'median', 'min', 'max', 'var', 'std', 'pv')
SIZE_METRICS = {'fwhm': 'fwhm', '1e': '1/e', '1e2': '1/e^2', 'abs': 0.3}
FNO, WVL = 8.0, 0.55
GAUSS_N, GAUSS_SIGMA = 256, 10.0


def az_inputs():
    """name -> (data, dx) of the azimuthal-statistics cases"""
    rng = np.random.default_rng(2024)
    out = {'odd11': (rng.standard_normal((11, 11)), DX),
           'odd255': (rng.random((255, 255)), DX),
           'rect96x128': (rng.random((96, 128)), DX)}
    d = rng.random((64, 64))
    y, x = np.mgrid[-32:32, -32:32]
    d[np.hypot(x - 5, y + 3) < 9] = np.nan                        # a NaN disk off centre
    out['nan_disk'] = (d, DX)
    d = rng.random((64, 64))
    d[rng.random((64, 64)) < 0.03] = np.nan                       # NaN nodes, some next to lattice points on nodes
    d[32, 35] = d[31, 32] = np.nan
    out['nan_nodes'] = (d, DX)
    d = rng.random((33, 48))
    d[16, 24] = np.nan                                            # the centre node: the rho = 0 column is all NaN
    out['nan_column'] = (d, DX)
    return out


def queries(shape, dx):
    """exact_* query points of the (ny, nx) grid fftrange * dx: interior nodes, lower and upper edges, between nodes,
    scalars and arrays"""
    ny, nx = shape
    x = (np.arange(nx) - nx // 2) * dx
    y = (np.arange(ny) - ny // 2) * dx
    xs = np.array([x[0], x[3], x[nx // 2], x[-1], 0.3 * dx + x[5], x[-2] + 0.75 * dx])
    ys = np.array([y[0], y[ny - 4], y[ny // 2], y[-1], y[7] + 0.125 * dx, y[1] + 0.5 * dx])
    rho = np.array([0.0, 1.3 * dx, 7.0 * dx, min(-x[0], x[-1], -y[0], y[-1]) - dx])
    phi = np.array([0.0, 0.4, np.pi / 2, 3.0])
    return {'xs': xs, 'ys': ys, 'rho': rho, 'phi': phi, 'x_scalar': float(x[-1]), 'y_scalar': float(y[0]),
            'rho_scalar': 2.5 * dx}


def gauss():
    x = (np.arange(GAUSS_N) - GAUSS_N // 2) * 1.0
    xx, yy = np.meshgrid(x, x)
    return np.exp(-(xx ** 2 + yy ** 2) / (2 * GAUSS_SIGMA ** 2))


def analytic_inputs():
    ext = 1 / (WVL / 1000 * FNO)
    return {'freqs': np.array([0.0, 0.1 * ext, 0.5 * ext, 0.999 * ext, ext, 1.5 * ext, -0.3 * ext]),
            'freq_scalar': 0.25 * ext, 'freq_above': 2.0 * ext,
            'airy_r': np.array([0.0, 1e-10, 0.5, 1.0, WVL * FNO * 1.22, 7.3, 20.0]),
            'airy_ft_r': np.array([0.0, 0.05, 0.1, 1 / (WVL * FNO), 0.5]),
            'ee_r': np.array([0.0, 0.5, 1.0, 5.0, 20.0])}


def reference_modules():
    from prysm.conf import config
    from prysm import psf, otf, _richdata
    config.precision = 64
    return types.SimpleNamespace(psf=psf, otf=otf, RichData=_richdata.RichData)


def _stats(sl):
    return {s: getattr(sl, 'az' + s)[1] for s in STATS}


def run(m, small):
    out = {}
    for name, (d, dx) in az_inputs().items():
        rd = m.RichData(d, dx, None)
        sl = rd.slices()
        out[f'{name}_data'] = d
        for s, v in _stats(sl).items():
            out[f'{name}_az{s}'] = v
        out[f'{name}_rho'] = sl.azavg[0]
    # the MTF of the small focus case, its slices and statistics, and the PSF's size metrics
    psf = small['wf_psf_intensity']
    mtf = m.otf.mtf_from_psf(psf, dx=float(small['wf_psf_dx']))
    sl = mtf.slices()
    out['mtf_data'] = mtf.data
    out['mtf_df'] = mtf.dx
    out['mtf_slice_x'], out['mtf_slice_y'] = sl.x[1], sl.y[1]
    one = mtf.slices(twosided=False)
    out['mtf_slice_x1_u'], out['mtf_slice_x1'] = one.x
    out['mtf_slice_y1_u'], out['mtf_slice_y1'] = one.y
    for s, v in _stats(sl).items():
        out[f'mtf_az{s}'] = v
    out['mtf_rho'] = sl.azavg[0]
    out['mtf_fwhm'] = m.psf.fwhm(psf, float(small['wf_psf_dx']))
    # exact sampling of the 96 x 128 case
    d, dx = az_inputs()['rect96x128']
    rd = m.RichData(d, dx, None)
    q = queries(d.shape, dx)
    out['xy_array'] = rd.exact_xy(q['xs'], q['ys'])
    out['xy_scalar'] = rd.exact_xy(q['x_scalar'], q['y_scalar'])
    out['xy_broadcast'] = rd.exact_xy(q['xs'], q['y_scalar'])
    out['polar_array'] = rd.exact_polar(q['rho'], q['phi'])
    out['polar_scalar'] = rd.exact_polar(q['rho_scalar'])
    out['ex_array'] = rd.exact_x(q['xs'])
    out['ex_scalar'] = rd.exact_x(q['x_scalar'])
    out['ey_array'] = rd.exact_y(q['ys'])
    out['ey_scalar'] = rd.exact_y(q['y_scalar'])
    # estimate_size
    g = gauss()
    out['gauss_data'] = g
    for key, metric in SIZE_METRICS.items():
        for crit in ('first', 'last'):
            out[f'size_{key}_{crit}'] = m.psf.estimate_size(g, metric, dx=1.0, criteria=crit)
    out['gauss_fwhm'] = m.psf.fwhm(g, 1.0)
    # analytic functions
    a = analytic_inputs()
    out['difflim_array'] = m.otf.diffraction_limited_mtf(FNO, WVL, a['freqs'].copy())
    out['difflim_scalar'] = m.otf.diffraction_limited_mtf(FNO, WVL, a['freq_scalar'])
    out['difflim_above'] = m.otf.diffraction_limited_mtf(FNO, WVL, a['freq_above'])
    out['difflim_none_f'], out['difflim_none'] = m.otf.diffraction_limited_mtf(FNO, WVL, samples=64)
    out['airy'] = m.psf.airydisk(a['airy_r'], FNO, WVL)
    out['airy_efield'] = m.psf.airydisk_efield(a['airy_r'], FNO, WVL)
    out['airy_ft'] = m.psf.airydisk_ft(a['airy_ft_r'].copy(), FNO, WVL)
    out['ee'] = m.otf.analytical_encircled_energy_circular_aperture(FNO, WVL, a['ee_r'])
    return {k: np.asarray(v) for k, v in out.items()}


def reference_outputs():
    from conftest import load_golden
    small = load_golden('small.npz')
    with reference.loaded(), warnings.catch_warnings():
        warnings.simplefilter('ignore')
        return run(reference_modules(), small)


def main():
    """Write tests/golden/analysis*.npz from the unmodified reference."""
    with reference.loaded():
        from make_golden import save      # imports the reference
        save('analysis.npz', reference_outputs())


if __name__ == '__main__':
    main()
