"""GPU: PSF / MTF analysis on the device -- RichData slices, azimuthal statistics and exact sampling, estimate_size and
its metrics, the Airy functions and diffraction_limited_mtf -- against the reference's fixtures
(tests/golden/analysis*.npz, written by tests/analysis_oracle.py) at precision 64 and 32; repeatability and launch
counts; the Lens MTF tutorial flow behind set_backend_to_b200(); and one 4096^2 MTF against the reference run on the
host."""
import warnings

import numpy as np
import pytest
import torch

from conftest import load_golden, within
from gpu_fixtures import pb  # noqa: F401
import analysis_oracle as O
import reference

pytestmark = pytest.mark.gpu

# max|engine - reference| / max|reference| over every key of a group, NaN where the reference is NaN.  Measured on an
# H100 SXM (700 W, 1980 MHz); each bound is the measured figure x 1.5 (at least 1e-15).  fp64: stats 2.2e-14 (the std
# of odd255, where a few columns have a small spread), mtf 1.5e-15, exact 0, size 1.8e-16, analytic 4.7e-16.  fp32 (the
# fixture data rounded once, then fp64 arithmetic): stats 8.5e-8, mtf 3.5e-7 (the fp32 transform of the PSF), exact
# 4.8e-8, size 2.1e-8, analytic 2.9e-8.
BOUNDS = {
    64: {'stats': 3.3e-14, 'mtf': 2.3e-15, 'exact': 1e-15, 'size': 2.7e-16, 'analytic': 7e-16},
    32: {'stats': 1.3e-7, 'mtf': 5.3e-7, 'exact': 7.2e-8, 'size': 3.2e-8, 'analytic': 4.4e-8},
}
# 4096^2 fp64 against the host reference: azavg 4.0e-15, azmedian 2.2e-16, fwhm 1.5e-16 (at least 1e-15: the host's
# own numpy sin / cos may round differently on another CPU)
BOUND_4096 = {'azavg': 6e-15, 'azmedian': 1e-15, 'fwhm': 1e-15}
# the tutorial at precision 32 on the device against precision 64 on the host: 7.5e-8 (the y slice)
BOUND_DROPIN = 1.1e-7


@pytest.fixture(scope='module')
def golden():
    return load_golden('analysis.npz')


def host(t):
    t = getattr(t, 'data', t)
    return t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)


def rel_err(got, want, key):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert got.shape == want.shape, (key, got.shape, want.shape)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), key
    if nan.all():
        return 0.0
    den = np.abs(want[~nan]).max()
    return float(np.abs(got[~nan] - want[~nan]).max() / (den if den > 0 else 1.0))


def engine_outputs(pb, golden, prec):
    """{group: {key: engine value}} for the fixture keys, inputs at precision `prec`"""
    pb.config.precision = prec
    rdt = torch.float64 if prec == 64 else torch.float32
    out = {g: {} for g in BOUNDS[prec]}
    for name, (_, dx) in O.az_inputs().items():
        rd = pb._richdata.RichData(pb.asdevice(golden[f'{name}_data']).to(rdt), dx, None)
        sl = rd.slices()
        for s in O.STATS:
            out['stats'][f'{name}_az{s}'] = host(getattr(sl, 'az' + s)[1])
        out['stats'][f'{name}_rho'] = host(sl.azavg[0])
    small = load_golden('small.npz')
    psf = pb.asdevice(small['wf_psf_intensity']).to(rdt)
    mtf = pb.otf.mtf_from_psf(psf, float(small['wf_psf_dx']))
    sl = mtf.slices()
    out['mtf']['mtf_data'] = host(mtf.data)
    out['mtf']['mtf_slice_x'], out['mtf']['mtf_slice_y'] = host(sl.x[1]), host(sl.y[1])
    one = mtf.slices(twosided=False)
    out['mtf']['mtf_slice_x1_u'], out['mtf']['mtf_slice_x1'] = host(one.x[0]), host(one.x[1])
    out['mtf']['mtf_slice_y1_u'], out['mtf']['mtf_slice_y1'] = host(one.y[0]), host(one.y[1])
    for s in O.STATS:
        out['mtf'][f'mtf_az{s}'] = host(getattr(sl, 'az' + s)[1])
    out['mtf']['mtf_rho'] = host(sl.azavg[0])
    out['size']['mtf_fwhm'] = pb.psf.fwhm(psf, float(small['wf_psf_dx']))
    d, dx = O.az_inputs()['rect96x128']
    rd = pb._richdata.RichData(pb.asdevice(golden['rect96x128_data']).to(rdt), dx, None)
    q = O.queries(d.shape, dx)
    e = out['exact']
    e['xy_array'] = host(rd.exact_xy(q['xs'], q['ys']))
    e['xy_scalar'] = host(rd.exact_xy(q['x_scalar'], q['y_scalar']))
    e['xy_broadcast'] = host(rd.exact_xy(q['xs'], q['y_scalar']))
    e['polar_array'] = host(rd.exact_polar(q['rho'], q['phi']))
    e['polar_scalar'] = host(rd.exact_polar(q['rho_scalar']))
    e['ex_array'] = host(rd.exact_x(q['xs']))
    e['ex_scalar'] = host(rd.exact_x(q['x_scalar']))
    e['ey_array'] = host(rd.exact_y(q['ys']))
    e['ey_scalar'] = host(rd.exact_y(q['y_scalar']))
    g = pb.asdevice(golden['gauss_data']).to(rdt)
    for key, metric in O.SIZE_METRICS.items():
        for crit in ('first', 'last'):
            out['size'][f'size_{key}_{crit}'] = pb.psf.estimate_size(g, metric, dx=1.0, criteria=crit)
    out['size']['gauss_fwhm'] = pb.psf.fwhm(g, 1.0)
    a = O.analytic_inputs()
    an = out['analytic']
    an['difflim_array'] = host(pb.otf.diffraction_limited_mtf(O.FNO, O.WVL, a['freqs']))
    an['difflim_scalar'] = pb.otf.diffraction_limited_mtf(O.FNO, O.WVL, a['freq_scalar'])
    an['difflim_above'] = pb.otf.diffraction_limited_mtf(O.FNO, O.WVL, a['freq_above'])
    f, m = pb.otf.diffraction_limited_mtf(O.FNO, O.WVL, samples=64)
    an['difflim_none_f'], an['difflim_none'] = host(f), host(m)
    an['airy'] = host(pb.psf.airydisk(a['airy_r'], O.FNO, O.WVL))
    an['airy_efield'] = host(pb.psf.airydisk_efield(a['airy_r'], O.FNO, O.WVL))
    an['airy_ft'] = host(pb.psf.airydisk_ft(a['airy_ft_r'], O.FNO, O.WVL))
    an['ee'] = host(pb.otf.analytical_encircled_energy_circular_aperture(O.FNO, O.WVL, a['ee_r']))
    pb.config.precision = 64
    return out


@pytest.mark.parametrize('prec', (64, 32))
def test_every_function_matches_the_reference(pb, golden, prec):
    out = engine_outputs(pb, golden, prec)
    for group, vals in out.items():
        worst, where = 0.0, None
        for key, v in vals.items():
            err = rel_err(v, golden[key], key)
            if err >= worst:
                worst, where = err, key
        within(f'analysis_{group}_fp{prec} ({where})', worst, BOUNDS[prec][group])


def test_value_dtypes_follow_the_data(pb, golden):
    """Coordinates fp64, values in the data's dtype (the reference returns float64 for float32 data)."""
    for rdt in (torch.float32, torch.float64):
        rd = pb._richdata.RichData(pb.asdevice(golden['odd255_data']).to(rdt), O.DX, None)
        r, v = rd.slices().azmedian
        assert r.dtype == torch.float64 and v.dtype == rdt
        assert rd.exact_xy([0.0, 1.0], 0.0).dtype == rdt
        assert rd.x.dtype == torch.float64 and rd.r.dtype == torch.float64
        c = pb._richdata.RichData(pb.asdevice(golden['odd255_data']).to(rdt) * (1 + 1j), O.DX, None)
        assert c.exact_polar([1.0, 2.0], 0.5).is_complex()


def test_fp32_statistics_are_the_fp64_ones_rounded_once(pb, golden):
    """float32 data is interpolated and reduced in fp64: every statistic of a float32 array is the float64 statistic of
    the same values rounded once, bit for bit (selection, min and max do no arithmetic at all)."""
    for name in ('odd255', 'nan_nodes', 'nan_column'):
        d32 = pb.asdevice(golden[f'{name}_data']).to(torch.float32)
        s32 = pb._richdata.RichData(d32, O.DX, None).slices()
        s64 = pb._richdata.RichData(d32.to(torch.float64), O.DX, None).slices()
        for s in ('avg', 'median', 'min', 'max', 'var'):
            a = getattr(s32, 'az' + s)[1]
            b = getattr(s64, 'az' + s)[1].to(torch.float32)
            assert torch.equal(torch.nan_to_num(a, nan=-7.0), torch.nan_to_num(b, nan=-7.0)), (name, s)


def test_repeated_calls_are_bit_identical(pb, golden):
    d = pb.asdevice(golden['nan_nodes_data'])
    res = []
    for _ in range(2):
        sl = pb._richdata.RichData(d, O.DX, None).slices()
        res.append([sl.azavg[1], sl.azvar[1], sl.azmedian[1], sl.azmin[1]])
    for a, b in zip(*res):
        assert torch.equal(torch.nan_to_num(a, nan=-7.0), torch.nan_to_num(b, nan=-7.0))
    g = pb.asdevice(golden['gauss_data'])
    assert pb.psf.fwhm(g, 1.0) == pb.psf.fwhm(g, 1.0)


def test_all_azimuthal_statistics_take_one_launch(pb, golden):
    from prysm_b200 import _ops
    sl = pb._richdata.RichData(pb.asdevice(golden['odd255_data']), O.DX, None).slices()
    torch.cuda.synchronize()
    n0 = _ops.launch_count()
    for s in ('azavg', 'azvar', 'azstd', 'azmin', 'azmax', 'azpv'):
        getattr(sl, s)
    assert _ops.launch_count() - n0 == 1
    sl.azmedian
    sl.azmedian
    assert _ops.launch_count() - n0 == 2


def test_no_crossing_raises_the_reference_error(pb, golden):
    g = pb.asdevice(golden['gauss_data'])
    with pytest.raises(ValueError, match='metric does not cross the sampled data'):
        pb.psf.estimate_size(g, 2.0, dx=1.0)


def test_uniform_cart_to_polar_is_the_lattice_the_statistics_reduce(pb, golden):
    """coordinates.uniform_cart_to_polar returns the lattice pb_azimuthal_stats walks: its NaN-ignoring column mean is
    azavg."""
    d = golden['nan_nodes_data']
    x = (np.arange(64) - 32) * O.DX
    rho, phi, polar = pb.coordinates.uniform_cart_to_polar(x, x, pb.asdevice(d))
    assert polar.shape == (64, 64) and rho.dtype == torch.float64
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')         # the all-NaN column
        mean = np.nanmean(host(polar), axis=0)
    np.testing.assert_allclose(mean, golden['nan_nodes_azavg'], rtol=1e-12, atol=0)


# ---- the drop-in: the Lens MTF tutorial flow --------------------------------------------------------------------------
def _tutorial(psf_mod, otf_mod, psf, dx):
    mtf = otf_mod.mtf_from_psf(psf, dx)
    s = mtf.slices()
    fx = s.x[0]
    df = 1000 / (psf.shape[0] * dx)
    rho = np.array([0.0, 2.5 * df, 20.0 * df])
    return {'x': s.x[1], 'y': s.y[1], 'azavg': s.azavg[1], 'azmedian': s.azmedian[1],
            'polar': mtf.exact_polar(rho, np.array([0.0, 0.3, 1.2])),
            'difflim': otf_mod.diffraction_limited_mtf(8.0, 0.55, np.abs(np.asarray(fx, dtype=np.float64))[:40]),
            'fwhm': psf_mod.fwhm(psf, dx)}


def test_lens_mtf_tutorial_runs_behind_the_backend(pb):
    if not reference.installed():
        pytest.skip('reference prysm not installed')
    small = load_golden('small.npz')
    psf, dx = small['wf_psf_intensity'], float(small['wf_psf_dx'])
    with reference.loaded(), warnings.catch_warnings():
        warnings.simplefilter('ignore')
        import prysm.otf as potf
        import prysm.psf as ppsf
        from prysm.conf import config
        from prysm._richdata import RichData
        orig_slices = RichData.slices
        config.precision = 64
        want = _tutorial(ppsf, potf, psf, dx)
        try:
            config.precision = 32
            pb.mathops.set_backend_to_b200()
            assert RichData.slices is not orig_slices
            got = _tutorial(ppsf, potf, pb.asdevice(psf.astype(np.float32)), dx)
            # a host RichData still takes the reference's own path
            h = RichData(psf, dx, None)
            assert type(h.slices()).__module__ == 'prysm._richdata'
            assert isinstance(h.exact_xy(0.0, 0.0), np.ndarray)
        finally:
            pb.mathops.set_backend_to_defaults()
            config.precision = 64
        assert RichData.slices is orig_slices
        pb.config.precision = 64
    for k, v in want.items():
        g = got[k]
        if k != 'fwhm':
            assert isinstance(g, torch.Tensor) and g.is_cuda, k
        within(f'analysis_dropin_fp32 {k}', rel_err(host(g), host(v), k), BOUND_DROPIN)


# ---- full size against the host reference -----------------------------------------------------------------------------
def test_4096_mtf_statistics_match_the_host_reference(pb):
    if not reference.installed():
        pytest.skip('reference prysm not installed')
    n, dx = 4096, 1.0
    rng = np.random.default_rng(5)
    x = np.arange(n) - n // 2
    r2 = x[None, :] ** 2 + x[:, None] ** 2
    psf = np.exp(-r2 / (2 * 40.0 ** 2)) * (1 + 0.05 * rng.random((n, n)))
    with reference.loaded(), warnings.catch_warnings():
        warnings.simplefilter('ignore')
        import prysm.otf as potf
        import prysm.psf as ppsf
        from prysm.conf import config
        config.precision = 64
        mtf = potf.mtf_from_psf(psf, dx)
        s = mtf.slices()
        want = {'azavg': s.azavg[1], 'azmedian': s.azmedian[1], 'fwhm': ppsf.fwhm(psf, dx)}
    pb.config.precision = 64
    m = pb.otf.mtf_from_psf(pb.asdevice(psf), dx)
    sl = m.slices()
    got = {'azavg': host(sl.azavg[1]), 'azmedian': host(sl.azmedian[1]), 'fwhm': pb.psf.fwhm(pb.asdevice(psf), dx)}
    for k in want:
        within(f'analysis_4096_fp64 {k}', rel_err(got[k], want[k], k), BOUND_4096[k])
