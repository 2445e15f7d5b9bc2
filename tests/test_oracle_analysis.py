"""CPU: the reference, where it is installed (oracle/_ref), re-derives every analysis fixture (tests/golden/analysis*.npz)
bit for bit; the azimuthal-statistics flags and row limit are consistent; and every argument error of the analysis
functions is raised with the reference's type and message before anything reaches the device (there is none here)."""
import warnings

import numpy as np
import pytest

from conftest import load_golden
import analysis_oracle as O
import reference


@pytest.fixture(scope='module')
def golden():
    return load_golden('analysis.npz')


def test_reference_rederives_the_fixtures(golden):
    if not reference.installed():
        pytest.skip('reference prysm not installed')
    mine = O.reference_outputs()
    assert sorted(mine) == sorted(golden)
    for k, v in golden.items():
        np.testing.assert_array_equal(np.asarray(mine[k]), v, err_msg=k)


def test_fixtures_cover_the_nan_cases(golden):
    """The NaN centre node makes every column whose circle lies within one sample of it all NaN, so every statistic
    there is NaN; further out the columns have numbers.  The NaN disk covers the centre: the columns inside it are NaN,
    those that cross its edge have numbers."""
    for s in O.STATS:
        assert np.isnan(golden[f'nan_column_az{s}'][:2]).all(), s
        assert np.isfinite(golden[f'nan_column_az{s}'][2:]).all(), s
        assert np.isnan(golden[f'nan_disk_az{s}'][:8]).all(), s
        assert np.isfinite(golden[f'nan_disk_az{s}'][8:]).all(), s
    assert golden['xy_scalar'].shape == () and golden['polar_scalar'].shape == () and golden['ex_scalar'].shape == ()
    assert golden['difflim_above'] == 0 and golden['difflim_scalar'].shape == ()


def test_azimuthal_flags_and_row_limit():
    from prysm_b200 import _capi
    assert _capi.AZ_ALL == (_capi.AZ_COUNT | _capi.AZ_MEAN | _capi.AZ_VAR | _capi.AZ_MIN | _capi.AZ_MAX | _capi.AZ_MEDIAN)
    # the column of samples and the kernel's own shared memory fit in the 227 KB a block may opt in to on sm_90
    assert _capi.AZ_MAX_NY * 8 + 2048 <= 227 * 1024


def _reference_error(fn):
    with reference.loaded(), warnings.catch_warnings():
        warnings.simplefilter('ignore')
        from prysm.conf import config
        config.precision = 64
        with pytest.raises(Exception) as ei:
            fn()
    return type(ei.value), str(ei.value)


def _grid(shape, dx):
    ny, nx = shape
    x = (np.arange(nx) - nx // 2) * dx
    y = (np.arange(ny) - ny // 2) * dx
    return np.meshgrid(x, y)


def _no_device(monkeypatch):
    """every route to the device raises, so an error that comes out was raised before it"""
    from prysm_b200 import _ops

    def refuse(*a, **k):
        raise AssertionError('reached the device')
    monkeypatch.setattr(_ops, '_call', refuse)
    monkeypatch.setattr(_ops, 'asdevice', refuse)


@pytest.mark.parametrize('metric,criteria', [('fwhm2', 'last'), ('FWHM', 'middle'), (None, 'first')])
def test_estimate_size_argument_errors(monkeypatch, metric, criteria):
    g = O.gauss()
    want = None
    if reference.installed():
        def ref():
            from prysm.psf import estimate_size
            estimate_size(g, metric, dx=1.0, criteria=criteria)
        want = _reference_error(ref)
    from prysm_b200 import psf
    _no_device(monkeypatch)
    with pytest.raises(ValueError) as ei:
        psf.estimate_size(g, metric, dx=1.0, criteria=criteria)
    if want is not None:
        assert (type(ei.value), str(ei.value)) == want
    else:
        assert str(ei.value) in ('unknown metric, use fwhm, 1/e, or 1/e^2', 'unknown criteria, use first or last')


# (method, args) whose points leave the 96 x 128 grid of dx 0.5 (x in [-32, 31.5], y in [-24, 23.5])
OUT_OF_RANGE = [
    ('exact_xy', (40.0, 0.0)), ('exact_xy', (0.0, 23.75)), ('exact_xy', ([0.0, -33.0], [0.0, 0.0])),
    ('exact_xy', (np.nan, 0.0)), ('exact_polar', (30.0, np.pi / 2)), ('exact_polar', ([1.0, 40.0],)),
    ('exact_x', (31.75,)), ('exact_x', ([-32.5, 1.0],)), ('exact_y', (-24.5,)), ('exact_y', ([0.0, 24.0],)),
]


@pytest.mark.parametrize('method,args', OUT_OF_RANGE)
def test_out_of_range_points_raise_the_reference_error(monkeypatch, method, args):
    d = np.random.default_rng(3).random((96, 128))
    x, y = _grid(d.shape, 0.5)
    want = None
    if reference.installed():
        def ref():
            from prysm._richdata import RichData
            getattr(RichData(d, 0.5, None), method)(*args)
        want = _reference_error(ref)
    from prysm_b200 import _richdata
    _no_device(monkeypatch)
    with pytest.raises(ValueError) as ei:
        getattr(_richdata, method)(d, x, y, *args)
    if want is not None:
        assert (type(ei.value), str(ei.value)) == want


def test_azimuthal_statistics_refuse_too_many_rows(monkeypatch):
    """A column of the polar lattice is held on chip: more than AZ_MAX_NY rows is a ValueError before any launch."""
    from prysm_b200 import _capi, _richdata
    _no_device(monkeypatch)
    ny = _capi.AZ_MAX_NY + 1
    sl = _richdata.Slices(np.zeros((ny, 4)), np.arange(4.0) - 2, np.arange(ny, dtype=np.float64) - ny // 2)
    for stat in ('azavg', 'azmedian', 'azstd', 'azpv'):
        with pytest.raises(ValueError, match=f'at most {_capi.AZ_MAX_NY} phi samples'):
            getattr(sl, stat)
