"""CPU: the reference, where it is installed (oracle/_ref), re-derives every interferogram fixture
(tests/golden/interferogram*.npz) bit for bit; the metrology entry points and enums parse through the header binding;
every argument error is raised with the reference's message (or the documented ValueError) before anything reaches the
device; and set_backend_to_b200() re-binds and restores every metrology name, with a host Interferogram behind it giving
the reference's own bits."""
import warnings

import numpy as np
import pytest

from conftest import load_golden
import interferogram_oracle as O
import reference


@pytest.fixture(scope='module')
def golden():
    return load_golden('interferogram.npz')


def test_reference_rederives_the_fixtures(golden):
    if not reference.installed():
        pytest.skip('reference prysm not installed')
    mine = O.reference_outputs()
    assert sorted(mine) == sorted(golden)
    for k, v in golden.items():
        np.testing.assert_array_equal(np.asarray(mine[k]), v, err_msg=k)


def test_fixtures_cover_the_cases(golden):
    assert np.isnan(golden['circ_data']).any() and np.isnan(golden['spiky_data']).any()
    assert np.isfinite(golden['rect_data']).all() and golden['rect_data'].shape == (200, 320)
    assert golden['circ_data'].shape == (255, 255) and golden['spiky_data'].shape == (256, 256)
    assert golden['circ_crop'].shape[0] < 255                     # cropped
    assert golden['spiky_crop'].shape == (256, 256)               # the early return
    assert np.isnan(golden['spiky_psd_nan']).all()                # any NaN makes every PSD sample NaN
    assert (golden['circ_window_2d_welch'] < 0).any()             # negative in the corners
    assert golden['circ_tis'].shape == O.TIS_ANGLES.shape


def test_header_entry_points_and_enums():
    from prysm_b200 import _capi
    for name in ('pb_nan_stats', 'pb_masked_gram', 'pb_psd_prologue', 'pb_psd_epilogue', 'pb_band_trapz', 'pb_filter_h',
                 'pb_filter_apply', 'pb_gradient2d', 'pb_finite_bounds', 'pb_metro_pointwise'):
        assert name in _capi.SIGNATURES, name
    assert _capi.GRAM_MAX_K == 64
    assert (_capi.WIN_AUTO, _capi.WIN_WELCH, _capi.WIN_HANN, _capi.WIN_USER) == (0, 1, 2, 3)
    assert (_capi.FILT_LOWPASS, _capi.FILT_HIGHPASS, _capi.FILT_BANDPASS, _capi.FILT_BANDREJECT) == (0, 1, 2, 3)
    assert _capi.PW_WELCH == 9


def _no_device(monkeypatch):
    """every route to the device raises, so an error that comes out was raised before it"""
    from prysm_b200 import _ops

    def refuse(*a, **k):
        raise AssertionError('reached the device')
    monkeypatch.setattr(_ops, '_call', refuse)
    monkeypatch.setattr(_ops, 'asdevice', lambda a, dtype=None: a)


def _reference_error(fn):
    with reference.loaded(), warnings.catch_warnings():
        warnings.simplefilter('ignore')
        with pytest.raises(Exception) as ei:
            fn()
    return type(ei.value), str(ei.value)


class _FakeTensor:
    """stands for a device array in the argument checks: a shape and nothing else"""
    dtype = None
    ndim = 2

    def __init__(self, shape):
        self.shape = shape


def test_bandlimited_rms_needs_a_band(monkeypatch):
    from prysm_b200 import interferogram as E
    _no_device(monkeypatch)
    with pytest.raises(ValueError, match='must specify either period'):
        E._band_limits(lambda: 1.0, None, None, None, None)
    if reference.installed():
        def ref():
            from prysm import interferogram
            interferogram.bandlimited_rms(np.ones((4, 4)), np.ones((4, 4)))
        assert _reference_error(ref) == (ValueError, 'must specify either period (wavelength) or frequency')


def test_band_limit_precedence_and_warnings():
    from prysm_b200 import interferogram as E
    top = lambda: 9.0  # noqa: E731
    # the reference's quirk: with wlhigh None, fhigh becomes the data's limit even when wllow set it
    assert E._band_limits(top, 0.5, None, None, None) == (0, 9.0)
    assert E._band_limits(top, None, 2.0, None, None) == (0.5, 9.0)
    assert E._band_limits(top, 0.5, 2.0, 7.0, 8.0) == (0.5, 2.0)
    assert E._band_limits(top, None, None, 0.5, None) == (0.5, 9.0)
    assert E._band_limits(top, None, None, None, 3.0) == (0, 3.0)


def test_window_and_filter_errors_before_the_device(monkeypatch):
    from prysm_b200 import interferogram as E
    _no_device(monkeypatch)
    with pytest.raises(ValueError, match='unknown window type'):
        E._window_args((8, 8), 1.0, 'triangle', 4)
    for typ in ('notch', 'LPX'):
        with pytest.raises(ValueError, match='unknown filter type'):
            E._filter_type(typ)
    assert E._filter_type('LowPass') == E.capi.FILT_LOWPASS
    if reference.installed():
        def ref():
            from prysm import interferogram
            interferogram.make_window(np.ones((8, 8)), 1.0, 'triangle')
        assert _reference_error(ref) == (ValueError, 'unknown window type')


def test_automatic_window_corners_follow_numpy_slices():
    from prysm_b200 import interferogram as E
    # 255: round(5.1) = 5 samples; 20: round(0.4) = 0, so [:0] is empty and [-0:] is the whole axis
    assert E._corners((255, 255))[:4] == [0, 5, 0, 5] and E._corners((255, 255))[12:] == [250, 255, 250, 255]
    assert E._corners((20, 100))[:4] == [0, 0, 0, 2] and E._corners((20, 100))[4:8] == [0, 0, 98, 100]
    assert E._corners((20, 100))[8:12] == [0, 20, 0, 2]


def test_pvr_and_pad_argument_errors(monkeypatch):
    from prysm_b200 import interferogram as E
    _no_device(monkeypatch)
    i = E.Interferogram.__new__(E.Interferogram)
    i._data = _FakeTensor((4, 6))
    i._x = i._y = i._r = i._t = 0
    with pytest.raises(ValueError, match='data must be square'):
        i.pvr()
    with pytest.raises(ValueError, match='Neither samples nor shape specified'):
        i.pad()
    with pytest.raises(ValueError, match='Both sampels and shape provided'):
        i.pad(samples=2, shape=8)


def test_lstsq_mode_limit_before_the_device(monkeypatch):
    from prysm_b200 import _ops
    monkeypatch.setattr(_ops, '_call', lambda *a, **k: (_ for _ in ()).throw(AssertionError('reached the device')))
    monkeypatch.setattr(_ops, 'metro_data', lambda d: d)
    with pytest.raises(ValueError, match='1 to 64 modes'):
        _ops.masked_gram([None] * 65, _FakeTensor((4, 4)))
    with pytest.raises(ValueError, match='1 to 64 modes'):
        _ops.masked_gram([], _FakeTensor((4, 4)))


def test_gram_solve_is_the_minimum_norm_answer():
    """pinv(A^T A) A^T d = pinv(A) d: a duplicated mode gets the reference's minimum-norm coefficients"""
    from prysm_b200.polynomials import solve_gram
    m, d = O.lstsq_inputs()
    keep = np.isfinite(d).ravel()
    A = np.vstack([m.reshape(6, -1)[:, keep], d.ravel()[keep][None]]).T
    packed = (A.T @ A)[np.triu_indices(7)]
    got = solve_gram(packed, 6)
    want = np.linalg.lstsq(A[:, :6], A[:, 6], rcond=None)[0]
    np.testing.assert_allclose(got, want, rtol=1e-10, atol=1e-12)


def test_backend_rebinds_and_restores_every_metrology_name():
    if not reference.installed():
        pytest.skip('reference prysm not installed')
    import prysm_b200 as pb
    d = O.maps()['circ']
    with reference.loaded(), warnings.catch_warnings():
        warnings.simplefilter('ignore')
        import importlib
        from prysm.conf import config
        config.precision = 64
        mods = {m: importlib.import_module(m) for m in pb.mathops._DISPATCHED}
        before = {(m, a): getattr(mods[m], a) for m, names in pb.mathops._DISPATCHED.items() for a in names}
        cls = mods['prysm.interferogram'].Interferogram
        members = {n: cls.__dict__[n] for n in pb.mathops._IFG_PROPERTIES + pb.mathops._IFG_METHODS}

        def host_run():
            i = cls(d.copy(), dx=O.DX)
            out = {'pv': i.pv, 'std': i.std, 'pvr': i.pvr()}
            i.remove_piston().remove_tiptilt().remove_power().crop().fill(0)
            out['data'] = i.data
            out['psd'] = i.psd().data
            out['blr'] = i.bandlimited_rms(flow=0.5)
            out['rms'] = mods['prysm.util'].rms(d)
            return out
        want = host_run()
        try:
            pb.mathops.set_backend_to_b200()
            for (m, a), orig in before.items():
                assert getattr(mods[m], a) is not orig, (m, a)
            for n, orig in members.items():
                assert cls.__dict__[n] is not orig, n
            got = host_run()
        finally:
            pb.mathops.set_backend_to_defaults()
        for (m, a), orig in before.items():
            assert getattr(mods[m], a) is orig, (m, a)
        for n, orig in members.items():
            assert cls.__dict__[n] is orig, n
    for k, v in want.items():
        np.testing.assert_array_equal(got[k], v, err_msg=k)


def test_switch_before_prysm_interferogram_is_imported():
    """prysm.interferogram binds fttools.pad2d at import: imported after the switch it would capture the engine's
    pad2d, and a host Interferogram.pad would hand back CUDA data and keep doing so after the restore."""
    if not reference.installed():
        pytest.skip('reference prysm not installed')
    import prysm_b200 as pb
    small = O.small_map()[0]

    def pad_run(ifg):
        i = ifg.Interferogram(small.copy(), dx=O.DX).pad(samples=(3, 4))
        return i.data, i.x
    with reference.loaded(), warnings.catch_warnings():
        warnings.simplefilter('ignore')
        from prysm import interferogram
        want = pad_run(interferogram)
    with reference.loaded(), warnings.catch_warnings():
        warnings.simplefilter('ignore')
        import sys
        import prysm  # noqa: F401
        from prysm.conf import config
        config.precision = 64
        assert 'prysm.interferogram' not in sys.modules
        try:
            pb.mathops.set_backend_to_b200()
            from prysm import fttools, interferogram
            assert interferogram.pad2d is not fttools.pad2d     # the reference's, not the engine's
            got = pad_run(interferogram)
        finally:
            pb.mathops.set_backend_to_defaults()
        assert interferogram.pad2d is fttools.pad2d
        after = pad_run(interferogram)
    for g in (got, after):
        for a, b in zip(g, want):
            assert isinstance(a, np.ndarray)
            np.testing.assert_array_equal(a, b)


def _refuse_device(monkeypatch):
    """the wrappers run on CPU tensors here; the library call itself is refused"""
    from prysm_b200 import _ops

    def refuse(*a, **k):
        raise AssertionError('reached the device')
    monkeypatch.setattr(_ops, '_call', refuse)
    monkeypatch.setattr(_ops, 'metro_data', lambda d: d.contiguous())
    monkeypatch.setattr(_ops, 'asdevice', lambda a, dtype=None: a if isinstance(a, __import__('torch').Tensor)
                        else __import__('torch').as_tensor(np.asarray(a)))
    return _ops


def test_operand_shapes_are_checked_before_the_device(monkeypatch):
    import torch
    from prysm_b200 import interferogram as E, _capi as capi
    _ops = _refuse_device(monkeypatch)
    h = torch.zeros((8, 6), dtype=torch.float64)
    # a window the reference would broadcast
    with pytest.raises(ValueError, match='window of shape'):
        E.psd(h, 0.1, window=np.ones(6))
    # r and a PSD of different shapes: numpy's IndexError, as the reference's work[r < flow] raises
    with pytest.raises(IndexError, match='boolean index did not match indexed array along axis 0'):
        E.bandlimited_rms(torch.zeros((7, 6), dtype=torch.float64), h, flow=0.1)
    with pytest.raises(ValueError, match='does not match the data shape'):
        _ops.band_trapz(h, r=torch.zeros((7, 6), dtype=torch.float64))
    # a mask of the wrong shape
    i = E.Interferogram.__new__(E.Interferogram)
    i._data = h
    i._x = i._y = i._r = i._t = None
    with pytest.raises(IndexError, match='along axis 1; size of axis is 6 but size of corresponding boolean axis is 5'):
        i.mask(np.ones((8, 5), dtype=bool))
    # the wrappers themselves
    for kw in (dict(u=torch.zeros(47, dtype=torch.float64)), dict(v=torch.zeros(49, dtype=torch.float64)),
               dict(m=torch.ones(47, dtype=torch.bool))):
        with pytest.raises(ValueError, match='elements for an operation over 48'):
            _ops.metro_pointwise(capi.PW_SUB, x=h, **kw)
    with pytest.raises(ValueError, match='data of 48 elements for an operation over 96'):
        _ops.metro_pointwise(capi.PW_REAL, x=h, shape=(8, 6), dtype=torch.float64)
    with pytest.raises(ValueError, match='does not match the data shape'):
        _ops.filter_h((8, 6), capi.FILT_H, torch.float64, h.device, r=torch.zeros((6, 8), dtype=torch.float64))


def test_pv_of_no_finite_sample_raises_the_references_error(monkeypatch):
    from prysm_b200 import util
    monkeypatch.setattr(util, 'nan_stats', lambda a: np.array([0.0, 0.0, np.inf, -np.inf, 0.0, 4.0, np.nan, 0.0, 0.0]))
    with pytest.raises(ValueError) as ei:
        util.pv(None)
    if reference.installed():
        def ref():
            from prysm import util as putil
            putil.pv(np.full(4, np.nan))
        assert _reference_error(ref) == (ValueError, str(ei.value))
