"""CPU: the reference, where it is installed (oracle/_ref), re-derives every optical-monitoring fixture
(tests/golden/monitoring*.npz) bit for bit; the fixtures hold the cases they are named for; the header's monitoring
enums are the values the binding reads; and argument errors are raised before anything reaches the device."""
import numpy as np
import pytest

from conftest import load_golden
import monitoring_oracle as O
import reference


@pytest.fixture(scope='module')
def golden():
    return load_golden('monitoring.npz')


def test_reference_rederives_the_fixtures(golden):
    if not reference.installed():
        pytest.skip('reference prysm not installed')
    mine = O.reference_outputs()
    assert sorted(mine) == sorted(golden)
    for k, v in golden.items():
        np.testing.assert_array_equal(mine[k], v, err_msg=k)


def test_fixtures_hold_the_named_cases(golden):
    N10 = len(O.stacks()['hl10'][0])
    # one grid point: the only sample, 1e-12, for every layer
    assert np.all(golden['run_level_n1'] == 1e-12)
    # fewer turning points than asked: the nominal thicknesses
    np.testing.assert_array_equal(golden['run_turning_fewer'], O.stacks()['hl10'][1])
    # a zero-error turning run lands on the quarter waves
    np.testing.assert_allclose(golden['run_turning'], O.stacks()['qw4'][1], atol=3e-4)
    # each strategy ignores the other's error vector
    np.testing.assert_array_equal(golden['run_level_ignores_th_err'], golden['run_level'])
    assert golden['run_level'].shape == (N10,)
    assert float(golden['cut_tie']) == 0.375 and float(golden['cut_none_tie']) == 0.5
    assert float(golden['cut_zero']) == 0.3 and golden['tp_short'].size == 0
    # the self-quarter-wave monitor is the worst candidate
    assert O.CANDIDATES[int(np.argmax(golden['choose_scores']))] == 0.55
    assert float(golden['choose_best']) != 0.55


def test_header_enums():
    from prysm_b200 import _capi as c
    assert (c.MON_LEVEL, c.MON_TURNING, c.MON_R, c.MON_T) == (0, 1, 0, 1)
    for n in ('pb_monitor_runs', 'pb_monitor_cut', 'pb_monitor_jacobian'):
        assert n in c.SIGNATURES


def _host_only(monkeypatch):
    """Uploads stay host tensors and any launch fails loudly: an error raised is known to come before the device."""
    import torch
    from prysm_b200 import coatings as c, _ops
    monkeypatch.setattr(_ops, '_call', lambda *a, **k: (_ for _ in ()).throw(AssertionError('reached the device')))
    monkeypatch.setattr(_ops, 'device', lambda: 'cpu')
    monkeypatch.setattr(c, '_real', lambda a: torch.as_tensor(np.asarray(a, dtype=np.float64)))
    monkeypatch.setattr(c, '_cplx', lambda a: torch.as_tensor(np.asarray(a, dtype=np.complex128)))
    return c


def _stack(c):
    return c.Stack([1.46, 2.05], [0.09, 0.067], 1.52)


@pytest.mark.parametrize('call, exc, msg', [
    (lambda c, s: c.simulate_run(s, 0.6, strategy='x'), ValueError, "strategy must be 'level' or 'turning'"),
    (lambda c, s: c.simulate_run(s, 0.6, n_points=-1), ValueError, 'Number of samples, -1, must be non-negative.'),
    (lambda c, s: c.simulate_run(s, 0.6, n_points=0), ValueError, 'attempt to get argmin of an empty sequence'),
    (lambda c, s: c.simulate_run(s, 0.6, strategy='turning', turning_index=0), IndexError,
     'turning_index must be 1 or more, got 0'),
    (lambda c, s: c.simulate_runs(s, [0.5, 0.6], signal_errors=np.zeros((3, 2))), ValueError,
     '2 monitor wavelengths and 3 error rows do not make one set of runs'),
    (lambda c, s: c.monitoring_error_sensitivity(s, 0.6, [0.5], signal_errors=np.zeros(2)), TypeError,
     "simulate_run() got multiple values for keyword argument 'signal_errors'"),
    (lambda c, s: c.monitoring_error_sensitivity(s, 0.6, [0.5], colour=1), TypeError,
     "simulate_run() got an unexpected keyword argument 'colour'"),
    (lambda c, s: c.choose_monitor_wavelength(s, [], [0.5]), ValueError, 'attempt to get argmin of an empty sequence'),
    (lambda c, s: c.level_cut([], [], 0.5), ValueError, 'attempt to get argmin of an empty sequence'),
    (lambda c, s: c.monitoring_error_sensitivity(s, 0.6, [0.5], design_pol='avg'), ValueError,
     "unknown polarization, use 'p' or 's'"),
    (lambda c, s: c.choose_monitor_wavelength(c.Stack([], [], 1.52), [0.5, 0.6], [0.5], design_pol='x'), ValueError,
     "unknown polarization, use 'p' or 's'"),
    (lambda c, s: c.simulate_run(s, 0.6, signal_errors=[1e-3]), IndexError,
     'index 1 is out of bounds for axis 0 with size 1'),
])
def test_argument_errors_before_any_launch(monkeypatch, call, exc, msg):
    c = _host_only(monkeypatch)
    with pytest.raises(exc) as e:
        call(c, _stack(c))
    assert str(e.value) == msg


def test_no_layers_neither_raises_nor_launches(monkeypatch):
    c = _host_only(monkeypatch)
    empty = c.Stack([], [], 1.52)
    assert len(c.simulate_run(empty, 0.6, strategy='x')) == 0
    assert tuple(c.simulate_runs(empty, [0.5, 0.6]).shape) == (2, 0)
    assert tuple(c.monitoring_error_sensitivity(empty, 0.6, [0.5, 0.6]).shape) == (2, 0)


@pytest.mark.skipif(not reference.installed(), reason='reference prysm not installed')
def test_reference_raises_the_same_errors():
    with reference.loaded():
        from prysm.x.coatings import Stack, monitoring as mon
        s = Stack([1.46, 2.05], [0.09, 0.067], 1.52)
        with pytest.raises(ValueError, match="strategy must be 'level' or 'turning'"):
            mon.simulate_run(s, 0.6, strategy='x')
        with pytest.raises(ValueError, match='Number of samples, -1, must be non-negative.'):
            mon.simulate_run(s, 0.6, n_points=-1)
        with pytest.raises(ValueError, match='attempt to get argmin of an empty sequence'):
            mon.simulate_run(s, 0.6, n_points=0)
        with pytest.raises(TypeError, match="got multiple values for keyword argument 'signal_errors'"):
            mon.monitoring_error_sensitivity(s, 0.6, [0.5], signal_errors=np.zeros(2))
        # turning_index 0 on a trace without turning points: the reference's IndexError
        with pytest.raises(IndexError):
            mon.simulate_run(s, 0.6, strategy='turning', turning_index=0, n_points=2)
        assert len(mon.simulate_run(Stack([], [], 1.52), 0.6, strategy='x')) == 0
        with pytest.raises(ValueError, match="unknown polarization, use 'p' or 's'"):
            mon.monitoring_error_sensitivity(s, 0.6, [0.5], design_pol='avg')
        with pytest.raises(ValueError, match="unknown polarization, use 'p' or 's'"):
            mon.choose_monitor_wavelength(Stack([], [], 1.52), [0.5, 0.6], [0.5], design_pol='x')
        with pytest.raises(IndexError, match='index 1 is out of bounds for axis 0 with size 1'):
            mon.simulate_run(s, 0.6, signal_errors=np.array([1e-3]))


def test_errors_past_the_last_layer_are_not_read(monkeypatch):
    c = _host_only(monkeypatch)
    e = c._err_rows(np.arange(5.0), 2)
    assert tuple(e.shape) == (1, 2) and e.tolist() == [[0.0, 1.0]]
    if reference.installed():
        with reference.loaded():
            from prysm.x.coatings import Stack, monitoring as mon
            s = Stack([1.46, 2.05], [0.09, 0.067], 1.52)
            # the reference takes a longer vector and reads its first N entries
            a = mon.simulate_run(s, 0.6, signal_errors=[1e-3, 2e-3, 5.0], n_points=57)
            b = mon.simulate_run(s, 0.6, signal_errors=[1e-3, 2e-3], n_points=57)
            np.testing.assert_array_equal(a.thicknesses, b.thicknesses)
