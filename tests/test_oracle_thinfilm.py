"""CPU: the reference, where it is installed (oracle/_ref), re-derives every thin-film fixture (tests/golden/thinfilm*.npz)
bit for bit; the fixtures hold the cases the GPU tests rely on (total internal reflection, a metal layer, a lossy
layer); and every argument error is raised with the reference's type and message before anything reaches the
device."""

import numpy as np
import pytest

from conftest import load_golden
import thinfilm_oracle as O
import reference


@pytest.fixture(scope='module')
def golden():
    return load_golden('thinfilm.npz')


@pytest.fixture(scope='module')
def ref():
    if not reference.installed():
        pytest.skip('reference prysm not installed')
    with reference.loaded():
        yield O.reference_modules()


def test_reference_rederives_the_fixtures(golden, ref):
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        mine = O.run(ref)
    assert sorted(mine) == sorted(golden)
    for k, v in golden.items():
        np.testing.assert_array_equal(mine[k], v, err_msg=k)


def test_fixtures_hold_tir_metal_and_lossy_cases(golden):
    # past the critical angle of the 1.7 -> 1.0 case every ray is reflected: |r| = 1 at 45 degrees and beyond
    for pol in O.POLS:
        R = golden[f'tir_{pol}_R']
        assert np.allclose(R[:, 2:], 1.0, atol=1e-12) and (R[:, :2] < 0.999).all()
        assert np.allclose(np.abs(golden[f'ml_tir_{pol}_r'][1:]), 1.0, atol=1e-12)
        # the metal and the lossy layer absorb
        assert golden[f'metal_{pol}_A'][1].min() > 1e-4
        assert golden[f'lossy_{pol}_A'][2].min() > 1e-3
        assert golden[f'l40_{pol}_A'].shape == (40,) + np.broadcast_shapes(O.GRID_WVL.shape, O.GRID_THETA.shape)


def _no_device(monkeypatch):
    """Make any upload or launch fail loudly, so that an error raised is known to come before the device."""
    from prysm_b200 import _ops

    def boom(*a, **k):
        raise AssertionError('reached the device')
    monkeypatch.setattr(_ops, 'device', boom)
    monkeypatch.setattr(_ops, '_call', boom)


@pytest.mark.parametrize('call, msg', [
    (lambda tf, c: tf.multilayer_stack_rt([1.38], [0.1], 0.55, 'x', 1.52), 'unknown polarization, use p or s'),
    (lambda tf, c: tf.multilayer_stack_rt([1.38, 2.0], [0.1, 0.2, 0.3], 0.55, 's', 1.52),
     'indices and thicknesses must be broadcastable to the same shape'),
    (lambda tf, c: tf.multilayer_stack_rt(np.zeros((0, 3)), np.zeros((0, 3)), 0.55, 's', 1.52),
     'indices and thicknesses must contain at least one film layer'),
    (lambda tf, c: tf.multilayer_stack_rt(np.ones((2, 3, 4)), np.ones((2, 3, 4)), 0.55, 's', np.ones(5)),
     'substrate_index must be broadcastable to the trailing layer dimensions'),
    (lambda tf, c: tf.multilayer_stack_rt(np.ones((2, 3, 4)), np.ones((2, 3, 4)), 0.55, 's', 1.5,
                                          aoi=np.zeros((3, 4))), None),
    (lambda tf, c: c.Stack([1.38, 2.0], [0.1], 1.52), 'indices and thicknesses must describe the same number of layers'),
    (lambda tf, c: c.RTA(c.Stack([1.38], [0.1], 1.52), 0.55, 0.0, 'x'), "unknown polarization, use 'p' or 's'"),
    (lambda tf, c: c.forward_eval(c.Stack([1.38], [0.1], 1.52), 0.55, 0.0, 'q'), "unknown polarization, use 'p' or 's'"),
    (lambda tf, c: c.field_at_depth(c.Stack([], [], 1.52), 0.0, 0.55, 0.0, 's'),
     'field_at_depth requires at least one layer'),
    (lambda tf, c: c.field_at_depth(c.Stack([1.38], [0.1], 1.52), [0.05, 0.2], 0.55, 0.0, 's'),
     'z must lie within the coating stack'),
])
def test_errors_match_the_reference_before_any_launch(call, msg, ref, monkeypatch):
    """Each call raises ValueError here, and the reference raises ValueError with the same message (a numpy
    broadcasting failure where msg is None)."""
    from prysm_b200 import coatings, thinfilm
    _no_device(monkeypatch)
    with pytest.raises(ValueError) as mine:
        call(thinfilm, coatings)
    with pytest.raises(ValueError) as theirs:
        call(ref.thinfilm, ref.coatings)
    if msg is not None:
        assert str(mine.value) == str(theirs.value) == msg
