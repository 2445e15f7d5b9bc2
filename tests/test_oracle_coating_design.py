"""CPU: the reference, where it is installed (oracle/_ref), re-derives every coating-design fixture
(tests/golden/coating_design*.npz) bit for bit; the header's coating-design enums are the values the binding reads;
and every argument error of the merit terms and the needle function is raised with the reference's type and message
before anything reaches the device."""
import numpy as np
import pytest

from conftest import load_golden
import coating_design_oracle as O
import reference


@pytest.fixture(scope='module')
def golden():
    return load_golden('coating_design.npz')


def test_reference_rederives_the_fixtures(golden):
    if not reference.installed():
        pytest.skip('reference prysm not installed')
    mine = O.reference_outputs()
    assert sorted(mine) == sorted(golden)
    for k, v in golden.items():
        np.testing.assert_array_equal(mine[k], v, err_msg=k)


def test_fixtures_hold_the_index_cases(golden):
    # the tie at a boundary listed twice keeps no seed (numpy's fancy assignment): the gradient is zero
    for pol in O.POLS:
        assert not golden[f'qw_mesh_{pol}_Ptie_gth'].any()
        assert golden[f'qw_mesh_{pol}_Pdup_gth'].any()
        # layer -1 averages boundaries N and 0, unlike the last layer's two boundaries
        assert golden[f'metal_mesh_{pol}_Lm1_value'] != golden[f'metal_mesh_{pol}_L0_value']
        assert golden[f'metal_mesh_{pol}_Am1_value'] > 0


def test_header_enums():
    from prysm_b200 import _capi as c
    assert (c.CM_IN_TARGET, c.CM_IN_WEIGHT, c.CM_IN_NEEDLE, c.CM_NOPS) == (6, 7, 8, 9)
    assert c.CM_NOPS > c.TF_NOPS and c.CM_IN_TARGET == c.TF_NOPS
    assert (c.CM_Q_R, c.CM_Q_T, c.CM_Q_ABS, c.CM_Q_ESQ, c.CM_Q_PEAK, c.CM_Q_LAYER) == tuple(range(6))
    assert c.CM_POL_AVG not in (c.TF_POL_S, c.TF_POL_P)
    flags = (c.CM_OUT_VALUE, c.CM_OUT_RESIDUALS, c.CM_OUT_GRAD_THICKNESS, c.CM_OUT_GRAD_INDEX, c.CM_ACCUMULATE)
    assert flags == (1, 2, 4, 8, 16)
    assert c.CM_OUT_GRAD_THICKNESS >> 2 == c.TF_GRAD_THICKNESS and c.CM_OUT_GRAD_INDEX >> 2 == c.TF_GRAD_INDEX
    assert 'pb_coating_merit' in c.SIGNATURES and 'pb_needle' in c.SIGNATURES


def _no_device(monkeypatch):
    """Make any upload or launch fail loudly, so that an error raised is known to come before the device."""
    from prysm_b200 import _ops

    def boom(*a, **k):
        raise AssertionError('reached the device')
    monkeypatch.setattr(_ops, 'device', boom)
    monkeypatch.setattr(_ops, '_call', boom)


W = np.linspace(0.45, 0.7, 5)


@pytest.mark.parametrize('make, exc, msg', [
    (lambda c: c.Reflectance(W, theta=np.linspace(0, 0.5, 3)), ValueError,
     'wvl and theta are both 1-D; pass meshgridded arrays for a spectral/angular grid'),
    (lambda c: c.Transmittance(W, target=np.zeros(4)), ValueError,
     'wvl, theta, target, and weight must be broadcast-compatible'),
    (lambda c: c.FieldInLayer(0, W, weight=np.ones(3)), ValueError,
     'wvl, theta, target, and weight must be broadcast-compatible'),
    (lambda c: c.Reflectance(W, pol='x'), ValueError, "pol must be 's', 'p', or 'avg'"),
])
def test_constructor_errors(monkeypatch, make, exc, msg):
    from prysm_b200 import coatings as c
    _no_device(monkeypatch)
    with pytest.raises(exc) as e:
        make(c)
    assert str(e.value) == msg
    if reference.installed():
        with reference.loaded():
            from prysm.x.coatings import merit
            with pytest.raises(exc) as r:
                make(merit)
            assert str(r.value) == msg


def _stack(c):
    return c.Stack([1.38, 2.05], [0.1, 0.07], 1.52)


@pytest.mark.parametrize('make, msg', [
    (lambda c: c.LayerAbsorptance(2, 0.55), 'index 2 is out of bounds for axis 0 with size 2'),
    (lambda c: c.LayerAbsorptance(-3, 0.55), 'index -3 is out of bounds for axis 0 with size 2'),
    (lambda c: c.FieldIntensityAtBoundary(3, 0.55), 'index 3 is out of bounds for axis 0 with size 3'),
    (lambda c: c.FieldIntensityAtBoundary(-4, 0.55), 'index -4 is out of bounds for axis 0 with size 3'),
    (lambda c: c.FieldInLayer(2, 0.55), 'index 3 is out of bounds for axis 0 with size 3'),
    (lambda c: c.PeakFieldAtInterfaces(0.55, boundaries=[0, 5]), 'index 5 is out of bounds for axis 0 with size 3'),
])
@pytest.mark.parametrize('call', ['value', 'residuals', 'value_and_grad'])
def test_index_errors_before_any_launch(monkeypatch, make, msg, call):
    from prysm_b200 import coatings as c, _ops
    _host_only(monkeypatch, c, _ops)
    t = make(c)
    st = _stack(c)
    with pytest.raises(IndexError) as e:
        getattr(t, call)(st)
    assert str(e.value) == msg
    if reference.installed():
        with reference.loaded():
            from prysm.x import coatings as rc
            with pytest.raises(IndexError) as r:
                getattr(make(rc), call)(_stack(rc))
            assert str(r.value) == msg


def _host_only(monkeypatch, c, _ops):
    """Uploads stay host tensors and any launch fails loudly: an error raised is known to come before the device."""
    import torch
    monkeypatch.setattr(_ops, '_call', lambda *a, **k: (_ for _ in ()).throw(AssertionError('reached the device')))
    monkeypatch.setattr(_ops, 'device', lambda: 'cpu')
    monkeypatch.setattr(c, '_real', lambda a: torch.as_tensor(np.asarray(a, dtype=np.float64)))
    monkeypatch.setattr(c, '_cplx', lambda a: torch.as_tensor(np.asarray(a, dtype=np.complex128)))


def test_empty_peak_list_and_bad_grad_fn_before_any_launch(monkeypatch):
    from prysm_b200 import coatings as c, _ops
    _host_only(monkeypatch, c, _ops)
    st = _stack(c)
    with pytest.raises(ValueError, match='zero-size array to reduction operation maximum which has no identity'):
        c.PeakFieldAtInterfaces(0.55, boundaries=[]).value(st)
    with pytest.raises(TypeError, match='grad_fn must be thickness_gradient or index_gradient'):
        c.Reflectance(0.55).value_and_grad(st, grad_fn=lambda f, **kw: None)


def test_needle_errors_before_any_launch(monkeypatch):
    from prysm_b200 import coatings as c, _ops
    _host_only(monkeypatch, c, _ops)
    st = _stack(c)
    for t in (c.LayerAbsorptance(0, 0.55), c.FieldIntensityAtBoundary(0, 0.55), c.PeakFieldAtInterfaces(0.55),
              c.FieldInLayer(0, 0.55), [c.Reflectance(0.55), c.FieldInLayer(0, 0.55)]):
        with pytest.raises(NotImplementedError, match='needle synthesis supports reflectance / transmittance targets'):
            c.needle_function(st, t, 1.38, [0.05])
    with pytest.raises(ValueError, match='needle_function requires at least one layer'):
        c.needle_function(c.Stack([], [], 1.52), c.Reflectance(0.55), 1.38, [0.0])


def test_as_merit_reads_reference_terms(monkeypatch):
    if not reference.installed():
        pytest.skip('reference prysm not installed')
    from prysm_b200 import coatings as c, _ops
    _host_only(monkeypatch, c, _ops)
    with reference.loaded():
        from prysm.x.coatings import merit
        wv = np.linspace(0.5, 0.6, 3)
        ref = merit.MeritFunction([merit.Reflectance(wv, pol='s', target=0.2, weight=2.0),
                                   merit.PeakFieldAtInterfaces(wv, boundaries=[0, 1]),
                                   merit.FieldInLayer(-1, wv), merit.LayerAbsorptance(1, wv),
                                   merit.FieldIntensityAtBoundary(2, wv)])
        m = c.as_merit(ref)
    assert [type(t).__name__ for t in m.terms] == ['Reflectance', 'PeakFieldAtInterfaces', 'FieldInLayer',
                                                   'LayerAbsorptance', 'FieldIntensityAtBoundary']
    assert m.terms[0].pol == 's' and float(m.terms[0].target) == 0.2 and float(m.terms[0].weight) == 2.0
    assert m.terms[1].boundaries == [0, 1] and m.terms[2].layer == -1 and m.terms[3].layer == 1
    assert m.terms[4].boundary == 2
    assert c.as_merit(m) is m
