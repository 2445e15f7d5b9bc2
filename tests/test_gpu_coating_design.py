"""GPU: coating design (prysm_b200.coatings merit terms and needle_function) against the reference's fp64 fixtures
(tests/golden/coating_design*.npz), the needle identities on the device, bit-identical repeats, the launch and copy
budget, and the reference's own refine and synthesize after set_backend_to_b200() where the reference is installed
(oracle/_ref).

Tolerances: values and residuals 1e-12 of the largest magnitude; gradients and P(z) 1e-10 of max(largest magnitude,
1) (the sample sums run in a different order).  fp32 storage (the chain still in fp64, each output rounded once):
FP32_BOUND for values and residuals, FP32_GRAD_BOUND for gradients and P."""
import numpy as np
import pytest
import torch

from conftest import load_golden, within
import coating_design_oracle as O
import reference
from gpu_fixtures import pb, host  # noqa: F401

pytestmark = pytest.mark.gpu
FP32_BOUND = 1.2e-6         # measured 7.6e-7 (H100 80GB HBM3, 700 W)
FP32_GRAD_BOUND = 4.5e-5    # measured 2.9e-5


@pytest.fixture(scope='module')
def gold():
    return load_golden('coating_design.npz')


def rel(got, ref, floor=0.0):
    got, ref = np.asarray(host(got), dtype=np.float64), np.asarray(ref, dtype=np.float64)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    if ref.size == 0:
        return 0.0
    den = max(float(np.abs(ref).max()), floor)
    return float(np.abs(got - ref).max()) / (den if den > 0 else 1.0)


def is_grad(k):
    return k.endswith(('_gth', '_gix')) or k.startswith('needle_')


def engine(pb):
    import types
    from prysm_b200 import coatings as c
    names = ('Reflectance', 'Transmittance', 'LayerAbsorptance', 'FieldIntensityAtBoundary', 'PeakFieldAtInterfaces',
             'FieldInLayer', 'MeritFunction', 'as_merit', 'Stack', 'needle_function', 'thickness_gradient',
             'index_gradient')
    return types.SimpleNamespace(host=host, **{n: getattr(c, n) for n in names})


def test_fixtures_fp64(pb, gold):
    pb.config.precision = 64
    got = O.run(engine(pb))
    assert sorted(got) == sorted(gold)
    bad = {}
    for k, ref in gold.items():
        e = rel(got[k], ref, 1.0 if is_grad(k) else 0.0)
        if not e < (1e-10 if is_grad(k) else 1e-12):
            bad[k] = e
    assert not bad, bad


def test_fixtures_fp32(pb, gold):
    pb.config.precision = 32
    try:
        got = O.run(engine(pb))
    finally:
        pb.config.precision = 64
    worst, worst_g = 0.0, 0.0
    for k, ref in gold.items():
        if is_grad(k):
            worst_g = max(worst_g, rel(got[k], ref, 1.0))
        else:
            worst = max(worst, rel(got[k], ref))
    within('coating_design_fp32', worst, FP32_BOUND)
    within('coating_design_fp32_grad', worst_g, FP32_GRAD_BOUND)


SUB = 1.52


def _three(c):
    return c.Stack([1.46, 2.2, 1.46], [0.10, 0.07, 0.12], SUB)


def _broadband(c, npts=9):
    return c.MeritFunction([c.Reflectance(np.linspace(0.45, 0.65, npts), pol='s', target=0.0)])


def test_host_material_needle_equals_thickness_gradient(pb):
    from prysm_b200 import coatings as c
    st, merit = _three(c), _broadband(c)
    _, grad = merit.value_and_grad(st)
    for k, (z, mat) in enumerate([(0.05, 1.46), (0.135, 2.2), (0.23, 1.46)]):
        P = float(host(c.needle_function(st, merit, mat, z))[0])
        assert P == pytest.approx(float(host(grad)[k]), rel=1e-9)


def _inserted(c, st, z, mat, dn):
    """insert_needle (needle.py:94-134) on this module's Stack"""
    Z = np.concatenate([[0.0], np.cumsum(st.thicknesses)])
    j = int(np.clip(np.searchsorted(Z, z, side='right') - 1, 0, len(st) - 1))
    idx, th = list(st.indices), list(st.thicknesses)
    return c.Stack(idx[:j] + [idx[j], mat, idx[j]] + idx[j + 1:],
                   th[:j] + [z - Z[j], dn, Z[j + 1] - z] + th[j + 1:], st.substrate_index, st.ambient_index)


@pytest.mark.parametrize('material', [2.05, 1.9])
@pytest.mark.parametrize('z', [0.05, 0.10, 0.22, 0.28])
@pytest.mark.parametrize('pol', ['s', 'avg'])
def test_needle_matches_finite_difference_of_insertion(pb, material, z, pol):
    from prysm_b200 import coatings as c
    st = _three(c)
    merit = c.MeritFunction([c.Reflectance(np.linspace(0.45, 0.65, 9)[:, None], theta=np.radians([0.0, 30.0])[None],
                                           pol=pol, target=0.0)])
    P = float(host(c.needle_function(st, merit, material, z))[0])
    dn = 1e-7
    fd = (merit.value(_inserted(c, st, z, material, dn)) - merit.value(st)) / dn
    assert np.isclose(P, fd, rtol=3e-3, atol=1e-6)


@pytest.mark.parametrize('material', [1.38, 2.05])
def test_needle_stationary_at_the_qwot_optimum(pb, material):
    from prysm_b200 import coatings as c
    n_ar = np.sqrt(SUB)
    ar = c.Stack([n_ar], [0.55 / (4 * n_ar)], SUB)
    merit = c.MeritFunction([c.Reflectance(0.55, pol='s', target=0.0)])
    P = host(c.needle_function(ar, merit, material, np.linspace(0, float(np.sum(ar.thicknesses)), 200)))
    assert P.shape == (200,) and P.min() >= -1e-9


def _big(c):
    hl = [2.35 if i % 2 == 0 else 1.46 for i in range(20)]
    st = c.Stack(hl, [0.55 / 4 / n for n in hl], SUB)
    w = np.linspace(0.4, 0.8, 2001)[:, None]
    th = np.radians(np.linspace(0, 60, 61))[None, :]
    return st, w, th


@pytest.mark.parametrize('term', ['R', 'Peak', 'A'])
def test_two_calls_are_bit_identical(pb, term):
    from prysm_b200 import coatings as c
    st, w, th = _big(c)
    t = {'R': lambda: c.Reflectance(w, theta=th, target=0.5, pol='avg'),
         'Peak': lambda: c.PeakFieldAtInterfaces(w, theta=th, pol='p', boundaries=[0, 3, 3, 7]),
         'A': lambda: c.LayerAbsorptance(-1, w, theta=th, pol='s')}[term]()
    for fn in (c.thickness_gradient, c.index_gradient):
        v1, g1 = t.value_and_grad(st, grad_fn=fn)
        v2, g2 = t.value_and_grad(st, grad_fn=fn)
        assert v1 == v2 and torch.equal(g1, g2)
    assert torch.equal(t.residuals(st), t.residuals(st))
    if term == 'R':
        z = np.linspace(0, float(np.sum(st.thicknesses)), 240)
        assert torch.equal(c.needle_function(st, t, 1.38, z), c.needle_function(st, t, 1.38, z))


def test_two_launches_per_term_and_one_copy(pb, monkeypatch):
    from prysm_b200 import coatings as c, _ops
    st, w, th = _big(c)
    merit = c.MeritFunction([c.Reflectance(w, theta=th, target=0.5, pol='avg'),
                             c.FieldInLayer(-1, w, theta=th, pol='s')])
    merit.value_and_grad(st)
    copies = []
    orig = torch.Tensor.item
    monkeypatch.setattr(torch.Tensor, 'item', lambda self: copies.append(1) or orig(self))
    n0 = _ops.launch_count()
    v, g = merit.value_and_grad(st)
    torch.cuda.synchronize()
    assert _ops.launch_count() - n0 == 4 and len(copies) == 1
    assert g.is_cuda and g.shape == (20,) and isinstance(v, float)
    n0 = _ops.launch_count()
    c.needle_function(st, merit.terms[:1], 1.38, np.linspace(0, 1, 240))
    torch.cuda.synchronize()
    assert _ops.launch_count() - n0 == 2


def test_more_than_four_dims_is_refused_before_a_launch(pb):
    from prysm_b200 import coatings as c, _ops
    st = c.Stack([1.38], [0.1], 1.52)
    w = np.linspace(0.4, 0.9, 30).reshape(2, 1, 3, 1, 5)
    t = c.Reflectance(w, theta=np.zeros((1, 2, 1, 2, 1)))
    n0 = _ops.launch_count()
    with pytest.raises(ValueError):
        t.value_and_grad(st)
    with pytest.raises(ValueError):
        c.needle_function(st, t, 1.38, [0.05])
    assert _ops.launch_count() == n0


# ---- the reference's own design loops after set_backend_to_b200()

@pytest.fixture(scope='module')
def refm():
    if not reference.installed():
        pytest.skip('reference prysm not installed')
    with reference.loaded():
        from prysm.conf import config
        config.precision = 64
        from prysm.x import coatings
        yield coatings


WVL, N_AR = 0.55, np.sqrt(SUB)
QWOT = WVL / (4 * N_AR)


def _switched(pb, fn):
    pb.mathops.set_backend_to_b200()
    try:
        return fn()
    finally:
        pb.mathops.set_backend_to_defaults()


def test_refine_recovers_the_qwot(pb, refm):
    from prysm.x.coatings.merit import Reflectance
    rc = refm

    def run():
        assert rc.refine.__module__ == 'prysm.x.coatings.refine'
        s0 = rc.Stack([N_AR], [QWOT * 1.3], SUB)
        res = rc.refine(s0, Reflectance(WVL, pol='s', target=0.0), ftol=0.0, gtol=1e-14, maxiter=500)
        R = float(host(rc.RTA(res.stack, WVL, 0.0, 's')[0]))
        return res, R
    res, R = _switched(pb, run)
    assert res.stack.thicknesses[0] == pytest.approx(QWOT, rel=1e-3)
    assert R < 1e-8


@pytest.mark.parametrize('method', ['lbfgsb', 'lm'])
def test_refine_thickness_both_methods(pb, refm, method):
    rc = refm
    indices = [1.38, 2.05, 1.38]
    truth = np.array([0.10, 0.065, 0.115])
    wvls = np.linspace(0.5, 0.6, 6)
    R_target = np.asarray(rc.RTA(rc.Stack(indices, truth, SUB), wvls, 0.0, 's')[0])

    def run():
        target = rc.Reflectance(wvls, pol='s', target=R_target)
        assert type(target).__module__ == 'prysm_b200.coatings'
        res = rc.refine(rc.Stack(indices, truth + 0.01, SUB), target, method=method)
        return host(rc.RTA(res.stack, wvls, 0.0, 's')[0])
    assert np.allclose(_switched(pb, run), R_target, atol=1e-4)


def test_refine_index_variable(pb, refm):
    rc = refm
    th = [0.10, 0.08, 0.10]
    wvls = np.linspace(0.5, 0.6, 7)
    R_target = np.asarray(rc.RTA(rc.Stack([1.40, 2.20, 1.45], th, SUB), wvls, 0.0, 's')[0])
    # a term built before the switch: as_merit reads its public attributes
    target = rc.Reflectance(wvls, pol='s', target=R_target)

    def run():
        res = rc.refine(rc.Stack([1.40, 1.90, 1.45], th, SUB), target, variables='index', variable_layers=[1],
                        bounds=(1.3, 2.4), maxiter=400)
        return res, host(rc.RTA(res.stack, wvls, 0.0, 's')[0])
    res, R_fit = _switched(pb, run)
    assert np.allclose(R_fit, R_target, atol=1e-5)
    assert float(res.stack.indices[1]) == pytest.approx(2.20, rel=1e-3)


def test_first_lbfgsb_iterates_match_the_host_run(pb, refm):
    rc = refm
    from prysm.x.coatings.problem import CoatingProblem
    from prysm.x.optym.optimizers import PrysmLBFGSB
    wvls = np.linspace(0.45, 0.65, 9)[:, None]
    theta = np.radians([0.0, 20.0, 40.0])[None]

    def iterates():
        merit = rc.Reflectance(wvls, theta=theta, pol='avg', target=0.0)
        prob = CoatingProblem(rc.Stack([1.38, 2.05, 1.38, 2.05], [0.1, 0.07, 0.1, 0.07], SUB), merit)
        opt = PrysmLBFGSB(prob.fg, prob.x0(), memory=10, lower_bounds=np.zeros(4), upper_bounds=np.full(4, np.inf))
        out = []
        for _ in range(5):
            opt.step()
            out.append(np.array(opt.x, dtype=np.float64))
        return out
    want = iterates()
    got = _switched(pb, iterates)
    for a, b in zip(got, want):
        assert np.max(np.abs(a - b) / np.abs(b)) < 1e-9


def test_synthesize_grows_a_broadband_ar(pb, refm):
    rc = refm
    wvls = np.linspace(0.45, 0.65, 7)

    def run():
        merit = rc.MeritFunction([rc.Reflectance(wvls, pol='s', target=0.0)])
        start = rc.Stack([1.38, 2.05], [0.10, 0.10], SUB)
        start_merit = merit.value(start)
        res = rc.synthesize(start, merit, [1.38, 2.05], z_samples=120, max_iters=8, max_layers=16)
        return start_merit, res, host(rc.RTA(res.stack, wvls, 0.0, 's')[0])
    start_merit, res, R = _switched(pb, run)
    assert res.n_layers > 2 and res.merit < start_merit / 100 and np.max(R) < 5e-3


def test_set_backend_to_defaults_restores_the_host_path(pb, refm):
    rc = refm
    from prysm.x.coatings import merit, problem, refine, needle
    before = {(m.__name__, n): getattr(m, n) for m in (rc, merit, problem, refine, needle)
              for n in ('as_merit', 'Reflectance', 'MeritFunction', 'needle_function', 'thickness_gradient')
              if hasattr(m, n)}
    pb.mathops.set_backend_to_b200()
    try:
        assert needle.needle_function is not before[('prysm.x.coatings.needle', 'needle_function')]
        assert rc.Reflectance is pb.coatings.Reflectance and problem.as_merit is pb.coatings._host_as_merit
    finally:
        pb.mathops.set_backend_to_defaults()
    for (mod, n), v in before.items():
        assert getattr(__import__(mod, fromlist=['x']), n) is v, (mod, n)
    st = rc.Stack([1.38], [0.1], SUB)
    v, g = rc.Reflectance(0.55, pol='s').value_and_grad(st)
    assert isinstance(g, np.ndarray)
