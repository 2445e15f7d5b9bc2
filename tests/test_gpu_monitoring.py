"""GPU: optical monitoring (prysm_b200.coatings monitoring_trace, turning_points, level_cut, cutoff_levels,
simulate_run, simulate_runs, monitoring_error_sensitivity, choose_monitor_wavelength) against the reference's fp64
fixtures (tests/golden/monitoring*.npz), the decision rules bit for bit on the reference's own traces, batched runs
equal to single runs, bit-identical repeats, the launch and copy budget, the reference's monitoring functions after
set_backend_to_b200() where the reference is installed (oracle/_ref), and the physics of the reference's own tests.

Tolerances: traces, levels and as-built thicknesses 1e-12 of the largest magnitude; J and scores 1e-9 of the largest
|J| (the realized reflectance runs in a different order of operations, and J divides its differences by eps = 1e-4);
the best wavelength exactly.  fp32 storage (the runs still in fp64, the thicknesses and outputs rounded to float32):
FP32_BOUND of the largest magnitude, FP32_J_BOUND for J and scores."""
import types

import numpy as np
import pytest
import torch

from conftest import load_golden, within
import monitoring_oracle as O
import reference
from gpu_fixtures import pb, host  # noqa: F401

pytestmark = pytest.mark.gpu
FP32_BOUND = 1.4e-6         # measured 9.1e-7 (H100 80GB HBM3, 700 W)
FP32_J_BOUND = 3.4e-6       # measured 2.2e-6


@pytest.fixture(scope='module')
def gold():
    return load_golden('monitoring.npz')


def rel(got, ref):
    got, ref = np.asarray(host(got), dtype=np.float64), np.asarray(ref, dtype=np.float64)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    if ref.size == 0:
        return 0.0
    den = float(np.abs(ref).max())
    return float(np.abs(got - ref).max()) / (den if den > 0 else 1.0)


def is_j(k):
    return k.startswith(('sens_', 'choose_scores'))


def to_dev(a):
    return torch.as_tensor(np.asarray(a, dtype=np.float64)).cuda()


def engine(pb):
    from prysm_b200 import coatings as c
    names = ('monitoring_trace', 'turning_points', 'level_cut', 'cutoff_levels', 'monitoring_error_sensitivity',
             'choose_monitor_wavelength')
    return types.SimpleNamespace(Stack=c.Stack, RTA=c.RTA, host=host, device=to_dev, run=c.simulate_run,
                                 **{n: getattr(c, n) for n in names})


def compare(got, gold, bound, jbound):
    assert sorted(got) == sorted(gold)
    worst, worst_j, bad = 0.0, 0.0, {}
    for k, ref in gold.items():
        if k == 'choose_best':
            if float(got[k]) != float(ref):
                bad[k] = (float(got[k]), float(ref))
            continue
        e = rel(got[k], ref)
        if is_j(k):
            worst_j = max(worst_j, e)
            if jbound is not None and not e < jbound:
                bad[k] = e
        else:
            worst = max(worst, e)
            if bound is not None and not e < bound:
                bad[k] = e
    return worst, worst_j, bad


def test_fixtures_fp64(pb, gold):
    pb.config.precision = 64
    _, _, bad = compare(O.run(engine(pb)), gold, 1e-12, 1e-9)
    assert not bad, bad


def test_fixtures_fp32(pb, gold):
    pb.config.precision = 32
    try:
        got = O.run(engine(pb))
    finally:
        pb.config.precision = 64
    worst, worst_j, bad = compare(got, gold, None, None)
    assert 'choose_best' not in bad
    within('monitoring_fp32', worst, FP32_BOUND)
    within('monitoring_fp32_J', worst_j, FP32_J_BOUND)


def test_decisions_bit_identical_on_reference_traces(pb, gold):
    from prysm_b200 import coatings as c
    pb.config.precision = 64
    for j in range(len(O.TRACES)):
        k = f'trace{j}_{O.TRACES[j][0]}'
        d, sig = gold[f'{k}_d'], gold[f'{k}_sig']
        tp = host(c.turning_points(to_dev(d), to_dev(sig)))
        np.testing.assert_array_equal(tp, gold[f'{k}_tp'], err_msg=k)
        mid = 0.5 * (float(np.min(sig)) + float(np.max(sig)))
        assert c.level_cut(to_dev(d), to_dev(sig), mid, target=0.5 * float(d[-1])) == float(gold[f'{k}_cut']), k
    for name, (d, sig, level, target) in O.analytic().items():
        if level is None:
            np.testing.assert_array_equal(host(c.turning_points(to_dev(d), to_dev(sig))), gold[name], err_msg=name)
        else:
            assert c.level_cut(to_dev(d), to_dev(sig), level, target) == float(gold[name]), name


def _hl(c, L, seed=3):
    n, d, sub, amb = O.hl(L, seed)
    return c.Stack(n, d, sub, amb)


@pytest.mark.parametrize('strategy', ['level', 'turning'])
def test_batched_runs_equal_single_runs(pb, strategy):
    from prysm_b200 import coatings as c
    pb.config.precision = 64
    st = _hl(c, 10)
    rng = np.random.default_rng(5)
    key = 'signal_errors' if strategy == 'level' else 'thickness_errors'
    e = (2e-3 if strategy == 'level' else 4e-3) * rng.standard_normal((6, 10))
    batch = host(c.simulate_runs(st, 0.6, strategy=strategy, **{key: e}))
    for r in range(6):
        one = c.simulate_run(st, 0.6, strategy=strategy, **{key: e[r]})
        np.testing.assert_array_equal(batch[r], np.asarray(one.thicknesses), err_msg=str(r))
    # one monitor wavelength per run
    wv = [0.5, 0.6, 0.65]
    per = host(c.simulate_runs(st, wv, strategy=strategy, **{key: e[:3]}))
    for r, w in enumerate(wv):
        np.testing.assert_array_equal(per[r], np.asarray(c.simulate_run(st, w, strategy=strategy,
                                                                        **{key: e[r]}).thicknesses))


def test_repeats_are_bit_identical(pb):
    from prysm_b200 import coatings as c
    pb.config.precision = 64
    st = _hl(c, 20, 4)
    e = 5e-4 * np.random.default_rng(2).standard_normal((64, 20))
    assert torch.equal(c.simulate_runs(st, 0.6, signal_errors=e), c.simulate_runs(st, 0.6, signal_errors=e))
    w = np.linspace(0.45, 0.65, 101)
    assert torch.equal(c.monitoring_error_sensitivity(st, 0.6, w), c.monitoring_error_sensitivity(st, 0.6, w))
    b1, s1 = c.choose_monitor_wavelength(st, [0.5, 0.6, 0.7], w)
    b2, s2 = c.choose_monitor_wavelength(st, [0.5, 0.6, 0.7], w)
    assert b1 == b2 and torch.equal(s1, s2)


def _budget(monkeypatch, fn):
    """(launches, device-to-host copies) of fn()"""
    from prysm_b200 import _ops
    copies = []
    item, cpu = torch.Tensor.item, torch.Tensor.cpu
    monkeypatch.setattr(torch.Tensor, 'item', lambda self: copies.append(1) or item(self))
    monkeypatch.setattr(torch.Tensor, 'cpu', lambda self, *a, **k: copies.append(1) or cpu(self, *a, **k))
    try:
        torch.cuda.synchronize()
        n0 = _ops.launch_count()
        fn()
        torch.cuda.synchronize()
        return _ops.launch_count() - n0, len(copies)
    finally:
        monkeypatch.setattr(torch.Tensor, 'item', item)
        monkeypatch.setattr(torch.Tensor, 'cpu', cpu)


@pytest.mark.parametrize('L', [4, 40])
@pytest.mark.parametrize('cands', [2, 7])
def test_launch_and_copy_budget(pb, monkeypatch, L, cands):
    from prysm_b200 import coatings as c
    pb.config.precision = 64
    st = _hl(c, L)
    w = np.linspace(0.45, 0.65, 31)
    cand = list(np.linspace(0.45, 0.75, cands))
    assert _budget(monkeypatch, lambda: c.simulate_run(st, 0.6, n_points=57 * cands)) == (2, 1)
    assert _budget(monkeypatch, lambda: c.simulate_run(st, 0.6, strategy='turning')) == (1, 1)
    assert _budget(monkeypatch, lambda: c.monitoring_error_sensitivity(st, 0.6, w)) == (4, 0)
    assert _budget(monkeypatch, lambda: c.monitoring_error_sensitivity(st, 0.6, w, strategy='turning')) == (3, 0)
    assert _budget(monkeypatch, lambda: c.choose_monitor_wavelength(st, cand, w)) == (4, 1)
    assert _budget(monkeypatch, lambda: c.simulate_runs(st, cand, n_points=1200)) == (2, 0)


def test_invalid_arguments_raise_before_any_launch(pb):
    from prysm_b200 import coatings as c, _ops
    st = _hl(c, 4)
    n0 = _ops.launch_count()
    for call, exc in ((lambda: c.simulate_run(st, 0.6, strategy='x'), ValueError),
                      (lambda: c.simulate_run(st, 0.6, n_points=0), ValueError),
                      (lambda: c.simulate_runs(st, 0.6, strategy='turning', turning_index=0), IndexError),
                      (lambda: c.monitoring_error_sensitivity(st, 0.6, [0.5], signal_errors=np.zeros(4)), TypeError),
                      (lambda: c.choose_monitor_wavelength(st, [], [0.5]), ValueError),
                      (lambda: c.level_cut(to_dev([]), to_dev([]), 0.5), ValueError)):
        with pytest.raises(exc):
            call()
    assert _ops.launch_count() == n0


# ---- the reference's monitoring module after set_backend_to_b200()

@pytest.fixture(scope='module')
def refmon():
    if not reference.installed():
        pytest.skip('reference prysm not installed')
    with reference.loaded():
        from prysm.conf import config
        config.precision = 64
        from prysm.x.coatings import monitoring
        yield monitoring


NAMES = ('monitoring_trace', 'turning_points', 'level_cut', 'cutoff_levels', 'simulate_run',
         'monitoring_error_sensitivity', 'choose_monitor_wavelength')


def test_dropin_gives_the_golden_values(pb, refmon, gold):
    import prysm.x.coatings as rc
    before = {(m.__name__, n): getattr(m, n) for m in (rc, refmon) for n in NAMES}
    pb.config.precision = 64
    pb.mathops.set_backend_to_b200()
    try:
        for n in ('simulate_run', 'monitoring_error_sensitivity', 'choose_monitor_wavelength'):
            assert getattr(refmon, n) is getattr(pb.coatings, n) and getattr(rc, n) is getattr(pb.coatings, n)
        m = types.SimpleNamespace(Stack=rc.Stack, RTA=rc.RTA, host=host, device=None, run=refmon.simulate_run,
                                  **{n: getattr(refmon, n) for n in NAMES if n != 'simulate_run'})
        got = O.run(m)
        assert type(m.run(rc.Stack([1.46], [0.09], 1.52), 0.6)) is rc.Stack
        # turning_points / level_cut reach the engine with a device signal
        d, sig = refmon.monitoring_trace(rc.Stack([1.46], [0.09], 1.52), 0, 0.6)
        assert d.is_cuda and sig.is_cuda and refmon.turning_points(d, sig).is_cuda
        assert isinstance(refmon.level_cut(d, sig, float(sig[5]), 0.05), float)
    finally:
        pb.mathops.set_backend_to_defaults()
    _, _, bad = compare(got, gold, 1e-12, 1e-9)
    assert not bad, bad
    for (mod, n), v in before.items():
        assert getattr(__import__(mod, fromlist=['x']), n) is v, (mod, n)


# ---- the reference's own physics, restated

W, SUB = 0.55, 1.52
FOUR = [1.46, 2.05, 1.46, 2.05]
DESIGN = np.array([0.09, 0.067, 0.10, 0.067])


def test_zero_error_runs_reproduce_the_design(pb):
    from prysm_b200 import coatings as c
    pb.config.precision = 64
    ab = c.simulate_run(c.Stack(FOUR, DESIGN, SUB), W, strategy='level', n_points=1200)
    np.testing.assert_allclose(ab.thicknesses, DESIGN, atol=2e-4)
    qw = np.array([W / (4 * n) for n in FOUR])
    ab = c.simulate_run(c.Stack(FOUR, qw, SUB), W, strategy='turning', n_points=2000)
    np.testing.assert_allclose(ab.thicknesses, qw, atol=3e-4)


def test_best_monitor_lowers_the_realized_spread(pb):
    from prysm_b200 import coatings as c
    pb.config.precision = 64
    des = c.Stack(FOUR, DESIGN, SUB)
    cands = [0.45, 0.50, 0.55, 0.60, 0.65]
    best, scores = c.choose_monitor_wavelength(des, cands, np.array([W]), strategy='level', design_pol='s')
    worst = cands[int(np.argmax(host(scores)))]
    assert worst == 0.55 and best != 0.55
    assert float(scores.max()) > 3 * float(scores.min())
    se = 5e-4 * np.random.default_rng(1).standard_normal((300, 4))

    def spread(wm):
        th = host(c.simulate_runs(des, wm, signal_errors=se, n_points=800))
        R = host(c.RTA(c.Stack(FOUR, th.T, SUB), W, 0.0, 's')[0])
        assert R.shape == (300,)
        return np.std(R)
    assert spread(best) < 0.5 * spread(worst)
