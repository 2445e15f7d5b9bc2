"""GPU: thin-film stacks (prysm_b200.thinfilm, prysm_b200.coatings) against the reference's fp64 fixtures
(tests/golden/thinfilm*.npz), energy conservation and finite differences on the device, bit-identical gradients,
and the reference run on the host where it is installed (oracle/_ref): a per-pixel 1024^2 stack, its own user code
after set_backend_to_b200(), and a coated fold mirror taken to focus as a Jones pupil.

Tolerances (max |got - ref| over the output's largest magnitude): fp64 1e-12; gradients 1e-10 of the largest
per-layer value (the sample sums run in a different order).  The per-layer absorptance and the gradients are measured
against max(largest magnitude, 1): in a lossless layer both are rounding noise around zero, and A is a fraction of the
incident power.  fp32 storage (the chain still in fp64, each output
rounded once): FP32_BOUND, gradients FP32_GRAD_BOUND."""
import numpy as np
import pytest
import torch

from conftest import load_golden, within
import thinfilm_oracle as O
import reference
from gpu_fixtures import pb, host  # noqa: F401

pytestmark = pytest.mark.gpu
FP32_BOUND = 1e-5          # measured 6.8e-6 (H100 80GB HBM3, 700 W)
FP32_GRAD_BOUND = 4.5e-5     # measured 3.0e-5


@pytest.fixture(scope='module')
def gold():
    return load_golden('thinfilm.npz')


def rel(got, ref, floor=0.0):
    got, ref = host(got).astype(np.complex128), np.asarray(ref)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    if ref.size == 0:
        return 0.0
    den = max(float(np.abs(ref).max()), floor)
    return float(np.abs(got - ref).max()) / (den if den > 0 else 1.0)


def floor_of(k):
    return 1.0 if k.endswith('_A') or '_gth_' in k or '_gix_' in k else 0.0


def outputs(pb, gold):
    """name -> (engine result, fixture) of every fixture; gradient keys hold 'gth' / 'gix'."""
    from prysm_b200 import coatings as c, thinfilm as tf
    out = {}
    for name, args in O.ml_cases().items():
        r, t = tf.multilayer_stack_rt(*args)
        out[f'{name}_r'], out[f'{name}_t'] = r, t
    for sname, (n, d, sub, amb) in O.stacks().items():
        st = c.Stack(n, d, sub, amb)
        for pol in O.POLS:
            k = f'{sname}_{pol}'
            out[f'{k}_r'], out[f'{k}_t'] = c.stack_rt(st, O.GRID_WVL, O.GRID_THETA, pol)
            out[f'{k}_E'], out[f'{k}_H'] = c.internal_fields(st, O.GRID_WVL, O.GRID_THETA, pol)
            out[f'{k}_R'], out[f'{k}_T'], out[f'{k}_A'] = c.RTA(st, O.GRID_WVL, O.GRID_THETA, pol)
            f = c.forward_eval(st, O.GRID_WVL, O.GRID_THETA, pol)
            for seed, kw in O.seeds(k, tuple(f.r.shape), len(st)).items():
                out[f'{k}_gth_{seed}'] = c.thickness_gradient(f, **kw)
                out[f'{k}_gix_{seed}'] = c.index_gradient(f, **kw)
            if len(st) and sname in O.FAD_STACKS:
                # depths accumulate in fp64 from the stack's thicknesses (at fp32 storage those are float32)
                Z = np.concatenate([[0.0], np.cumsum(np.asarray(st.thicknesses, dtype=np.float64))])
                for zname, z in (('bound', Z), ('dense', np.linspace(0.0, Z[-1], 12001))):
                    E, H = c.field_at_depth(st, z, O.FAD_WVL, O.FAD_THETA, pol)
                    out[f'fad_{k}_{zname}_E'], out[f'fad_{k}_{zname}_H'] = E, H
                E, H = c.field_at_depth(st, 0.7 * Z[-1], O.GRID_WVL, O.GRID_THETA, pol)
                out[f'fad_{k}_grid_E'], out[f'fad_{k}_grid_H'] = E, H
    assert sorted(out) == sorted(gold)
    return {k: (v, gold[k]) for k, v in out.items()}


def test_fixtures_fp64(pb, gold):
    pb.config.precision = 64
    bad = {}
    for k, (got, ref) in outputs(pb, gold).items():
        assert host(got).dtype in (np.float64, np.complex128), k
        bound = 1e-10 if '_gth_' in k or '_gix_' in k else 1e-12
        if not rel(got, ref, floor_of(k)) < bound:
            bad[k] = rel(got, ref, floor_of(k))
        if k.startswith(('gap_', 'ml_gap_')) and k.endswith(('_r', '_t')):
            # through the evanescent gap t falls to about 1e-33: hold every sample to its own magnitude
            g, f = host(got).astype(np.complex128), np.asarray(ref)
            err = float(np.max(np.abs(g - f) / np.abs(f)))
            if not err < 1e-10:
                bad[k + ' (per sample)'] = err
    assert not bad, bad


def test_fixtures_fp32(pb, gold):
    pb.config.precision = 32
    try:
        worst, worst_g = 0.0, 0.0
        for k, (got, ref) in outputs(pb, gold).items():
            assert host(got).dtype in (np.float32, np.complex64), k
            if '_gth_' in k or '_gix_' in k:
                worst_g = max(worst_g, rel(got, ref, floor_of(k)))
            else:
                worst = max(worst, rel(got, ref, floor_of(k)))
    finally:
        pb.config.precision = 64
    within('thinfilm_fp32', worst, FP32_BOUND)
    within('thinfilm_fp32_grad', worst_g, FP32_GRAD_BOUND)


def _lossy_40():
    return O.stacks()['l40']


def test_energy_conservation_on_a_lossy_grid(pb):
    from prysm_b200 import coatings as c
    n, d, sub, amb = _lossy_40()
    st = c.Stack(n, d, sub, amb)
    w = np.linspace(0.4, 0.9, 2001)[:, None]
    th = np.radians(np.linspace(0, 60, 61))[None, :]
    for pol in O.POLS:
        R, T, A = c.RTA(st, w, th, pol)
        total = host(R) + host(T) + host(A).sum(axis=0)
        assert host(A)[5].min() > 0
        assert np.abs(total - 1).max() < 1e-12


@pytest.mark.parametrize('pol', ['s', 'p'])
@pytest.mark.parametrize('aoi', [0.0, 30.0])
@pytest.mark.parametrize('key', ['R', 'T', 'A', 'E'])
def test_gradients_match_finite_differences(pb, pol, aoi, key):
    """test_diff.py's central differences (h = 1e-7; rtol 2e-5 thickness, 3e-5 index, atol 1e-8), of the engine's own
    forward evaluation."""
    from prysm_b200 import coatings as c
    indices = [1.38, 2.05, 1.5 + 0.2j, 2.2]
    th = np.array([0.10, 0.07, 0.05, 0.06])
    wv, theta = np.array([0.5, 0.55, 0.6]), np.radians(aoi)

    def value(idx, d):
        f = c.forward_eval(c.Stack(idx, d, 1.52), wv, theta, pol)
        q = {'R': f.R_value, 'T': f.T_value, 'A': f.A_value, 'E': f.Esq_value}[key]
        return float((q ** 2).sum())

    f0 = c.forward_eval(c.Stack(indices, th, 1.52), wv, theta, pol)
    q = {'R': f0.R_value, 'T': f0.T_value, 'A': f0.A_value, 'E': f0.Esq_value}[key]
    kw = {{'R': 'dR', 'T': 'dT', 'A': 'dA', 'E': 'dEsq'}[key]: 2 * q}
    gth, gix = host(c.thickness_gradient(f0, **kw)), host(c.index_gradient(f0, **kw))
    h = 1e-7
    fd_th, fd_ix = np.zeros(4), np.zeros(4)
    for i in range(4):
        tp, tm = th.copy(), th.copy()
        tp[i] += h
        tm[i] -= h
        fd_th[i] = (value(indices, tp) - value(indices, tm)) / (2 * h)
        ip, im = list(indices), list(indices)
        ip[i] += h
        im[i] -= h
        fd_ix[i] = (value(ip, th) - value(im, th)) / (2 * h)
    assert np.allclose(gth, fd_th, rtol=2e-5, atol=1e-8)
    assert np.allclose(gix, fd_ix, rtol=3e-5, atol=1e-8)


def test_gradients_are_bit_identical_and_two_launches(pb):
    from prysm_b200 import coatings as c, _ops
    n, d, sub, amb = _lossy_40()
    st = c.Stack(n, d, sub, amb)
    w = np.linspace(0.4, 0.9, 2001)[:, None]
    th = np.radians(np.linspace(0, 60, 61))[None, :]
    f = c.forward_eval(st, w, th, 's')
    dA = np.ones((40, 2001, 61))
    a = c.index_gradient(f, dR=1.0, dA=dA)
    n0 = _ops.launch_count()
    b = c.index_gradient(f, dR=1.0, dA=dA)
    torch.cuda.synchronize()
    assert _ops.launch_count() - n0 == 2
    assert torch.equal(a, b)
    assert torch.equal(c.thickness_gradient(f, dR=1.0), c.thickness_gradient(f, dR=1.0))


def test_fp32_fields_through_thick_metal_stay_finite(pb):
    """2 um of silver: |v| grows by about e^180 through the layer before the fields are scaled by t, beyond float32's
    range; the float outputs are staged in fp64 and agree with the fp64 run."""
    from prysm_b200 import coatings as c
    w, th = np.linspace(0.45, 0.65, 5), np.radians(20.0)
    out = {}
    for prec in (64, 32):
        pb.config.precision = prec
        try:
            st = c.Stack([1.46, 0.05 + 3.9j], [0.08, 2.0], 1.52)
            R, T, A = c.RTA(st, w, th, 's')
            E, H = c.internal_fields(st, w, th, 's')
            out[prec] = [host(v) for v in (R, A, E, H)]
        finally:
            pb.config.precision = 64
    for a, b in zip(out[32], out[64]):
        assert np.isfinite(a).all()
        assert rel(a, b, 1.0) < 1e-6


def test_more_than_four_dims_is_refused_before_a_launch(pb):
    from prysm_b200 import coatings as c, _ops
    st = c.Stack([1.38], [0.1], 1.52)
    w = np.linspace(0.4, 0.9, 30).reshape(2, 1, 3, 1, 5)
    th = np.zeros((1, 2, 1, 2, 1))
    n0 = _ops.launch_count()
    with pytest.raises(ValueError):
        c.RTA(st, w, th, 's')
    assert _ops.launch_count() == n0


@pytest.fixture(scope='module')
def refm():
    if not reference.installed():
        pytest.skip('reference prysm not installed')
    with reference.loaded():
        yield O.reference_modules()


def test_per_pixel_1024_against_the_reference(pb, refm):
    from prysm_b200 import thinfilm as tf
    N = 1024
    rng = np.random.default_rng(0)
    idx = np.array([1.38, 2.05, 1.38, 2.05])[:, None, None] * np.ones((1, N, N))
    th = np.array([0.1, 0.07, 0.1, 0.07])[:, None, None] * (1 + 0.02 * rng.standard_normal((1, N, N)))
    for pol in O.POLS:
        r, t = tf.multilayer_stack_rt(idx, th, 0.55, pol, 1.52, aoi=10)
        s = (slice(None), slice(3, None, 37), slice(5, None, 41))
        rr, tr = refm.thinfilm.multilayer_stack_rt(idx[s], th[s], 0.55, pol, 1.52, aoi=10)
        assert rel(host(r)[s[1:]], rr) < 1e-12
        assert rel(host(t)[s[1:]], tr) < 1e-12


def test_reference_user_code_after_set_backend(pb, refm):
    from prysm.mathops import array_to_true_numpy as tn
    from prysm.x import coatings as rc
    from prysm import thinfilm as rtf
    st = rc.Stack([1.38, 2.05, 1.5 + 0.3j, 2.05], [0.12, 0.08, 0.05, 0.10], 1.52)
    w, th = np.linspace(0.45, 0.65, 5), np.radians(20.0)

    def user():
        R, T, A = rc.RTA(st, w, th, 'p')
        f = rc.diff.forward_eval(st, w, th, 's')
        g = rc.thickness_gradient(f, dR=np.ones(5))
        r, t = rtf.multilayer_stack_rt([1.38, 2.05], [0.1, 0.07], 0.55, 's', 1.52, aoi=np.linspace(0, 40, 12))
        E, H = rc.field_at_depth(st, np.linspace(0, 0.3, 31), 0.55, th, 's')
        return [tn(v) for v in (R, T, A, g, r, t, E, H)]

    want = user()
    pb.mathops.set_backend_to_b200()
    try:
        assert rc.RTA is pb.coatings.RTA and rtf.multilayer_stack_rt is pb.thinfilm.multilayer_stack_rt
        got = user()
    finally:
        pb.mathops.set_backend_to_defaults()
    assert rc.RTA is not pb.coatings.RTA
    for a, b in zip(got, want):
        assert rel(a, b) < 1e-10


def test_coated_fold_mirror_jones_pupil_to_focus(pb, refm):
    """A 45-degree fold mirror with a protected-silver coating: the AOI map across a 128^2 pupil gives r_s, r_p per
    pixel, diag(r_s, r_p) is the Jones pupil, and jones_adapter(focus) takes it to focus; the reference runs the same
    chain on the host."""
    from prysm_b200 import thinfilm as tf, polarization as pol, propagation as P
    from prysm.x import polarization as rpol
    from prysm.propagation import focus as rfocus
    N = 128
    v = (np.arange(N) - N / 2) / (N / 2)
    x, y = np.meshgrid(v, v)
    aoi = 45.0 + 8.0 * x + 2.0 * y * x          # degrees, across an f/3-ish beam
    amp = (x * x + y * y <= 1).astype(np.float64)
    layers = ([1.46, 0.05 + 3.9j], [0.08, 0.12])

    def jones(rs, rp, zeros):
        J = zeros((N, N, 2, 2))
        J[..., 0, 0] = rs * amp
        J[..., 1, 1] = rp * amp
        return J

    rs_r, _ = refm.thinfilm.multilayer_stack_rt(*layers, 0.55, 's', 1.0, aoi=aoi)
    rp_r, _ = refm.thinfilm.multilayer_stack_rt(*layers, 0.55, 'p', 1.0, aoi=aoi)
    want = rpol.jones_adapter(rfocus)(jones(rs_r, rp_r, lambda s: np.zeros(s, dtype=np.complex128)), 2)
    rs, _ = tf.multilayer_stack_rt(*layers, 0.55, 's', 1.0, aoi=aoi)
    rp, _ = tf.multilayer_stack_rt(*layers, 0.55, 'p', 1.0, aoi=aoi)
    assert rel(rs, rs_r) < 1e-12 and rel(rp, rp_r) < 1e-12
    J = jones(host(rs), host(rp), lambda s: np.zeros(s, dtype=np.complex128))
    got = pol.jones_adapter(P.focus)(J, 2)
    assert rel(got, want) < 1e-10
