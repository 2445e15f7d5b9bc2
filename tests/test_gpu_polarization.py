"""GPU: Jones calculus on the device (prysm_b200.polarization) against the reference's fixtures
(tests/golden/polarization*.npz, written by tests/polarization_oracle.py), the batched Jones propagation against the
engine's scalar calls, the layout and launch bookkeeping, adjoint identities, and the drop-in path executed against
the unmodified reference."""
import os

import numpy as np
import pytest
import torch

from conftest import load_golden, rel_linf, within
from gpu_fixtures import pb  # noqa: F401
import polarization_oracle as O
import reference

pytestmark = pytest.mark.gpu

BOUND = {32: 1e-6, 64: 1e-12}
# The coronagraph's final plane is what the vortex lets through: its peak is 20x below that of the same chain without
# the vortex (1.00 against 20.3 in the fixture case), so the fp32 transforms' error, ~1e-7 of the field they carry,
# is ~2e-6 of the suppressed output.  Measured on an H100: 2.0e-6 (final plane), 1.3e-6 (its sums of |.|).
BOUND_SUPPRESSED_32 = 3e-6


@pytest.fixture(scope='module')
def golden():
    return load_golden('polarization.npz')


def to_numpy(t):
    return t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)


def inputs_at(prec):
    """The fixture inputs at the working precision (the fp64 fixtures then measure the engine, not input rounding
    plus the engine: at precision 32 the difference includes one rounding of each input)."""
    g = O.inputs()
    if prec == 32:
        g = {k: v.astype(np.complex64 if np.iscomplexobj(v) else np.float32) for k, v in g.items()}
    return g


@pytest.mark.parametrize('prec', [32, 64])
def test_every_fixture(pb, golden, prec):
    pb.config.precision = prec
    g = inputs_at(prec)
    rdt = np.float32 if prec == 32 else np.float64
    cdt = np.complex64 if prec == 32 else np.complex128

    def asarray(a):
        return pb.asdevice(np.asarray(a).astype(cdt if np.iscomplexobj(a) else rdt))
    mine = O.run(pb.polarization, pb.propagation, g, to_numpy=to_numpy, asarray=asarray)
    mine['diattenuator_plane'] = to_numpy(pb.polarization.linear_diattenuator(g['alpha'], theta=-0.6, shape=O.SHAPE))
    assert sorted(mine) == sorted(golden)
    bad = {}
    for k in sorted(golden):
        assert mine[k].shape == golden[k].shape, k
        err = rel_linf(mine[k], golden[k])
        bound = BOUND_SUPPRESSED_32 if prec == 32 and k.startswith('vvc_final') else BOUND[prec]
        if err < bound:
            within(f'polarization{prec}_{k}', err, bound)
        else:
            bad[k] = err
    assert not bad, {k: f'{v:.2e}' for k, v in bad.items()}


def test_vvr_leaves_theta_alone(pb):
    theta = pb.asdevice(O.inputs()['theta'])
    before = theta.clone()
    pb.polarization.vector_vortex_retarder(2, theta)
    assert torch.equal(theta, before)


def jones_field(pb, n, prec=32, seed=1):
    """An element-planar Jones field: a scalar field through a per-pixel retarder."""
    pb.config.precision = prec
    rng = np.random.default_rng(seed)
    f = rng.standard_normal((n, n)) + 1j * rng.standard_normal((n, n))
    f = f.astype(np.complex64 if prec == 32 else np.complex128)
    ret = rng.uniform(0, 1, (n, n))
    return pb.polarization.apply_polarization_optic(f, pb.polarization.linear_retarder(ret, theta=0.2, shape=(n, n)))


@pytest.mark.parametrize('n', [256, 512])
def test_jones_focus_is_the_scalar_focus_per_element(pb, n):
    P, pol = pb.propagation, pb.polarization
    J = jones_field(pb, n)
    Jf = pol.jones_adapter(P.focus)(J, 2)
    Jp = pol.jones_adapter(P.unfocus)(Jf, 1)
    for i in range(2):
        for j in range(2):
            assert torch.equal(Jf[..., i, j], P.focus(J[..., i, j], 2)), (i, j)
            assert torch.equal(Jp[..., i, j], P.unfocus(Jf[..., i, j], 1)), (i, j)
    pb.config.precision = 64


def test_layout_and_launches(pb):
    P, pol = pb.propagation, pb.polarization
    n = 256
    J = jones_field(pb, n)
    stack = J.permute(2, 3, 0, 1).reshape(4, n, n).clone()
    focus, unfocus = pol.jones_adapter(P.focus), pol.jones_adapter(P.unfocus)

    def launches(fn, *args):
        torch.cuda.synchronize()
        n0 = pb._ops.launch_count()
        out = fn(*args)
        return out, pb._ops.launch_count() - n0
    _, batch = launches(P.focus, stack, 2)
    _, batch_back = launches(P.unfocus, P.focus(stack, 2), 2)
    Jf, d = launches(focus, J, 2)
    assert d == batch                          # a planar-backed field: no pb_jones_planar
    Jb, d = launches(unfocus, Jf, 2)
    assert d == batch_back
    host = to_numpy(J).copy()                  # interleaved contiguous (n, n, 2, 2) on the host
    assert host.flags.c_contiguous
    Jh, d = launches(focus, host, 2)
    assert d == batch + 1                      # exactly one conversion
    assert torch.equal(Jh, Jf)
    for out, m in ((Jf, 2 * n), (Jb, 4 * n), (Jh, 2 * n)):
        assert tuple(out.shape) == (m, m, 2, 2)
        assert out.permute(2, 3, 0, 1).is_contiguous()     # element-planar storage
    pb.config.precision = 64


def inner(a, b):
    return complex(np.vdot(to_numpy(b).ravel(), to_numpy(a).ravel()))     # sum a * conj(b)


def test_adjoint_identities(pb):
    pb.config.precision = 64
    P, pol = pb.propagation, pb.polarization
    rng = np.random.default_rng(5)

    def rand(*shape):
        return rng.standard_normal(shape) + 1j * rng.standard_normal(shape)
    A, B, X, Y = (rand(37, 53, 2, 2) for _ in range(4))
    lhs, rhs = inner(pol.jones_matmul(A, X), Y), inner(X, pol.jones_matmul(A, Y, adjoint_a=True))
    within('polarization_adjoint_matmul_b', abs(lhs - rhs) / abs(lhs), 1e-12)
    lhs, rhs = inner(pol.jones_matmul(X, B), Y), inner(X, pol.jones_matmul(Y, B, adjoint_b=True))
    within('polarization_adjoint_matmul_a', abs(lhs - rhs) / abs(lhs), 1e-12)
    ex = P.prepare_executor(0.01, (48, 64), 0.5, (40, 56), 0.6, 50.0)
    X, Y = rand(48, 64, 2, 2), rand(40, 56, 2, 2)
    fwd = pol.jones_adapter(P.focus_dft)(X, ex)
    adj = pol.jones_adapter(P.focus_dft_adjoint)(Y, ex)
    assert tuple(fwd.shape) == (40, 56, 2, 2) and tuple(adj.shape) == (48, 64, 2, 2)
    lhs, rhs = inner(fwd, Y), inner(X, adj)
    within('polarization_adjoint_focus_dft', abs(lhs - rhs) / abs(lhs), 1e-12)
    # the FFT adjoints run as one batched call with a crop
    Xf, Yf = rand(32, 40, 2, 2), rand(64, 80, 2, 2)
    lhs = inner(pol.jones_adapter(P.focus)(Xf, 2), Yf)
    rhs = inner(Xf, pol.jones_adapter(P.focus_adjoint)(Yf, 2))
    within('polarization_adjoint_focus', abs(lhs - rhs) / abs(lhs), 1e-12)


def test_adapter_refuses_other_ranks(pb):
    pol, P = pb.polarization, pb.propagation
    with pytest.raises(ValueError):
        pol.jones_adapter(P.focus)(np.zeros((4, 4, 2, 3)), 2)
    with pytest.raises(ValueError):
        pol.jones_adapter(P.focus)(np.zeros((2, 4, 4, 2, 2)), 2)


# ---- drop-in: the reference's own test_make_propagation_polarized user code ------------------------------------

def polarized_user_code():
    """tests/x/test_polarization.py:131-176 of the reference, returning the Jones results as host arrays."""
    from prysm.coordinates import make_xy_grid, cart_to_polar
    from prysm.geometry import circle
    from prysm.mathops import array_to_true_numpy
    import prysm.x.polarization as pol
    xi, eta = make_xy_grid(256, diameter=10)
    r, t = cart_to_polar(xi, eta)
    A = circle(5, r)
    wave = 1
    samples = A.shape[0]
    dx = 5 / samples
    J = np.zeros([*A.shape, 2, 2])
    J[..., 0, 0] = A
    J[..., 1, 1] = A
    pol.add_jones_propagation()
    from prysm.propagation import focus, unfocus, angular_spectrum, focus_dft, unfocus_dft, prepare_executor
    J_psf = focus(J, Q=2)
    J_pupil = unfocus(J_psf, Q=1)
    J_prop = angular_spectrum(J_pupil, wvl=wave, dx=dx, z=5e1, Q=1)
    mdft = prepare_executor(pupil_dx=dx, pupil_samples=samples, focal_dx=1000e-3, focal_samples=256, wavelength=wave,
                            efl=50)
    J_psf_fixed = focus_dft(J, mdft)
    J_pupil_fixed = unfocus_dft(J_psf_fixed, mdft)
    return [array_to_true_numpy(v) for v in (J_psf, J_pupil, J_prop, J_psf_fixed, J_pupil_fixed)]


def test_dropin_add_jones_propagation(pb):
    if not reference.installed():
        pytest.skip('oracle/_ref is not installed')
    with reference.loaded():
        import prysm.propagation as pprop
        import prysm.x.polarization  # noqa: F401
        assert os.path.realpath(pprop.__file__).startswith(os.path.realpath(reference.REF))
        from prysm_b200 import mathops
        saved = {n: getattr(pprop, n) for n in prysm.x.polarization.supported_propagation_funcs}
        try:
            want = polarized_user_code()                     # numpy, the reference's adapter
        finally:
            for n, f in saved.items():
                setattr(pprop, n, f)
        mathops.set_backend_to_b200()
        try:
            got = polarized_user_code()                      # the engine's functions, wrapped by the engine's adapter
            assert prysm.x.polarization.jones_adapter is pb.polarization.jones_adapter
        finally:
            mathops.set_backend_to_defaults()
        assert all(getattr(pprop, n) is f for n, f in saved.items())
        for i, (g, w) in enumerate(zip(got, want)):
            assert g.shape == w.shape
            within(f'polarization_dropin_{i}', rel_linf(g, w), 1e-6)
