"""GPU: the Forbes polynomials (prysm_b200.qpoly) against the reference's fp64 fixtures (tests/golden/qpoly*.npz), against
their own basis and finite differences, one launch per call, argument checks before any launch, and a freeform pupil
taken to focus against the reference's host pipeline.

Tolerances (relative L-inf per plane, over the plane's largest magnitude): fp64 vs the reference's fp64 fixtures
1e-12.  fp32 storage (the inputs rounded once to float32, the recurrences still in fp64, the result rounded once):
FP32_BOUND, 1.5x the largest figure measured on an H100 over every plane of every case; the error is the input
rounding carried through the order-12 (radial) and |m| = 20 recurrences."""
import numpy as np
import pytest
import torch

from conftest import load_golden, within
import qpoly_oracle as O
from gpu_fixtures import host

pytestmark = pytest.mark.gpu
FP32_BOUND = 3.5e-6      # measured 2.3e-6 (H100 80GB HBM3, 700 W)


@pytest.fixture(scope='module')
def gold():
    return load_golden('qpoly.npz')


@pytest.fixture(scope='module')
def Q():
    if not torch.cuda.is_available():
        pytest.skip('needs a CUDA device')
    from prysm_b200 import qpoly
    return qpoly


def plane_err(got, ref):
    """Largest over the leading-axis planes of max|got - ref| / max|ref| (absolute where a plane is all zero)."""
    got, ref = np.asarray(got, dtype=np.float64), np.asarray(ref)
    got, ref = got.reshape((-1,) + ref.shape[-2:]), ref.reshape((-1,) + ref.shape[-2:])
    assert got.shape == ref.shape
    err = 0.0
    for a, b in zip(got, ref):
        den = float(np.abs(b).max())
        err = max(err, float(np.abs(a - b).max()) / (den if den > 0 else 1.0))
    return err


def cases(Q, g, grid, dt):
    """name -> (engine output as numpy, reference fixture) for every function on one grid, inputs of dtype dt."""
    x, y, r, t = (torch.as_tensor(g[f'{grid}_{k}'].astype(dt)).cuda() for k in 'xyrt')
    out = {}
    out['qbfs'] = Q.Qbfs_seq(O.NS, r)
    out['qbfs_der'] = Q.Qbfs_der_seq(O.NS, r)
    out['qcon'] = Q.Qcon_seq(O.NS, r)
    out['qcon_der'] = Q.Qcon_der_seq(O.NS, r)
    out['q2d'] = Q.Q2d_seq(O.NMS, r, t)
    out['q2d_dr'], out['q2d_dt'] = Q.Q2d_der_seq(O.NMS, r, t)
    out['q2d_dx'], out['q2d_dy'] = Q.Q2d_der_xy_seq(O.NMS, x, y)
    for name, c in O.RADIAL_SUMS.items():
        out[f'zbfs_{name}'] = Q.compute_z_Qbfs(c, r, r * r)
        out[f'zbfs_{name}_z'], out[f'zbfs_{name}_dr'] = Q.compute_z_zprime_Qbfs(c, r, r * r)
        out[f'zcon_{name}_z'], out[f'zcon_{name}_dr'] = Q.compute_z_zprime_Qcon(c, r, r * r)
    for name, (cm0, ams, bms) in O.Q2D_SUMS.items():
        out[f'z2d_{name}'] = Q.compute_z_Q2d(cm0, ams, bms, r, t)
        out[f'z2d_{name}_z'], out[f'z2d_{name}_dr'], out[f'z2d_{name}_dt'] = Q.compute_z_zprime_Q2d(cm0, ams, bms, r, t)
    for k, v in out.items():
        assert v.dtype == (torch.float64 if dt == np.float64 else torch.float32), k
    return {k: (host(v), g[f'{grid}_{k}']) for k, v in out.items()}


@pytest.mark.parametrize('grid', ['odd', 'even'])
def test_fixtures_fp64(Q, gold, grid):
    for k, (got, ref) in cases(Q, gold, grid, np.float64).items():
        assert plane_err(got, ref) < 1e-12, k


@pytest.mark.parametrize('grid', ['odd', 'even'])
def test_fixtures_fp32(Q, gold, grid):
    worst = max(plane_err(got, ref) for got, ref in cases(Q, gold, grid, np.float32).values())
    within(f'qpoly_fp32_{grid}', worst, FP32_BOUND)


def test_sums_equal_the_weighted_basis(Q, gold):
    r, t = (torch.as_tensor(gold[f'odd_{k}']).cuda() for k in 'rt')
    for name, c in O.RADIAL_SUMS.items():
        ns = list(range(len(c)))
        z, dr = Q.compute_z_zprime_Qbfs(c, r)
        assert plane_err(host(z), np.tensordot(c, host(Q.Qbfs_seq(ns, r)), 1)) < 1e-13
        assert plane_err(host(dr), np.tensordot(c, host(Q.Qbfs_der_seq(ns, r)), 1)) < 1e-13
        z, dr = Q.compute_z_zprime_Qcon(c, r)
        assert plane_err(host(z), np.tensordot(c, host(Q.Qcon_seq(ns, r)), 1)) < 1e-13
        assert plane_err(host(dr), np.tensordot(c, host(Q.Qcon_der_seq(ns, r)), 1)) < 1e-13
    for name, (cm0, ams, bms) in O.Q2D_SUMS.items():
        nms = [(n, 0) for n in range(len(cm0))]
        coefs = list(cm0)
        for i, (a, b) in enumerate(zip(ams, bms)):
            nms += [(n, i + 1) for n in range(len(a))] + [(n, -(i + 1)) for n in range(len(b))]
            coefs += list(a) + list(b)
        z, dr, dt = Q.compute_z_zprime_Q2d(cm0, ams, bms, r, t)
        bdr, bdt = Q.Q2d_der_seq(nms, r, t)
        assert plane_err(host(z), np.tensordot(coefs, host(Q.Q2d_seq(nms, r, t)), 1)) < 1e-13, name
        assert plane_err(host(dr), np.tensordot(coefs, host(bdr), 1)) < 1e-13, name
        assert plane_err(host(dt), np.tensordot(coefs, host(bdt), 1)) < 1e-13, name


def test_derivatives_against_finite_differences(Q):
    h = 1e-6
    rng = np.random.default_rng(3)
    rv = torch.as_tensor(rng.uniform(0.05, 1.0, 400)).cuda()
    tv = torch.as_tensor(rng.uniform(-np.pi, np.pi, 400)).cuda()
    ns = [0, 1, 2, 5, 9]
    for seq, der in ((Q.Qbfs_seq, Q.Qbfs_der_seq), (Q.Qcon_seq, Q.Qcon_der_seq)):
        fd = (host(seq(ns, rv + h)) - host(seq(ns, rv - h))) / (2 * h)
        assert plane_err(host(der(ns, rv)), fd) < 1e-7
    nms = [(0, 0), (4, 0), (2, 1), (6, 1), (3, -2), (5, 3), (2, -7), (1, 12)]
    dr, dt = Q.Q2d_der_seq(nms, rv, tv)
    fdr = (host(Q.Q2d_seq(nms, rv + h, tv)) - host(Q.Q2d_seq(nms, rv - h, tv))) / (2 * h)
    fdt = (host(Q.Q2d_seq(nms, rv, tv + h)) - host(Q.Q2d_seq(nms, rv, tv - h))) / (2 * h)
    assert plane_err(host(dr), fdr) < 1e-7
    assert plane_err(host(dt), fdt) < 1e-7
    x, y = rv * torch.cos(tv), rv * torch.sin(tv)
    dx, dy = Q.Q2d_der_xy_seq(nms, x, y)
    # chain rule: d/dx = cos t d/dr - sin t / r d/dt, d/dy = sin t d/dr + cos t / r d/dt
    c, s, r = host(torch.cos(tv)), host(torch.sin(tv)), host(rv)
    assert plane_err(host(dx), c * host(dr) - s / r * host(dt)) < 1e-11
    assert plane_err(host(dy), s * host(dr) + c / r * host(dt)) < 1e-11

    def polar(xx, yy):
        return torch.hypot(xx, yy), torch.atan2(yy, xx)

    fdx = (host(Q.Q2d_seq(nms, *polar(x + h, y))) - host(Q.Q2d_seq(nms, *polar(x - h, y)))) / (2 * h)
    fdy = (host(Q.Q2d_seq(nms, *polar(x, y + h))) - host(Q.Q2d_seq(nms, *polar(x, y - h)))) / (2 * h)
    assert plane_err(host(dx), fdx) < 1e-7
    assert plane_err(host(dy), fdy) < 1e-7


def test_der_xy_finite_at_origin(Q, gold):
    z = torch.zeros(5, dtype=torch.float64, device='cuda')
    nms = [(n, m) for m in range(-6, 7) for n in range(6)]
    dx, dy = Q.Q2d_der_xy_seq(nms, z, z)
    assert torch.isfinite(dx).all() and torch.isfinite(dy).all()
    # and equal to the reference there (the fixtures' origin sample)
    i = np.argwhere(gold['odd_r'] == 0)[0]
    x, y = (torch.as_tensor(gold[f'odd_{k}']).cuda() for k in 'xy')
    dx, dy = Q.Q2d_der_xy_seq(O.NMS, x, y)
    ref = gold['odd_q2d_dx'][:, i[0], i[1]]
    assert np.abs(host(dx)[:, i[0], i[1]] - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max())


def test_one_launch_per_call(Q, gold):
    from prysm_b200 import _ops
    x, y, r, t = (torch.as_tensor(gold[f'even_{k}']).cuda() for k in 'xyrt')
    cm0, ams, bms = O.Q2D_SUMS['mixed']
    calls = [lambda: Q.Qbfs_seq(O.NS, r), lambda: Q.Qbfs_der_seq(O.NS, r), lambda: Q.Qcon_seq(O.NS, r),
             lambda: Q.Qcon_der_seq(O.NS, r), lambda: Q.Q2d_seq(O.NMS, r, t), lambda: Q.Q2d_der_seq(O.NMS, r, t),
             lambda: Q.Q2d_der_xy_seq(O.NMS, x, y), lambda: Q.compute_z_Qbfs([1.0, 0.5], r),
             lambda: Q.compute_z_zprime_Qbfs([1.0, 0.5], r), lambda: Q.compute_z_zprime_Qcon([1.0, 0.5], r),
             lambda: Q.compute_z_Q2d(cm0, ams, bms, r, t), lambda: Q.compute_z_zprime_Q2d(cm0, ams, bms, r, t),
             lambda: Q.compute_z_Q2d([0.0], [[0.0]], [[0.0]], r, t)]
    for call in calls:
        call()                                              # warm (handle creation)
        before = _ops.launch_count()
        call()
        assert _ops.launch_count() - before == 1


def test_validation_before_any_launch(Q):
    from prysm_b200 import _ops, B200Error
    r = torch.linspace(0, 1, 50, dtype=torch.float64, device='cuda')
    Q.Qbfs_seq([1], r)
    before = _ops.launch_count()
    with pytest.raises(ValueError):
        Q.Qbfs_seq([2, -1], r)
    with pytest.raises(ValueError):
        Q.Q2d_seq([(-1, 2)], r, r)
    with pytest.raises(B200Error):
        Q.Qcon_seq([65], r)
    with pytest.raises(B200Error):
        Q.Q2d_seq([(0, 65)], r, r)
    with pytest.raises(B200Error):                          # 5 recurrences x 64 orders > 256 steps
        Q.Q2d_seq([(63, m) for m in range(1, 6)], r, r)
    with pytest.raises(B200Error):
        Q.compute_z_Qbfs([0.0] * 65 + [1.0], r)
    assert _ops.launch_count() == before


def test_unsorted_orders_return_their_planes(Q):
    """The reference's 1-D sequences assume ascending ns; the engine returns plane i for ns[i] in any order."""
    r = torch.linspace(0, 1, 101, dtype=torch.float64, device='cuda')
    ns = [8, 0, 3, 3, 1]
    for seq in (Q.Qbfs_seq, Q.Qbfs_der_seq, Q.Qcon_seq, Q.Qcon_der_seq):
        got = seq(ns, r)
        for i, n in enumerate(ns):
            assert torch.equal(got[i], seq([n], r)[0])
    got = Q.Q2d_seq([(2, 2), (0, 0), (2, 2)], r, r)
    assert torch.equal(got[0], got[2]) and torch.equal(got[0], Q.Q2d(2, 2, r, r))


def test_freeform_pupil_to_psf(Q, gold):
    """coefficients -> compute_z_Q2d -> OPD -> Wavefront.from_amp_and_phase -> focus, all on the device, against the
    reference's host pipeline."""
    import prysm_b200 as pb
    pb.config.precision = 64
    amp, u, t, dx = O.psf_inputs()
    cm0, ams, bms = Q.Q2d_nm_c_to_a_b(O.PSF_NMS, O.PSF_COEFS)
    opd = Q.compute_z_Q2d(cm0, ams, bms, torch.as_tensor(u).cuda(), torch.as_tensor(t).cuda())
    assert plane_err(host(opd), gold['psf_opd']) < 1e-12
    wf = pb.Wavefront.from_amp_and_phase(torch.as_tensor(amp).cuda(), opd * 1e3, O.PSF_WVL, dx)
    psf = wf.focus(O.PSF_EFL, Q=O.PSF_Q).intensity
    within('qpoly_freeform_psf_fp64', plane_err(host(psf.data), gold['psf']), 1e-12)
