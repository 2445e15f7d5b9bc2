"""GPU: the orthogonal polynomials, Zernike derivatives and polynomial sums (prysm_b200.polynomials, .orthopoly)
against the reference's fp64 fixtures (tests/golden/polynomials*.npz), against their own basis and finite
differences, one launch per call, argument checks before any launch, a captured graph, and two end-to-end cases: a
36-mode slope map and an XY pupil taken to focus, both against the reference's host pipeline.

Tolerances (relative L-inf per plane, over the plane's largest magnitude): fp64 vs the reference's fp64 fixtures
1e-12.  fp32 storage (inputs rounded once to float32, recurrences still in fp64, each output rounded once):
FP32_BOUND, 1.5x the largest figure measured on an H100 over every plane of every case; the error is the input
rounding carried through orders up to 34 (Hermite on [-6, 6] and Laguerre on [0, 20] amplify it most)."""
import numpy as np
import pytest
import torch

from conftest import load_golden, within
import polynomials_oracle as O
from gpu_fixtures import host

pytestmark = pytest.mark.gpu
FP32_BOUND = 5.3e-6      # measured 3.5e-6 (H100 80GB HBM3, 700 W)


@pytest.fixture(scope='module')
def gold():
    return load_golden('polynomials.npz')


@pytest.fixture(scope='module')
def P():
    if not torch.cuda.is_available():
        pytest.skip('needs a CUDA device')
    from prysm_b200 import polynomials
    return polynomials


def dev(a, dt=np.float64):
    return torch.as_tensor(np.asarray(a).astype(dt)).cuda()


def plane_err(got, ref):
    """Largest over the planes (all axes but the last 1 or 2) of max|got - ref| / max|ref| (absolute where a plane is
    all zero)."""
    got, ref = np.asarray(got, dtype=np.float64), np.asarray(ref)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    tail = 1 if ref.shape[-1] == O.LINE else 2
    got, ref = got.reshape((-1,) + ref.shape[-tail:]), ref.reshape((-1,) + ref.shape[-tail:])
    err = 0.0
    for a, b in zip(got, ref):
        den = float(np.abs(b).max())
        err = max(err, float(np.abs(a - b).max()) / (den if den > 0 else 1.0))
    return err


def extra(fam):
    return O.FAMILIES[fam][1]


def cases(P, g, dt):
    """name -> (engine output as numpy, reference fixture) for every function, inputs of dtype dt."""
    out = {}
    for fam in O.FAMILIES:
        x = dev(g[f'line_{fam}_x'], dt)
        out[f'line_{fam}'] = getattr(P, f'{fam}_seq')(O.NS, *extra(fam), x)
        out[f'line_{fam}_der'] = getattr(P, f'{fam}_der_seq')(O.NS, *extra(fam), x)
    x = dev(g['line_jacobi_x'], dt)
    out['line_jacobi_wd_v'], out['line_jacobi_wd_d'] = P.jacobi_seq_with_der(O.NS, O.ALPHA, O.BETA, x)
    for name, s in O.CLEN_S.items():
        out[f'clen_{name}'] = P.jacobi_sum_clenshaw(s, O.ALPHA, O.BETA, x)
        for j in O.CLEN_J:
            out[f'clen_{name}_j{j}'] = P.jacobi_sum_clenshaw_der(s, O.ALPHA, O.BETA, x, j=j)
    for grid in ('odd', 'even'):
        x, y, r, t = (dev(g[f'{grid}_{k}'], dt) for k in 'xyrt')
        out[f'{grid}_zder'] = P.zernike_nm_der_seq(O.ZNMS, r, t)
        out[f'{grid}_zder_xy'] = P.zernike_nm_der_xy_seq(O.ZNMS, x, y)
        out[f'{grid}_zder_raw'] = P.zernike_nm_der_seq(O.ZNMS, r, t, norm=False)
        for name, (c, nms) in O.ZSUMS.items():
            out[f'{grid}_zsum_{name}'] = torch.stack(P.zernike_sum_der_xy(c, nms, x, y))
        for name, (c, ns) in O.RADIAL.items():
            out[f'{grid}_rad_{name}'] = P.jacobi_radial_sum(c, ns, O.ALPHA, O.BETA, x, y, O.RADIAL_R)
            out[f'{grid}_rad_{name}_der'] = torch.stack(P.jacobi_radial_sum_der_xy(c, ns, O.ALPHA, O.BETA, x, y, O.RADIAL_R))
        for kind in ('', '_der_x', '_der_y', '_der_xy'):
            fn = getattr(P, f'xy{kind}_seq')
            out[f'{grid}_xy{kind}'] = fn(O.XY_MNS, x, y)
            out[f'{grid}_xy{kind}_elem'] = fn(O.XY_MNS, x, y, cartesian_grid=False)
        out[f'{grid}_xysum'] = P.xy_sum(O.XY_COEFS, O.XY_MNS, x, y)
        out[f'{grid}_xysum_der'] = torch.stack(P.xy_sum_der_xy(O.XY_COEFS, O.XY_MNS, x, y))
        out[f'{grid}_xysum_elem'] = P.xy_sum(O.XY_COEFS, O.XY_MNS, x, y, cartesian_grid=False)
        out[f'{grid}_chsum'] = P.cheby1_2d_sum(O.CHEB_COEFS, O.CHEB_MNS, x, y)
        out[f'{grid}_chsum_der'] = torch.stack(P.cheby1_2d_sum_der_xy(O.CHEB_COEFS, O.CHEB_MNS, x, y, *O.CHEB_NORM))
    for k, v in out.items():
        assert v.dtype == (torch.float64 if dt == np.float64 else torch.float32), k
    return {k: (host(v), g[k]) for k, v in out.items()}


def test_fixtures_fp64(P, gold):
    bad = {k: e for k, (got, ref) in cases(P, gold, np.float64).items() if (e := plane_err(got, ref)) >= 1e-12}
    assert not bad, bad


def test_fixtures_fp32(P, gold):
    worst = max(plane_err(got, ref) for got, ref in cases(P, gold, np.float32).values())
    within('polynomials_fp32', worst, FP32_BOUND)


def test_permuted_and_repeated_orders(P, gold):
    """The reference's 1-D sequences assume ascending ns; plane i is ns[i] in any order, repeats included."""
    perm = [5, 0, 9, 2, 2, 7, 1]
    for fam in O.FAMILIES:
        x = dev(gold[f'line_{fam}_x'])
        for suffix, fn in (('', f'{fam}_seq'), ('_der', f'{fam}_der_seq')):
            got = host(getattr(P, fn)([O.NS[i] for i in perm], *extra(fam), x))
            assert plane_err(got, gold[f'line_{fam}{suffix}'][perm]) < 1e-12, (fam, suffix)
    z = P.zernike_nm_der_xy_seq([O.ZNMS[i] for i in (4, 1, 4)], dev(gold['odd_x']), dev(gold['odd_y']))
    assert torch.equal(z[0], z[2])
    assert P.legendre_seq([], dev(gold['line_legendre_x'])).shape == (0, O.LINE)


def test_jacobi_seq_entry_point_is_the_same_kernel(P, gold):
    """pb_jacobi_seq (orders by slot) and pb_poly_seq (orders by plane) run the same recurrence: equal bit for bit."""
    from prysm_b200 import _ops
    for dt in (np.float64, np.float32):
        x = dev(gold['line_jacobi_x'], dt)
        ns = [0, 1, 2, 5, 9, 34, 120]
        assert torch.equal(_ops.jacobi_seq(ns, O.ALPHA, O.BETA, x), P.jacobi_seq(ns, O.ALPHA, O.BETA, x))


def test_sums_equal_the_weighted_basis(P, gold):
    x, y, r, t = (dev(gold[f'odd_{k}']) for k in 'xyrt')
    for name, (c, nms) in O.ZSUMS.items():
        W, dx, dy = (host(v) for v in P.zernike_sum_der_xy(c, nms, x, y))
        basis = host(P.zernike_nm_seq(nms, r, t))
        der = host(P.zernike_nm_der_xy_seq(nms, x, y))
        assert plane_err(W, np.tensordot(c, basis, 1)) < 1e-13, name
        assert plane_err(dx, np.tensordot(c, der[:, 0], 1)) < 1e-13, name
        assert plane_err(dy, np.tensordot(c, der[:, 1], 1)) < 1e-13, name
    for name, (c, ns) in O.RADIAL.items():
        u = 2 * (x * x + y * y) / O.RADIAL_R ** 2 - 1
        z, dzx, _ = (host(v) for v in P.jacobi_radial_sum_der_xy(c, ns, O.ALPHA, O.BETA, x, y, O.RADIAL_R))
        basis = host(P.jacobi_seq(ns[:len(c)], O.ALPHA, O.BETA, u))
        assert plane_err(z, np.tensordot(c, basis, 1)) < 1e-13, name
        dbasis = host(P.jacobi_der_seq(ns[:len(c)], O.ALPHA, O.BETA, u))
        assert plane_err(dzx, np.tensordot(c, dbasis, 1) * 4 * host(x) / O.RADIAL_R ** 2) < 1e-12, name
    z, dzx, dzy = (host(v) for v in P.xy_sum_der_xy(O.XY_COEFS, O.XY_MNS, x, y))
    assert plane_err(z, np.tensordot(O.XY_COEFS, host(P.xy_seq(O.XY_MNS, x, y)), 1)) < 1e-13
    assert plane_err(dzx, np.tensordot(O.XY_COEFS, host(P.xy_der_x_seq(O.XY_MNS, x, y)), 1)) < 1e-13
    assert plane_err(dzy, np.tensordot(O.XY_COEFS, host(P.xy_der_y_seq(O.XY_MNS, x, y)), 1)) < 1e-13
    s = O.CLEN_S['dense']
    xl = dev(gold['line_jacobi_x'])
    basis = host(P.jacobi_seq(range(len(s)), O.ALPHA, O.BETA, xl))
    assert plane_err(host(P.jacobi_sum_clenshaw(s, O.ALPHA, O.BETA, xl)), np.tensordot(s, basis, 1)) < 1e-13
    tab = host(P.jacobi_sum_clenshaw_der(s, O.ALPHA, O.BETA, xl, j=1))
    dbasis = host(P.jacobi_der_seq(range(len(s)), O.ALPHA, O.BETA, xl))
    assert plane_err(tab[1, 0], np.tensordot(s, dbasis, 1)) < 1e-12
    assert np.array_equal(host(P.jacobi_sum_clenshaw_der(s, O.ALPHA, O.BETA, xl, j=0))[0], tab[0])


def test_derivatives_against_finite_differences(P):
    h = 1e-6
    rng = np.random.default_rng(5)
    xl = dev(rng.uniform(-0.95, 0.95, 300))
    ns = [0, 1, 2, 5, 9, 14]
    for fam in O.FAMILIES:
        seq, der = getattr(P, f'{fam}_seq'), getattr(P, f'{fam}_der_seq')
        fd = (host(seq(ns, *extra(fam), xl + h)) - host(seq(ns, *extra(fam), xl - h))) / (2 * h)
        assert plane_err(host(der(ns, *extra(fam), xl)), fd) < 1e-6, fam
    rv, tv = dev(rng.uniform(0.05, 1.0, 300)), dev(rng.uniform(-np.pi, np.pi, 300))
    nms = [(0, 0), (4, 0), (1, 1), (5, -1), (6, 2), (7, -3), (12, 12), (9, -5)]
    d = host(P.zernike_nm_der_seq(nms, rv, tv))
    fdr = (host(P.zernike_nm_seq(nms, rv + h, tv)) - host(P.zernike_nm_seq(nms, rv - h, tv))) / (2 * h)
    fdt = (host(P.zernike_nm_seq(nms, rv, tv + h)) - host(P.zernike_nm_seq(nms, rv, tv - h))) / (2 * h)
    assert plane_err(d[:, 0], fdr) < 1e-7 and plane_err(d[:, 1], fdt) < 1e-7
    x, y = rv * torch.cos(tv), rv * torch.sin(tv)
    dxy = host(P.zernike_nm_der_xy_seq(nms, x, y))
    c, s, r = host(torch.cos(tv)), host(torch.sin(tv)), host(rv)
    # the polar and Cartesian derivatives agree through the chain rule away from the origin
    assert plane_err(dxy[:, 0], c * d[:, 0] - s / r * d[:, 1]) < 1e-11
    assert plane_err(dxy[:, 1], s * d[:, 0] + c / r * d[:, 1]) < 1e-11
    W = lambda xx, yy: host(P.zernike_sum_der_xy(O.ZSUMS['mixed'][0], O.ZSUMS['mixed'][1], xx, yy)[0])  # noqa: E731
    _, wx, wy = (host(v) for v in P.zernike_sum_der_xy(*O.ZSUMS['mixed'], x, y))
    assert plane_err(wx, (W(x + h, y) - W(x - h, y)) / (2 * h)) < 1e-7
    assert plane_err(wy, (W(x, y + h) - W(x, y - h)) / (2 * h)) < 1e-7
    Z = lambda xx, yy: host(P.xy_sum(O.XY_COEFS, O.XY_MNS, xx, yy, cartesian_grid=False))  # noqa: E731
    _, zx, zy = (host(v) for v in P.xy_sum_der_xy(O.XY_COEFS, O.XY_MNS, x, y, cartesian_grid=False))
    assert plane_err(zx, (Z(x + h, y) - Z(x - h, y)) / (2 * h)) < 1e-7
    assert plane_err(zy, (Z(x, y + h) - Z(x, y - h)) / (2 * h)) < 1e-7


def test_one_launch_per_call(P, gold):
    from prysm_b200 import _ops
    x, y, r, t = (dev(gold[f'even_{k}']) for k in 'xyrt')
    xl = dev(gold['line_legendre_x'])
    c, nms = O.ZSUMS['mixed']
    calls = [lambda: P.legendre_seq(O.NS, xl), lambda: P.hermite_H_der_seq(O.NS, xl), lambda: P.laguerre_der_seq(O.NS, 0.5, xl),
             lambda: P.jacobi_seq_with_der(O.NS, 1, 2, xl), lambda: P.jacobi_sum_clenshaw_der([1, 2, 3], 0, 1, xl, j=2),
             lambda: P.zernike_nm_der_seq(O.ZNMS, r, t), lambda: P.zernike_nm_der_xy_seq(O.ZNMS, x, y),
             lambda: P.zernike_sum_der_xy(c, nms, x, y), lambda: P.jacobi_radial_sum_der_xy([1, 2], [0, 2], 0, 0, x, y, 1),
             lambda: P.xy_der_xy_seq(O.XY_MNS, x, y), lambda: P.xy_sum_der_xy(O.XY_COEFS, O.XY_MNS, x, y),
             lambda: P.cheby1_2d_sum_der_xy(O.CHEB_COEFS, O.CHEB_MNS, x, y)]
    for call in calls:
        call()                                              # warm (handle creation)
        before = _ops.launch_count()
        call()
        assert _ops.launch_count() - before == 1
    before = _ops.launch_count()
    assert P.cheby2_seq([], xl).shape == (0, O.LINE) and P.zernike_nm_der_xy_seq([], x, y).shape == (0, 2) + x.shape
    assert _ops.launch_count() == before


def test_validation_before_any_launch(P):
    from prysm_b200 import _ops, B200Error
    x = torch.linspace(-1, 1, 50, dtype=torch.float64, device='cuda')
    P.legendre_seq([1], x)
    before = _ops.launch_count()
    with pytest.raises(ValueError):
        P.legendre_seq([2, -1], x)
    with pytest.raises(B200Error):
        P.hermite_He_seq([121], x)
    with pytest.raises(ValueError):
        P.zernike_nm_der_seq([(3, 2)], x, x)             # n - |m| odd
    with pytest.raises(ValueError):
        P.zernike_nm_der_xy_seq([(2, 4)], x, x)          # |m| > n
    with pytest.raises(ValueError):
        P.jacobi_sum_clenshaw_der([1.0], 0, 0, x, j=9)
    with pytest.raises(IndexError):
        P.jacobi_radial_sum([1.0, 2.0, 3.0], [0, 2], 0, 0, x, x, 1.0)
    assert _ops.launch_count() == before


def test_zernike_sum_der_xy_graph_replays(P, gold):
    from prysm_b200 import graphs
    x, y = dev(gold['odd_x']), dev(gold['odd_y'])
    c, nms = O.ZSUMS['mixed']
    step = graphs.capture(lambda xx, yy: torch.stack(P.zernike_sum_der_xy(c, nms, xx, yy)), x, y)
    direct = torch.stack(P.zernike_sum_der_xy(c, nms, x * 0.5, y * 0.5))
    a = step(x * 0.5, y * 0.5).clone()
    b = step(x * 0.5, y * 0.5).clone()
    assert torch.equal(a, b) and torch.equal(a, direct)


def test_slope_map_end_to_end(P, gold):
    """36 Noll coefficients -> W, dW/dx, dW/dy at 256^2 in one launch, against the reference's zernike_sum_der_xy."""
    x, y, coefs = O.slope_inputs()
    nms = [P.noll_to_nm(j) for j in range(2, 38)]
    got = torch.stack(P.zernike_sum_der_xy(coefs, nms, dev(x), dev(y)))
    ref = np.stack([gold['slope_W'], gold['slope_dx'], gold['slope_dy']])
    within('polynomials_slope_map_fp64', plane_err(host(got), ref), 1e-12)


def test_xy_pupil_to_psf(P, gold):
    """coefficients -> xy_sum -> OPD -> Wavefront.from_amp_and_phase -> focus, all on the device, against the
    reference's host pipeline."""
    import prysm_b200 as pb
    pb.config.precision = 64
    amp, u, w, dx = O.xypsf_inputs()
    opd = P.xy_sum(O.XYPSF_COEFS, O.XYPSF_MNS, dev(u), dev(w))
    assert plane_err(host(opd), gold['xypsf_opd']) < 1e-12
    wf = pb.Wavefront.from_amp_and_phase(dev(amp), opd * 1e3, O.XYPSF_WVL, dx)
    psf = wf.focus(O.XYPSF_EFL, Q=O.XYPSF_Q).intensity
    within('polynomials_xy_psf_fp64', plane_err(host(psf.data), gold['xypsf']), 1e-12)
