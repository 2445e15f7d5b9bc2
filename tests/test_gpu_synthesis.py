"""GPU parity of the SURVEY.md 8(f) rank-3 row -- pupil synthesis on the device (grids, circular masks, Jacobi and
Zernike recurrences, coefficient-weighted Zernike sums) -- against the reference's golden outputs
(tests/golden/synthesis.npz) and the CPU oracle, then end to end: coefficients -> OPD -> pupil -> focus against the
reference's stored C1 field.

Tolerances (relative L-inf): fp64 vs the reference's fp64 golden 1e-12; fp32 storage vs the fp64 golden 1e-6."""
import numpy as np
import pytest
import torch

import prysm_oracle as O
from conftest import rel_linf, load_golden
from gpu_fixtures import pb, host  # noqa: F401

pytestmark = pytest.mark.gpu
HeNe = 0.6328


@pytest.fixture(scope='module')
def gold():
    return load_golden('synthesis.npz')


def setprec(pb, prec):
    pb.config.precision = prec
    return (np.float64, 1e-12) if prec == 64 else (np.float32, 1e-6)


@pytest.mark.parametrize('prec', [64, 32])
def test_grids_and_masks(pb, gold, prec):
    rdt, tol = setprec(pb, prec)
    g = gold
    C, G = pb.coordinates, pb.geometry
    x, y = C.make_xy_grid((33, 40), dx=0.06)
    assert x.dtype == (torch.float64 if prec == 64 else torch.float32) and tuple(x.shape) == (33, 40)
    if prec == 64:
        assert (host(x) == g['grid_x']).all() and (host(y) == g['grid_y']).all()        # exact: one rounding per op
    else:
        assert (host(x) == (O.fftrange(40, np.float32) * np.float32(0.06))[None, :]).all()
    r, t = C.cart_to_polar(x, y)
    assert rel_linf(host(r), g['grid_r']) < tol and rel_linf(host(t), g['grid_t']) < tol
    r2, t2 = C.make_polar_grid((33, 40), dx=0.06)
    assert torch.equal(r2, r) and torch.equal(t2, t)
    xv, yv = C.make_xy_grid((33, 40), dx=0.06, grid=False)
    assert tuple(xv.shape) == (40,) and tuple(yv.shape) == (33,)
    rv, tv = C.cart_to_polar(xv, yv)                                                # vectors -> grid
    assert torch.equal(rv, r)
    xd, yd = C.make_xy_grid(32, diameter=2.0)
    assert rel_linf(host(xd), g['grid_xd']) < tol and rel_linf(host(yd), g['grid_yd']) < tol
    m = G.circle(1.0, r)
    assert m.dtype == torch.bool
    if prec == 64:
        assert (host(m) == g['circle']).all()
        assert rel_linf(host(G.antialias(G.circle_sdf(1.0, r), 0.06)), g['grey']) < tol
        assert rel_linf(host(G.grey_circle(1.0, r, 0.06)), g['grey']) < tol
    else:
        assert (host(m) != g['circle']).sum() <= 2          # a sample exactly on the edge may flip at fp32
        assert np.abs(host(G.grey_circle(1.0, r, 0.06)) - g['grey']).max() < 5e-6


@pytest.mark.parametrize('prec', [64, 32])
@pytest.mark.parametrize('i', range(4))
def test_jacobi(pb, gold, prec, i):
    rdt, tol = setprec(pb, prec)
    al, be = (float(v) for v in gold[f'jac{i}_ab'])
    x = gold['jac_x'].astype(rdt)
    got = pb.polynomials.jacobi_seq([0, 1, 2, 5, 9, 14], al, be, x)
    assert tuple(got.shape) == (6, 65)
    assert rel_linf(host(got), gold[f'jac{i}']) < tol * 3
    assert rel_linf(host(pb.polynomials.jacobi(9, al, be, x)), gold[f'jac{i}'][4]) < tol * 3
    assert rel_linf(host(pb.polynomials.jacobi_seq([5], al, be, x)), gold[f'jac{i}'][3:4]) < tol * 3
    with pytest.raises(pb.B200Error):
        pb.polynomials.jacobi(121, al, be, x)


@pytest.mark.parametrize('prec', [64, 32])
def test_zernike_seq_and_sum(pb, gold, prec):
    rdt, tol = setprec(pb, prec)
    g = gold
    Z = pb.polynomials
    nms = [tuple(int(v) for v in nm) for nm in g['z_nms']]
    assert nms == [Z.noll_to_nm(j) for j in range(1, 38)]
    r, t = (g['grid_r'] / 1.2).astype(rdt), g['grid_t'].astype(rdt)
    ztol = tol * 5                     # radial order 7: the recurrence amplifies the input rounding a few times
    assert rel_linf(host(Z.zernike_nm_seq(nms, r, t, norm=True)), g['z_seq_norm']) < ztol
    assert rel_linf(host(Z.zernike_nm_seq(nms, r, t, norm=False)), g['z_seq_raw']) < ztol
    assert rel_linf(host(Z.zernike_nm(5, -3, r, t)), g['z_single']) < ztol
    x, y = (g['grid_x'] / 1.2).astype(rdt), (g['grid_y'] / 1.2).astype(rdt)
    s = Z.zernike_sum(g['z_coefs'], nms, x, y)
    assert rel_linf(host(s), g['z_sum']) < ztol
    # the sum equals the weighted mode sum of the materialised basis (the reference's two-step route)
    basis = Z.zernike_nm_seq(nms, r, t)
    assert rel_linf(host(Z.sum_of_2d_modes(basis, g['z_coefs'].astype(rdt))), g['z_sum']) < ztol
    assert float(Z.zernike_sum([], [], x, y).abs().max()) == 0.0
    assert float(Z.zernike_sum([0.0, 0.0], [(2, 0), (2, 2)], x, y).abs().max()) == 0.0
    with pytest.raises(ValueError):
        Z.zernike_nm(3, 2, r, t)                     # n - |m| must be even
    assert Z.zernike_norm(2, 0) == pytest.approx(np.sqrt(3)) and Z.zernike_norm(3, 1) == pytest.approx(np.sqrt(8))
    assert Z.fringe_to_nm(9) == (4, 0)


def test_many_modes_split_over_plans(pb):
    """More modes than one kernel plan holds (96 terms / 64 recurrence steps): Noll 1..231 (n <= 20)."""
    pb.config.precision = 64
    Z = pb.polynomials
    nms = [Z.noll_to_nm(j) for j in range(1, 232)]
    x, y = O.make_xy_grid(48, diameter=2.0)
    r, t = O.cart_to_polar(x, y)
    ref = O.zernike_nm_seq(nms, r, t)
    got = Z.zernike_nm_seq(nms, r, t)
    assert rel_linf(host(got), ref) < 1e-11
    c = np.random.default_rng(5).standard_normal(231)
    assert rel_linf(host(Z.zernike_sum(c, nms, x, y)), O.zernike_sum(c, nms, x, y)) < 1e-11


def test_baseline_pupil_from_coefficients_to_focus(pb):
    """The SURVEY 8(d) pupil built entirely on the device from 36 coefficients, then C1 (256^2 -> 512^2, fp64)
    against the reference's stored field window: coefficients are the only host input."""
    pb.config.precision = 64
    N = 256
    C, G, Z, P = pb.coordinates, pb.geometry, pb.polynomials, pb.propagation
    x, y = C.make_xy_grid(N, diameter=10.0)
    r, _ = C.cart_to_polar(x, y)
    amp = G.circle(5.0, r)
    coefs = np.random.default_rng(20260923).normal(0, 30.0, 36)
    nms = [Z.noll_to_nm(j) for j in range(2, 38)]
    opd = Z.zernike_sum(coefs, nms, x / 5.0, y / 5.0)
    amp_o, opd_o, dx = O.synthetic_pupil(N, np.float64)
    assert (host(amp) == amp_o).all()
    assert np.abs((host(opd) - opd_o) * amp_o).max() < 1e-9
    psf = P.Wavefront.from_amp_and_phase(amp, opd, HeNe, dx).focus(100.0, Q=2)
    g = load_golden('full_c1.npz')
    cy = psf.data.shape[0] // 2
    assert rel_linf(host(psf.data[cy - 32:cy + 32, cy - 32:cy + 32]), g['field_win']) < 1e-9
