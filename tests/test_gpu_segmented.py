"""GPU: the signed-distance geometry and CompositeHexagonalAperture (prysm_b200.geometry, prysm_b200.segmented)
against the reference's fixtures (tests/golden/segmented*.npz), the adjoint's dot-product identity, graph capture
and determinism, and a JWST pupil end to end through focus."""
import numpy as np
import pytest

from conftest import load_golden, rel_linf, within
import reference
import segmented_oracle as O

pytestmark = pytest.mark.gpu
TOL = {32: 1e-6, 64: 1e-12}


@pytest.fixture(scope='module')
def golden():
    return load_golden('segmented.npz')


@pytest.fixture()
def precision(request):
    import prysm_b200 as pb
    pb.config.precision = request.param
    yield request.param
    pb.config.precision = 64


def tonp(t):
    import torch
    return t.cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)


def dtype_of(prec):
    return np.float32 if prec == 32 else np.float64


def mask_mismatch(got, want, sdf64, dx):
    """Samples where two bool masks differ; any such sample must lie within 1e-9 dx of the edge."""
    bad = got != want
    near = np.abs(sdf64) < 1e-9 * dx
    assert not np.any(bad & ~near), f'{int(np.sum(bad & ~near))} mask samples differ away from the edge'
    return int(bad.sum())


@pytest.mark.parametrize('precision', [32, 64], indirect=True)
def test_geometry_matches_the_reference(golden, precision):
    import prysm_b200 as pb
    x, y = (pb.asdevice(a) for a in O.grid(O.SHAPE, O.DX, dtype_of(precision)))
    r = pb.asdevice(np.hypot(*(a.astype(np.float64) for a in O.grid(O.SHAPE, O.DX, dtype_of(precision)))).astype(dtype_of(precision)))
    got = O.geometry_cases(pb.geometry, x, y, r)
    xh, yh = (a.astype(np.float64) for a in O.grid(O.SHAPE, O.DX, dtype_of(precision)))
    rh = tonp(r).astype(np.float64)
    verts = O.regular_vertices(6, 1.07, (-0.05, 0.11), 90, dtype_of(precision))
    sdf_of = {'regpoly_mask': lambda: O.polygon_sdf(verts, xh, yh),                    # fp64 distances of the masks
              'spider_mask': lambda: O.spider_sdf(3, 0.097, xh, yh, rotation=-75),
              'rect_mask': lambda: O.rectangle_sdf(0.61, xh, yh, angle=90),
              'fillet_mask': lambda: O.fillet_sdf(0.9, 0.6, 0.21, xh, yh, rotation=12),
              'annulus_mask': lambda: O.annulus_sdf(0.4, 1.1, rh),
              'offset_circle': lambda: np.hypot(xh - 0.2, yh + 0.1) - 0.7}
    for k, v in got.items():
        want = golden[f'geom{precision}_{k}']
        v = tonp(v)
        assert v.shape == want.shape, (k, v.shape, want.shape)
        if want.dtype == bool:
            n = mask_mismatch(v, want, sdf_of[k](), O.DX)
            assert n == 0, (k, n)
        elif v.size:
            assert v.dtype == dtype_of(precision), (k, v.dtype)
            within(f'geom_{k}_fp{precision}', rel_linf(v, want), TOL[precision])


def test_separable_inputs_give_the_grid_result():
    import prysm_b200 as pb
    x, y = O.grid(O.SHAPE, O.DX, np.float64)
    a = tonp(pb.geometry.polygon_sdf(O.CONCAVE, pb.asdevice(x), pb.asdevice(y)))
    b = tonp(pb.geometry.polygon_sdf(O.CONCAVE, pb.asdevice(x[:1]), pb.asdevice(y[:, :1])))
    assert np.array_equal(a, b)
    assert np.array_equal(a, O.polygon_sdf(O.CONCAVE, x, y)) or rel_linf(a, O.polygon_sdf(O.CONCAVE, x, y)) < 1e-15


def test_combinators_broadcast_and_propagate_nan_like_numpy():
    import prysm_b200 as pb
    a = np.array([[0.5, np.nan, -1.0, 2.0]])
    b = np.array([[np.nan, 0.25, 3.0, -2.0]])
    col = np.array([[1.0], [-0.5]])
    for got, want in ((pb.geometry.union(a, b), np.minimum(a, b)), (pb.geometry.union(b, a), np.minimum(b, a)),
                      (pb.geometry.intersect(a, b), np.maximum(a, b)), (pb.geometry.subtract(a, b), np.maximum(a, -b)),
                      (pb.geometry.union(a, col), np.minimum(a, col)), (pb.geometry.subtract(col, a), np.maximum(col, -a))):
        assert np.array_equal(tonp(got), want, equal_nan=True), (tonp(got), want)


def test_polygon_vertex_limit_is_a_value_error():
    import prysm_b200 as pb
    x, y = (pb.asdevice(a) for a in O.grid(O.SHAPE, O.DX, np.float64))
    t = np.linspace(0, 2 * np.pi, 128, endpoint=False)
    pb.geometry.polygon_sdf(np.stack([np.cos(t), np.sin(t)], 1), x, y)
    t = np.linspace(0, 2 * np.pi, 129, endpoint=False)
    with pytest.raises(ValueError, match='at most 128'):
        pb.geometry.polygon_sdf(np.stack([np.cos(t), np.sin(t)], 1), x, y)


def test_basis_modes_are_broadcast_to_the_window_or_refused():
    """A mode that is a scalar or a row broadcasts against the mask in the reference; the packed basis holds it at
    the window's shape.  A mode that cannot broadcast is refused rather than read past the packed buffer."""
    import prysm_b200 as pb
    cha = adjoint_setup(64)

    def partly_constant(orders, x, y):
        return [pb.asdevice(np.array(1.0)), x[:1] * 0 + 2.0, y]

    cha.prepare_opd_bases(partly_constant, None)
    assert all(tuple(b.shape) == (3,) + tuple(m.shape) for b, m in zip(cha.opd_bases, cha.local_masks))
    c = np.random.default_rng(8).standard_normal((len(cha.windows), 3))
    want = np.zeros(tuple(cha.x.shape))
    for (win, grid, m, cc) in zip(cha.windows, cha.opd_grids, cha.local_masks, c):
        yy = tonp(grid[1])          # the grid the shared basis was made on (the cache is keyed on x and shape only)
        want[win] += (cc[0] + 2 * cc[1] + cc[2] * yy) * tonp(m)
    assert rel_linf(tonp(cha.compose_opd(c)), want) < 1e-13

    def wrong_shape(orders, x, y):
        return [x[:3, :3]]

    with pytest.raises(ValueError, match='does not broadcast'):
        cha.prepare_opd_bases(wrong_shape, None)


def engine_hex(name, prec):
    import prysm_b200 as pb
    case = O.HEX_CASES[name]
    x, y = (pb.asdevice(a) for a in O.grid(case[0], case[1], dtype_of(prec)))
    return O.run_hex(pb.segmented, pb.polynomials, name, x, y, to_numpy=tonp)


@pytest.mark.parametrize('precision', [32, 64], indirect=True)
@pytest.mark.parametrize('name', sorted(O.HEX_CASES))
def test_hex_aperture_matches_the_reference(golden, name, precision):
    got, cha = engine_hex(name, precision)
    for k, v in got.items():
        want = golden[f'hex{precision}_{name}_{k}']
        assert v.shape == want.shape, (k, v.shape, want.shape)
        if k in ('windows', 'segment_ids'):
            assert np.array_equal(v, want), k
        elif k in ('all_centers', 'vtov'):
            assert np.array_equal(v, want), k
        else:
            within(f'hex_{name}_{k}_fp{precision}', rel_linf(v, want), TOL[precision])
    # the reference's own test: the OPD is nonzero exactly where the amplitude is
    if 'zern_opd' in got:
        assert np.array_equal(got['zern_opd'] != 0, got['amp'] != 0)


def test_empty_windows_raise_like_the_reference():
    import prysm_b200 as pb
    _, cha = engine_hex('offgrid', 64)
    assert any(0 in m.shape for m in cha.local_masks)
    with pytest.raises(IndexError):
        cha.prepare_opd_bases(pb.polynomials.zernike_nm_seq, O.NMS)
    with pytest.raises(ValueError, match='cartesian axis'):
        pb.segmented.CompositeHexagonalAperture(cha.x, cha.y, 1, 0.3, 0.01, segment_angle=45)


@pytest.mark.parametrize('precision', [32, 64], indirect=True)
@pytest.mark.parametrize('name', sorted(O.LARGE_CASES))
def test_large_apertures_at_full_size(golden, name, precision):
    import prysm_b200 as pb
    n, diameter, *_ = O.LARGE_CASES[name]
    x, y = (pb.asdevice(a) for a in O.large_grid(n, diameter, dtype_of(precision)))
    got = O.run_large(pb.segmented, pb.polynomials, name, x, y, to_numpy=tonp)
    for k, v in got.items():
        want = golden[f'large{precision}_{k}']
        if k.endswith('_windows'):
            assert np.array_equal(v, want)
        elif k.endswith('_abssum'):          # the whole array: no cancellation in a sum of magnitudes
            within(f'large_{k}_fp{precision}', abs(float(v) - float(want)) / float(want), TOL[precision])
        elif k.endswith('_sum'):             # the signed OPD sum cancels: its relative error says nothing
            continue
        else:
            within(f'large_{k}_fp{precision}', rel_linf(v, want), TOL[precision])


def adjoint_setup(prec=64):
    import prysm_b200 as pb
    case = O.HEX_CASES['overlap']
    x, y = (pb.asdevice(a) for a in O.grid(case[0], case[1], dtype_of(prec)))
    cha = pb.segmented.CompositeHexagonalAperture(x, y, *case[2:5], segment_angle=case[5], exclude=case[6])
    cha.prepare_opd_bases(pb.polynomials.zernike_nm_seq, O.NMS)
    return cha


def test_adjoint_dot_product_identity_and_windowed_loop():
    import prysm_b200 as pb
    cha = adjoint_setup(64)
    nseg, k = len(cha.windows), len(O.NMS)
    rng = np.random.default_rng(5)
    c = rng.standard_normal((nseg, k))
    g = rng.standard_normal(tuple(cha.x.shape))
    lhs = float((tonp(cha.compose_opd(c)) * g).sum())
    adj = tonp(cha.compose_opd_adjoint(pb.asdevice(g)))
    rhs = float((c * adj).sum())
    assert abs(lhs - rhs) <= 1e-12 * max(abs(lhs), 1.0), (lhs, rhs)
    gd = pb.asdevice(g)
    for s, (win, m, b) in enumerate(zip(cha.windows, cha.local_masks, cha.opd_bases)):
        want = pb.polynomials.sum_of_2d_modes_adjoint(b, gd[win] * m)
        assert np.allclose(adj[s], want, rtol=1e-12, atol=1e-12 * np.abs(want).max())


def test_graph_replay_and_repeated_calls_are_bit_identical():
    import torch
    import prysm_b200 as pb
    pb.config.precision = 32
    try:
        cha = adjoint_setup(32)
        nseg, k = len(cha.windows), len(O.NMS)
        c = pb.asdevice(np.random.default_rng(6).standard_normal((nseg, k)))
        g = torch.randn(tuple(cha.x.shape), dtype=cha.x.dtype, device=cha.x.device,
                        generator=torch.Generator('cuda').manual_seed(2))
        e1 = cha.compose_opd(c).clone()
        assert torch.equal(e1, cha.compose_opd(c))
        a1 = cha.compose_opd_adjoint(g).clone()
        assert torch.equal(a1, cha.compose_opd_adjoint(g))
        fwd = pb.graphs.capture(lambda cc: cha.compose_opd(cc), c)
        back = pb.graphs.capture(lambda gg: cha.compose_opd_adjoint(gg), g)
        assert torch.equal(fwd(c), e1)
        assert torch.equal(back(g), a1)
        # a replay reads new coefficients / gradients from the captured buffers in place
        c2 = pb.asdevice(np.random.default_rng(7).standard_normal((nseg, k)))
        g2 = torch.randn_like(g)
        assert torch.equal(fwd(c2), cha.compose_opd(c2))
        assert torch.equal(back(g2), cha.compose_opd_adjoint(g2))
        assert not torch.equal(fwd(c2), e1)
        fwd.close()
        back.close()
    finally:
        pb.config.precision = 64


@pytest.fixture(scope='module')
def prysm_ref():
    if not reference.installed():
        pytest.skip('oracle/_ref is not installed (run oracle/install_reference.py)')
    with reference.loaded():
        import prysm
        import prysm.segmented  # noqa: F401
        import prysm.propagation  # noqa: F401
        yield prysm


def jwst_pupil(geometry, segmented, polynomials, x, y, c):
    """JWST: 18 hexagons with the three secondary struts cut out, and a per-segment OPD."""
    cha = segmented.CompositeHexagonalAperture(x, y, 2, 1.32, 0.007, exclude=(0,))
    struts = [geometry.spider(1, .1, x, y, rotation=r) for r in (-120, -60, 90)]    # True inside a vane
    cha.prepare_opd_bases(polynomials.zernike_nm_seq, O.LARGE_NMS)
    return cha.amp * ~(struts[0] | struts[1] | struts[2]), cha.compose_opd(c)


def at_focus(propagation, amp, opd, dx):
    return propagation.Wavefront.from_amp_and_phase(amp, opd, 0.6328, dx).focus(100.0, Q=2).data


def test_jwst_pupil_end_to_end_through_focus(prysm_ref):
    """A JWST pupil with spiders and a per-segment OPD -> from_amp_and_phase -> focus(Q=2): the engine at fp32 against
    the reference's pupil, OPD and fp64 field.  Like the fixtures, the reference builds the pupil with
    config.precision = 32 (float32 vertex rules) on the float32 grid promoted to float64, and propagates at 64."""
    from prysm import geometry as G, segmented as S, propagation as P, polynomials as PP
    from prysm.conf import config
    import prysm_b200 as pb
    x32, y32 = O.large_grid(512, 6.6, np.float32)
    dx = float(x32[0, 1] - x32[0, 0])
    c = O.hex_coefs('jwst_e2e', 18, len(O.LARGE_NMS)) * 10.0        # nm: up to ~1.6 rad of phase at 633 nm
    xr, yr = x32.astype(np.float64), y32.astype(np.float64)
    try:
        config.precision = 32
        amp_ref, opd_ref = jwst_pupil(G, S, PP, xr, yr, c)
        _, flat_opd = jwst_pupil(G, S, PP, xr, yr, np.zeros_like(c))
        config.precision = 64
        want = at_focus(P, amp_ref.astype(np.float64), opd_ref, dx)
        flat = at_focus(P, amp_ref.astype(np.float64), flat_opd, dx)
    finally:
        config.precision = 64
    assert (amp_ref > 0).mean() > 0.4                          # 18 segments: about 60 % of the 6.6 m grid
    assert (amp_ref == 0).sum() > 0 and np.abs(want).max() > 0
    assert rel_linf(want, flat) > 0.02, 'the OPD must change the field'     # 0.051 with these coefficients
    pb.config.precision = 32
    try:
        amp, opd = jwst_pupil(pb.geometry, pb.segmented, pb.polynomials, pb.asdevice(x32), pb.asdevice(y32), c)
        got = tonp(at_focus(pb.propagation, amp, opd, dx))
    finally:
        pb.config.precision = 64
    within('jwst512_amp_fp32', rel_linf(tonp(amp), amp_ref), 1e-6)
    within('jwst512_opd_fp32', rel_linf(tonp(opd), opd_ref), 1e-6)
    within('jwst512_focus_fp32', rel_linf(got, want), 1e-6)
