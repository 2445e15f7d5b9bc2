"""CPU: the fp64 restatement of the geometry and of compose_opd (tests/segmented_oracle.py) replays the reference's
fixtures (tests/golden/segmented*.npz), and the engine's host tables of CompositeHexagonalAperture (windows, centres,
ids, the keys that decide which segments share a basis) match the fixtures and, where it is installed, the reference."""
import numpy as np
import pytest

from conftest import load_golden, rel_linf
import segmented_oracle as O
import reference


@pytest.fixture(scope='module')
def golden():
    return load_golden('segmented.npz')


@pytest.fixture(scope='module')
def ref():
    if not reference.installed():
        pytest.skip('reference prysm not installed')
    with reference.loaded():
        from prysm.conf import config
        from prysm import segmented
        yield config, segmented


def dtype_of(prec):
    return np.float32 if prec == 32 else np.float64


@pytest.mark.parametrize('prec', [32, 64])
def test_restatement_replays_the_geometry_fixtures(golden, prec):
    x, y = (a.astype(np.float64) for a in O.grid(O.SHAPE, O.DX, dtype_of(prec)))
    r = np.hypot(x, y)
    mine = {
        'poly_ccw': O.polygon_sdf(O.CONVEX, x, y),
        'poly_cw': O.polygon_sdf(O.CONVEX[::-1], x, y),
        'poly_concave': O.polygon_sdf(O.CONCAVE, x, y),
        'regpoly': O.polygon_sdf(O.regular_vertices(7, 0.93, (0.13, -0.21), 17, dtype_of(prec)), x, y),
        'spider_deg': O.spider_sdf(4, 0.083, x, y, rotation=30, center=(0.1, 0.05)),
        'spider_rad': O.spider_sdf(3, 0.097, x, y, rotation=0.4, rotation_is_rad=True),
        'rect': O.rectangle_sdf(0.83, x, y, height=0.47),
        'rect90': O.rectangle_sdf(0.83, x, y, height=0.47, angle=90),
        'rect_rot': O.rectangle_sdf(0.83, x, y, height=0.47, angle=23),
        'fillet': O.fillet_sdf(0.9, 0.6, 0.21, x, y, center=(0.1, -0.05)),
        'fillet_rot': O.fillet_sdf(0.9, 0.6, 0.21, x, y, center=(0.1, -0.05), rotation=12),
        'annulus': O.annulus_sdf(0.4, 1.1, r),
        'offset_circle': O.offset_circle(0.7, x, y, center=(0.2, -0.1)),
    }
    for k, v in mine.items():
        want = golden[f'geom{prec}_{k}']
        if want.dtype == bool:
            assert np.array_equal(v, want), k
        else:
            assert rel_linf(v, want) <= 1e-15, (k, rel_linf(v, want))
    assert golden[f'geom{prec}_poly_empty'].shape == (0, O.SHAPE[1])


def _windows(ws):
    return np.array([[w[0].start, w[0].stop, w[1].start, w[1].stop] for w in ws]).reshape(-1, 4)


@pytest.mark.parametrize('prec', [32, 64])
@pytest.mark.parametrize('name', sorted(O.HEX_CASES))
def test_engine_host_tables_match_the_fixtures(golden, name, prec):
    from prysm_b200.segmented import hex_layout, grid_keys
    shape, dx, rings, diam, sep, angle, exclude, with_bases = O.HEX_CASES[name]
    x, _ = O.grid(shape, dx, dtype_of(prec))
    vtov, _, all_centers, ids, centers, windows = hex_layout(shape, x[0, 1] - x[0, 0], rings, diam, sep, angle, exclude)
    g = lambda k: golden[f'hex{prec}_{name}_{k}']  # noqa: E731
    assert np.array_equal(_windows(windows), g('windows'))
    assert np.array_equal(np.array(all_centers).reshape(-1, 2), g('all_centers'))
    assert np.array_equal(np.array(ids), g('segment_ids'))
    assert vtov == float(g('vtov'))
    if not with_bases:
        with pytest.raises(IndexError):
            grid_keys([x[w[0].start, w[1].start] if w[0].stop > w[0].start and w[1].stop > w[1].start else 0.0
                       for w in windows], centers, windows)
        return
    keys = grid_keys([x[w[0].start, w[1].start] for w in windows], centers, windows)
    hw = [(k[1], k[2]) for k in keys]
    offs = np.concatenate([[0], np.cumsum([h * w for h, w in hw])])[:-1]
    if prec == 64:        # the fixture's local x is the reference's own local grid: its first sample is the key
        lx = g('local_x')
        assert [float(lx[o]) for o in offs] == [k[0] for k in keys]


@pytest.mark.parametrize('name', sorted(n for n, c in O.HEX_CASES.items() if c[-1]))
def test_restatement_of_compose_replays_the_fixtures(golden, name):
    shape, *_ = O.HEX_CASES[name]
    g = lambda k: golden[f'hex64_{name}_{k}']  # noqa: E731
    wins = [(slice(a, b), slice(c, d)) for a, b, c, d in g('windows')]
    hw = [(b - a, d - c) for a, b, c, d in g('windows')]
    offs = np.concatenate([[0], np.cumsum([h * w for h, w in hw])])
    masks = [g('masks')[offs[i]:offs[i + 1]].reshape(hw[i]) for i in range(len(hw))]
    for tag, orders in (('zern', O.NMS), ('xy', O.MONOMIALS)):
        k = len(orders)
        bases = [g(f'{tag}_bases')[k * offs[i]:k * offs[i + 1]].reshape((k,) + hw[i]) for i in range(len(hw))]
        c = O.hex_coefs(name, len(hw), k)
        for key, cc, out0 in ((f'{tag}_opd', c, np.zeros(shape)), (f'{tag}_opd_out', c, O.hex_out0(name, shape)),
                              (f'{tag}_opd_short', c[:len(hw) - 2], np.zeros(shape))):
            assert rel_linf(O.compose(wins, masks, bases, cc, out0), g(key)) <= 1e-14, key


@pytest.mark.parametrize('prec', [32, 64])
@pytest.mark.parametrize('name', sorted(O.LARGE_CASES))
def test_engine_host_tables_match_the_reference_at_full_size(ref, name, prec):
    from prysm_b200.segmented import hex_layout, grid_keys
    config, segmented = ref
    n, diameter, rings, diam, sep, exclude = O.LARGE_CASES[name]
    x, y = O.large_grid(n, diameter, dtype_of(prec))
    config.precision = prec
    cha = segmented.CompositeHexagonalAperture(x, y, rings, diam, sep, exclude=exclude)
    config.precision = 64
    vtov, _, all_centers, ids, centers, windows = hex_layout(x.shape, x[0, 1] - x[0, 0], rings, diam, sep, 90, exclude)
    assert windows == cha.windows
    assert np.array_equal(np.array(all_centers), np.array(cha.all_centers))
    assert [int(i) for i in cha.segment_ids] == ids
    keys = grid_keys([x[w[0].start, w[1].start] for w in windows], centers, windows)
    want = [(float(lx[0, 0]), *lx.shape) for lx, _ in cha.local_coords]
    assert keys == want
    if name == 'luvoira2048':
        assert len(windows) == 120 and len(set(keys)) == 13
