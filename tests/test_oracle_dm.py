"""CPU: the fp64 DM restatement (tests/dm_oracle.py) replays the reference's fixtures (tests/golden/dm.npz), the host-side
lattice and projection matrices of prysm_b200.dm match the reference's own functions, and scipy's warp rules that the
spline kernel reproduces are pinned."""
import numpy as np
import pytest
from scipy import ndimage

from conftest import load_golden, rel_linf
import dm_oracle as D
import reference


@pytest.fixture(scope='module')
def golden():
    return load_golden('dm.npz')


@pytest.fixture(scope='module')
def ref_dm():
    if not reference.installed():
        pytest.skip('reference prysm not installed')
    with reference.loaded():
        from prysm.conf import config
        import prysm.x.dm as rdm
        config.precision = 64
        yield rdm


@pytest.mark.parametrize('name', sorted(D.SMALL_CASES))
def test_oracle_replays_the_reference_fixtures(golden, name):
    shape, kw = D.SMALL_CASES[name]
    got = D.run_case(D.DM, name, shape, kw)
    for k, v in got.items():
        want = golden[f'{name}_{k}']
        assert v.shape == want.shape, (k, v.shape, want.shape)
        assert rel_linf(v, want) <= 4e-15, (name, k, rel_linf(v, want))


def test_oracle_replays_the_large_512_fixture(golden):
    shape, kw = D.LARGE_CASES['large512']
    got = D.run_case(D.DM, 'large512', shape, kw)
    for k, v in got.items():
        s = D.summarize(f'large512_{k}', v) if v.size > 4096 else {f'large512_{k}': v}
        scale = np.abs(v).max()
        for key, val in s.items():
            assert np.allclose(val, golden[key], rtol=1e-12, atol=1e-12 * scale * v.size), key


@pytest.mark.parametrize('name', sorted(D.SMALL_CASES))
def test_oracle_matches_the_reference(ref_dm, name):
    """To the last bits of fp64: the two differ only in how numpy orders the FFT and matrix sums of one call."""
    shape, kw = D.SMALL_CASES[name]
    ours = D.run_case(D.DM, name, shape, kw)
    theirs = D.run_case(ref_dm.DM, name, shape, kw)
    for k in ours:
        assert ours[k].shape == theirs[k].shape
        assert rel_linf(ours[k], theirs[k]) <= 4e-15, (name, k, rel_linf(ours[k], theirs[k]))


@pytest.mark.parametrize('shape,Nact,sep', [((64, 64), (7, 7), (6, 6)), ((64, 64), (8, 8), (6, 6)),
                                            ((48, 80), (10, 6), (6, 6)), ((63, 63), (8, 8), (6, 6)),
                                            ((72, 72), (8, 9), (7, 6)), ((2048, 2048), (64, 64), (24, 24)),
                                            ((101, 64), (9, 5), (4, 11))])
def test_engine_lattice_matches_the_reference(ref_dm, shape, Nact, sep):
    from prysm_b200.dm import actuator_lattice
    out = ref_dm.prepare_actuator_lattice(shape, Nact, sep, np.float64)
    iyy, ixx = out['iyy'], out['ixx']
    y0, sy, x0, sx = actuator_lattice(shape, Nact, sep)
    probe = np.arange(np.prod(shape)).reshape(shape)
    want = probe[iyy, ixx]
    got = probe[y0:y0 + sy * Nact[1]:sy, x0:x0 + sx * Nact[0]:sx]
    assert np.array_equal(got, want)


@pytest.mark.parametrize('shape', [(64, 64), (63, 63), (48, 80)])
@pytest.mark.parametrize('rot', [(12.5, 0, 0), (0, 0, 17.0), (0, 14.0, 0), (5.0, 7.0, 10.0)])
def test_engine_projection_matrices_match_the_reference(ref_dm, shape, rot):
    from prysm_b200.dm import projection_matrices, rotation_matrix
    from prysm.coordinates import make_rotation_matrix
    assert np.allclose(rotation_matrix(rot), make_rotation_matrix(rot), rtol=0, atol=1e-15)
    Mfwd, Mifwd = projection_matrices(shape, rot)
    (xf, yf), (xr, yr) = ref_dm.prepare_fwd_reverse_projection_coordinates(shape, rot)
    y, x = np.mgrid[0:shape[0], 0:shape[1]].astype(np.float64)
    for M, (wx, wy) in ((Mifwd, (xf, yf)), (Mfwd, (xr, yr))):
        w = M[2, 0] * x + M[2, 1] * y + M[2, 2]
        assert np.abs((M[0, 0] * x + M[0, 1] * y + M[0, 2]) / w - wx).max() < 1e-11
        assert np.abs((M[1, 0] * x + M[1, 1] * y + M[1, 2]) / w - wy).max() < 1e-11


def test_warp_rules_the_kernel_reproduces():
    """mode='constant': a coordinate on the last sample interpolates, one just outside [0, n-1] gives cval, and the
    prefilter of mode='constant' is the mirror one."""
    a = np.arange(1, 7, dtype=np.float64)
    assert abs(ndimage.map_coordinates(a, [[5.0]])[0] - 6.0) < 1e-14
    assert ndimage.map_coordinates(a, [[5.0 + 1e-9]])[0] == 0.0
    assert ndimage.map_coordinates(a, [[-1e-12]])[0] == 0.0
    rng = np.random.default_rng(2)
    img = rng.standard_normal((9, 13))
    assert np.array_equal(ndimage.spline_filter(img, 3, output=np.float64, mode='constant'),
                          ndimage.spline_filter(img, 3, output=np.float64, mode='mirror'))
    x = rng.uniform(-1, 13, (5, 5))
    y = rng.uniform(-1, 9, (5, 5))
    assert np.array_equal(D.warp(img, x, y), ndimage.map_coordinates(img, (y, x), order=3, mode='constant', cval=0.0))
