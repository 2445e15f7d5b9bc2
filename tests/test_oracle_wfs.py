"""CPU: the reference, where it is installed (oracle/_ref), re-derives every wavefront-sensing fixture
(tests/golden/wfs*.npz) from the inputs tests/wfs_oracle.py builds; the engine's host mode finder matches the fixtures
and cutoff theory."""
import numpy as np
import pytest
from scipy import special

from conftest import load_golden
import wfs_oracle as O
import reference


@pytest.fixture(scope='module')
def golden():
    return load_golden('wfs.npz')


@pytest.fixture(scope='module')
def fibers():
    try:
        from prysm_b200 import fibers
    except ImportError as exc:
        pytest.skip(f'prysm_b200 does not import here: {exc}')
    return fibers


def test_fixture_inputs_are_deterministic():
    a, b = O.inputs(), O.inputs()
    assert sorted(a) == sorted(b)
    for k in a:
        assert np.array_equal(a[k], b[k]), k


def test_fixture_grid_spacings_are_float32_exact():
    for dx in (O.LP['dx'], O.SMF['dx'], O.TPF['dx'], O.TPF['fib_dx'], O.SRI['diameter'] / O.SRI['n'],
               O.PDI['diameter'] / O.PDI['n'], 2 * 12.5 * O.SRI['fiber_a'] / O.SRI['fiber_samples']):
        assert float(np.float32(dx)) == dx, dx


def test_reference_rederives_the_fixtures(golden):
    if not reference.installed():
        pytest.skip('reference prysm not installed')
    mine = O.reference_outputs()
    assert sorted(mine) == sorted(golden)
    for k, v in golden.items():
        np.testing.assert_array_equal(np.asarray(mine[k]), v, err_msg=k)


@pytest.mark.parametrize('V', O.V_FIND)
def test_find_all_modes_matches_the_fixtures(golden, fibers, V):
    from prysm_b200.conf import config
    config.precision = 64
    fam = fibers.find_all_modes(V)
    assert list(fam) == list(golden[f'fam_V{V}_keys'])
    for l, b in fam.items():
        ref = golden[f'fam_V{V}_{l}']
        assert b.shape == ref.shape
        assert np.abs(b - ref).max() <= 1e-12, (V, l)
    cnt = fibers.find_all_modes(V, count_only=True)
    assert [[l, c] for l, c in cnt.items()] == golden[f'cnt_V{V}'].tolist()


@pytest.mark.parametrize('V', (0.5, 2.3, 2.5, 3.0, 5.5, 10, 20, 33.3))
def test_find_all_modes_follows_cutoff_theory(fibers, V):
    """LP_{0,m} cuts off at 0 and the zeros of J1, LP_{l,m} (l >= 1) at the zeros of J_{l-1}: below V = 2.405 the fiber
    is single-mode, each family has as many modes as cutoffs below V, and the b values lie in (0, 1), in the reference's
    ascending order (the lowest-order radial mode last), with the +-l pairs equal."""
    from prysm_b200.conf import config
    config.precision = 64
    fam = fibers.find_all_modes(V)
    cnt = fibers.find_all_modes(V, count_only=True)
    if V < special.jn_zeros(0, 1)[0]:
        assert list(fam) == [0] and len(fam[0]) == 1
    for l, n in cnt.items():
        order = 1 if l == 0 else abs(l) - 1
        zeros = special.jn_zeros(order, int(V) + 4)
        expect = int((zeros < V).sum()) + (1 if l == 0 else 0)
        assert n == expect, (l, n, expect)
        b = fam[l]
        assert len(b) == n
        assert np.all((b > 0) & (b < 1)) and np.all(np.diff(b) > 0)
        if l > 0:
            assert np.array_equal(fam[-l], b)
    if V == 20:
        assert sum(cnt.values()) == 105


def test_find_all_modes_precision_32(fibers):
    from prysm_b200.conf import config
    config.precision = 32
    try:
        fam = fibers.find_all_modes(10)
    finally:
        config.precision = 64
    assert all(b.dtype == np.float32 for b in fam.values())
