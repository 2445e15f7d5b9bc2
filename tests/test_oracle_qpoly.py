"""CPU: the reference, where it is installed (oracle/_ref), re-derives every Forbes-polynomial fixture
(tests/golden/qpoly*.npz) bit for bit; the engine's C++ recurrence tables (pb_qpoly_tables, the ones its kernels are
planned with) match the reference's scalar functions; and the host-only Q2d_nm_c_to_a_b keeps the reference's
semantics."""
import numpy as np
import pytest

from conftest import load_golden
import qpoly_oracle as O
import reference


@pytest.fixture(scope='module')
def golden():
    return load_golden('qpoly.npz')


@pytest.fixture(scope='module')
def ref():
    if not reference.installed():
        pytest.skip('reference prysm not installed')
    with reference.loaded():
        yield O.reference_modules()


@pytest.fixture(scope='module')
def Q():
    from prysm_b200 import qpoly
    return qpoly


def test_reference_rederives_the_fixtures(golden, ref):
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        mine = O.run(ref)
    assert sorted(mine) == sorted(golden)
    for k, v in golden.items():
        np.testing.assert_array_equal(mine[k], v, err_msg=k)


def test_fixtures_cover_the_edges(golden):
    """Both grids hold the origin and the unit circle; the 2D-Q set has repeats, m = 1 beyond n = 3 and |m| = 20."""
    for g in ('odd', 'even'):
        r = golden[f'{g}_r']
        assert (r == 0).sum() == 1 and (r == 1).any()
    assert O.NMS.count((2, 2)) == 2 and (5, 1) in O.NMS and max(abs(m) for _, m in O.NMS) == 20
    assert np.abs(golden['odd_z2d_zeros']).max() == 0
    # abc_q2d divides by zero at (n, m) = (1, 1), (0, 2), (0, 3) and nowhere else in the table
    bad = np.argwhere(np.isnan(golden['tab_q2d'][..., 0]))
    assert sorted((int(n), int(m) + 1) for m, n in bad) == [(0, 2), (0, 3), (1, 1)]


def _rel(a, b):
    a, b = np.asarray(a), np.asarray(b)
    ok = np.isfinite(b)
    assert np.array_equal(ok, np.isfinite(a))
    return float(np.max(np.abs(a[ok] - b[ok]) / np.maximum(np.abs(b[ok]), 1e-300)))


def test_cpp_tables_match_the_reference(golden, Q):
    from prysm_b200 import _ops, _capi
    assert _rel(_ops.qpoly_tables(_capi.QPOLY_BFS, 0, O.NMAX)[:, :3], golden['tab_qbfs']) < 1e-13
    assert _rel(_ops.qpoly_tables(_capi.QPOLY_CON, 0, O.NMAX)[:, :3], golden['tab_qcon']) < 1e-14
    mine = np.stack([_ops.qpoly_tables(_capi.QPOLY_2D, m, O.NMAX) for m in range(1, O.TAB_M + 1)])
    assert _rel(mine, golden['tab_q2d']) < 1e-12
    # the Python scalar functions read the same tables
    assert Q.f_qbfs(7) == golden['tab_qbfs'][7, 0] or abs(Q.f_qbfs(7) / golden['tab_qbfs'][7, 0] - 1) < 1e-13
    assert abs(Q.g_q2d(5, 4) / golden['tab_q2d'][3, 5, 5] - 1) < 1e-12
    with pytest.raises(ZeroDivisionError):
        Q.abc_q2d(1, 1)
    with pytest.raises(ValueError):
        Q.f_q2d(65, 2)


NM_C_CASES = [
    ([(0, 0), (2, 1), (1, -2), (3, -2), (3, -2)], [1.0, 2.0, 3.0, 0.0, 0.0]),
    ([(4, 0), (1, 0), (0, 3), (2, -1), (2, -1)], [0.5, 0.0, 0.25, 1.0, 2.0]),    # a later repeat wins
    ([(0, 0), (1, 1)], [0.0, 0.0]),                                             # nothing left
    ([(2, -3), (0, 5)], [1.0, 0.0]),                                            # empty cosine orders
]


def test_q2d_nm_c_to_a_b_literal(Q):
    assert Q.Q2d_nm_c_to_a_b(*NM_C_CASES[0]) == ([1.0], [[0, 0, 2.0], []], [[], [0, 3.0]])
    assert Q.Q2d_nm_c_to_a_b(*NM_C_CASES[2]) == ([], [], [])


@pytest.mark.parametrize('case', range(len(NM_C_CASES)))
def test_q2d_nm_c_to_a_b_matches_the_reference(ref, Q, case):
    assert Q.Q2d_nm_c_to_a_b(*NM_C_CASES[case]) == ref.q.Q2d_nm_c_to_a_b(*NM_C_CASES[case])
