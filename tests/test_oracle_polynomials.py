"""CPU: the reference, where it is installed (oracle/_ref), re-derives every orthogonal-polynomial fixture
(tests/golden/polynomials*.npz) bit for bit, and the host-only index helpers (xy_j_to_mn, ansi_j_to_nm, nm_to_ansi_j,
nm_to_fringe, beside noll_to_nm and fringe_to_nm) equal the reference's over a range."""
import numpy as np
import pytest

from conftest import load_golden
import polynomials_oracle as O
import reference


@pytest.fixture(scope='module')
def golden():
    return load_golden('polynomials.npz')


@pytest.fixture(scope='module')
def ref():
    if not reference.installed():
        pytest.skip('reference prysm not installed')
    with reference.loaded():
        yield O.reference_modules()


@pytest.fixture(scope='module')
def P():
    from prysm_b200 import polynomials
    return polynomials


def test_reference_rederives_the_fixtures(golden, ref):
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        mine = O.run(ref)
    assert sorted(mine) == sorted(golden)
    for k, v in golden.items():
        np.testing.assert_array_equal(mine[k], v, err_msg=k)


def test_fixtures_cover_the_edges(golden):
    """Both grids hold the origin and the unit circle; the orders hold 0, 1, gaps and 30+; the Zernike set has m = 0,
    +-1, sine and cosine terms and |m| = 12 at n = 20; the sums hold zero, trailing-zero and duplicate coefficients."""
    for g in ('odd', 'even'):
        r = golden[f'{g}_r']
        assert (r == 0).sum() == 1 and (r == 1).any()
        assert np.abs(golden[f'{g}_zsum_zeros']).max() == 0
    assert {0, 1}.issubset(O.NS) and max(O.NS) >= 30 and any(b - a > 1 for a, b in zip(O.NS, O.NS[1:]))
    ms = [m for _, m in O.ZNMS]
    assert {0, 1, -1}.issubset(ms) and max(abs(m) for m in ms) == 12 and (20, 12) in O.ZNMS
    nms = O.ZSUMS['dups'][1]
    assert len(set(nms)) < len(nms)
    assert 0.0 in O.ZSUMS['trailing'][0][-2:] and len(O.CLEN_S['one']) == 1
    # a row of the Clenshaw table past the degree is zero
    assert np.abs(golden['clen_one_j3'][1:]).max() == 0


def test_index_helpers_match_the_reference(ref, P):
    from prysm_b200 import orthopoly
    p = ref.p
    for j in range(1, 200):
        assert orthopoly.xy_j_to_mn(j) == p.xy_j_to_mn(j), j
    for j in range(0, 200):
        assert P.ansi_j_to_nm(j) == p.ansi_j_to_nm(j), j
    for n in range(0, 20):
        for m in range(-n, n + 1, 2):
            assert P.nm_to_ansi_j(n, m) == p.nm_to_ansi_j(n, m), (n, m)
            assert P.nm_to_fringe(n, m) == p.nm_to_fringe(n, m), (n, m)
    for j in range(1, 120):
        assert P.noll_to_nm(j) == p.noll_to_nm(j)
        assert P.fringe_to_nm(j) == p.fringe_to_nm(j)


def test_index_helpers_literal(P):
    from prysm_b200 import orthopoly
    assert orthopoly.xy_j_to_mn(1) == (0, 0) and orthopoly.xy_j_to_mn(2) == (1, 0) and orthopoly.xy_j_to_mn(3) == (0, 1)
    with pytest.raises(ValueError):
        orthopoly.xy_j_to_mn(0)
    assert P.ansi_j_to_nm(4) == (2, 0) and P.nm_to_ansi_j(2, 0) == 4
    assert P.nm_to_fringe(0, 0) == 1 and P.nm_to_fringe(1, 1) == 2 and P.nm_to_fringe(2, 0) == 4


def test_every_reference_name_is_exported(ref, P):
    """prysm_b200.polynomials carries every evaluation name of the reference's prysm.polynomials this engine covers."""
    import inspect
    out_of_scope = {'hopkins', 'lstsq', 'normalize_modes', 'orthogonalize_modes', 'zernikes_to_magnitude_angle',
                    'zernikes_to_magnitude_angle_nmkey', 'zernike_zero_separation', 'nm_to_name', 'zernike_barplot',
                    'zernike_barplot_magnitudes', 'top_n'}
    names = [n for n in dir(ref.p) if not n.startswith('_') and callable(getattr(ref.p, n))
             and not inspect.ismodule(getattr(ref.p, n)) and n not in out_of_scope]
    for n in names:
        assert hasattr(P, n), n
        mine = inspect.signature(getattr(P, n)).parameters
        theirs = inspect.signature(getattr(ref.p, n)).parameters
        assert list(mine) == list(theirs), n
