"""CPU: the reference, where it is installed (oracle/_ref), re-derives every Shack-Hartmann fixture
(tests/golden/shack_hartmann*.npz) bit for bit; the fixtures pin the reference's multi-claimed edges; and the numpy
statement of spot_centroids (tests/shack_hartmann_oracle.py) agrees with an independent per-subaperture
scipy.ndimage.center_of_mass."""
import warnings

import numpy as np
import pytest
from scipy import ndimage

from conftest import load_golden
import shack_hartmann_oracle as O
import reference


@pytest.fixture(scope='module')
def golden():
    return load_golden('shack_hartmann.npz')


def test_reference_rederives_the_fixtures(golden):
    if not reference.installed():
        pytest.skip('reference prysm not installed')
    mine = O.reference_outputs()
    assert sorted(mine) == sorted(golden)
    for k, v in golden.items():
        np.testing.assert_array_equal(np.asarray(mine[k]), v, err_msg=k)


def test_fixtures_pin_the_shared_edges(golden):
    """At 256^2, dx = 0.01, pitch 0.32 and 8 x 8 lenslets, 956 samples take the phase of two to four lenslets."""
    claims = golden['claims_rect_edges']
    assert int((claims >= 2).sum()) == 956
    assert int(claims.max()) == 4
    # the polar path's tolerance is exercised: at angle 180 every edge sample sits a few ulp from its lenslet's edge;
    # at angle 30 no sample comes that close, so that case must match exactly
    assert int(golden['near_rect_angle180'].sum()) == 3792
    assert not golden['near_rect_angle30'].any()
    for name in O.CASES:
        assert golden[f'screen_{name}'].shape == O.CASES[name][0]
        assert golden[f'screen_{name}'].dtype == np.complex128


def _scipy_centroids(frame, x, y, pitch, n, shift, threshold):
    """Per subaperture with scipy.ndimage.center_of_mass on the uniform grid: index -> coordinate by x0 + k dx."""
    xc, yc = O.centres(pitch, n, shift)
    xv, yv = x[0], y[:, 0]
    dxx, dyy = xv[1] - xv[0], yv[1] - yv[0]
    disp = np.full((2, len(yc), len(xc)), np.nan)
    flux = np.zeros((len(yc), len(xc)))
    for j, yy in enumerate(yc):
        rows = np.flatnonzero((yv >= yy - pitch / 2) & (yv < yy + pitch / 2))
        for i, xx in enumerate(xc):
            cols = np.flatnonzero((xv >= xx - pitch / 2) & (xv < xx + pitch / 2))
            sub = frame[np.ix_(rows, cols)].astype(np.float64)
            if sub.size == 0:
                continue
            flux[j, i] = sub.sum()
            w = np.clip(sub - threshold * sub.max(), 0, None)
            if w.sum() == 0:
                continue
            cy, cx = ndimage.center_of_mass(w)
            disp[0, j, i] = xv[cols[0]] + cx * dxx - xx
            disp[1, j, i] = yv[rows[0]] + cy * dyy - yy
    return disp, flux


# pitches whose subaperture edges fall between samples: there the half-open intervals need no tie rule, which
# test_numpy_statement_breaks_ties_to_the_lower_lenslet covers
@pytest.mark.parametrize('threshold', (0.0, 0.3))
@pytest.mark.parametrize('shift,n,shape,pitch', [(False, 8, (256, 256), 0.325), (True, (5, 8), (250, 256), 0.3225),
                                                 (True, 7, (231, 231), 0.3275)])
def test_numpy_statement_matches_scipy_center_of_mass(threshold, shift, n, shape, pitch):
    rng = np.random.default_rng(7)
    x, y = O.grid(shape, 0.01)
    frame = rng.gamma(0.5, 10.0, shape)
    frame[rng.random(shape) < 0.3] = 0
    xc, yc = O.centres(pitch, n, shift)
    # one subaperture left dark: its displacement is NaN and its flux 0
    dark = (np.abs(x - xc[1]) <= pitch / 2 + 0.01) & (np.abs(y - yc[0]) <= pitch / 2 + 0.01)
    frame[dark] = 0
    disp, flux = O.centroids_numpy(frame, x, y, pitch, n, shift, threshold)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        ref_disp, ref_flux = _scipy_centroids(frame, x, y, pitch, n, shift, threshold)
    assert np.array_equal(np.isnan(disp), np.isnan(ref_disp))
    assert np.isnan(disp[:, 0, 1]).all() and flux[0, 1] == 0
    ok = ~np.isnan(ref_disp)
    assert ok.sum() > 20
    np.testing.assert_allclose(disp[ok], ref_disp[ok], rtol=0, atol=1e-12)
    np.testing.assert_allclose(flux, ref_flux, rtol=1e-13, atol=0)


def test_numpy_statement_owns_each_sample_once():
    """Half-open intervals: summed over subapertures, the flux of a frame of ones counts every sample inside the
    array's footprint exactly once (shifted 8 x 0.325 covers [-1.3, 1.3), all 256 samples)."""
    x, y = O.grid((256, 256), 0.01)
    _, flux = O.centroids_numpy(np.ones((256, 256)), x, y, 0.325, 8, shift=True)
    assert flux.sum() == 256 * 256
    assert flux.min() >= 30 * 30 and flux.max() <= 33 * 33


def test_numpy_statement_breaks_ties_to_the_lower_lenslet():
    """Where rounding lets two half-open intervals overlap, the lower index owns the sample; past the last upper
    edge and before the first lower edge nothing does."""
    c = np.array([0.0, 1.0])
    coords = np.array([-0.6, -0.5, 0.49, np.nextafter(0.5, 0), 0.5, 1.49, 1.5])
    assert O.owners(coords, c, 1.0).tolist() == [-1, 0, 0, 0, 1, 1, -1]
    assert O.owners(np.array([0.5]), c, np.nextafter(1.0, 2)).tolist() == [0]
