"""CPU: the references of tests/analysis_reference.py against scipy's RegularGridInterpolator, numpy's nan statistics and
the estimate_size loop restated from its definition; every GPU case free of ambiguous points and flagged crossing
rows; the committed Bessel fixture against scipy; and every defect model against the GPU test's ceilings: each faithful
model stays under its ceiling and each defect lands 10x or more above (the margin is printed)."""
import warnings

import numpy as np
import pytest
import scipy.special as sps
from scipy.interpolate import RegularGridInterpolator

import analysis_reference as A
from conftest import load_golden
from test_gpu_analysis_vs_fp64 import CEIL

LD = A.LDBL


def margin(name, fig, ceiling):
    print(f'{name}: {fig:.3e} is {fig / ceiling:.3g}x the ceiling {ceiling:.3g}')
    assert fig > 10 * ceiling, name


# ---- launch rules --------------------------------------------------------------------------------------------------
def test_launch_rules():
    assert A.grid_for(1, 132) == 1 and A.grid_for(10 ** 9, 132) == 132 * 16
    assert A.sweep(132) == 540672 and A.sweep_counts(132)[-1] == 3 * 540672
    assert [A.chunk_len(n) for n in A.CROSS_NX] == [1, 1, 1, 2, 2, 16, 79]
    assert (A.crossing_launches(False), A.crossing_launches(True)) == (3, 4)
    assert A.AZ_MAX_NY * 8 == 224 * 1024


# ---- the interpolator against scipy ----------------------------------------------------------------------------------
def scipy_interp(d, x, y, px, py, fill):
    return RegularGridInterpolator((y, x), d, method='linear', bounds_error=False, fill_value=fill)((py, px))


@pytest.mark.parametrize('shape', ((29, 43), (1, 43), (29, 1)))
def test_interp_matches_scipy(shape):
    """nodes, both ends, one ulp outside, interior points, non-uniform axes, single-sample axes (scipy needs two
    samples, so those compare against the axis duplicated), NaN corners of weight 0"""
    ny, nx = shape
    rng = np.random.default_rng(3)
    d = rng.uniform(0.5, 2.0, shape)
    x = np.cumsum(rng.uniform(0.3, 1.7, nx)) - 9.0 if nx > 1 else np.array([0.25])
    y = np.cumsum(rng.uniform(0.3, 1.7, ny)) - 7.0 if ny > 1 else np.array([-0.5])
    px = np.concatenate((np.repeat(x, 3), [x[0], x[-1], np.nextafter(x[0], -9), np.nextafter(x[-1], 9)],
                         rng.uniform(x[0], x[-1], 500)))
    py = np.concatenate((np.resize(y, 3 * nx), [y[0], y[-1], y[0], y[-1]], rng.uniform(y[0], y[-1], 500)))
    got, maj = A.interp_ref(d, x, y, px, py, 0.75)
    dd, xx, yy = d, x, y
    if nx == 1:
        dd, xx = np.concatenate((dd, dd), axis=1), np.array([x[0], x[0] + 1.0])
    if ny == 1:
        dd, yy = np.concatenate((dd, dd), axis=0), np.array([y[0], y[0] + 1.0])
    want = scipy_interp(dd, xx, yy, px, py, 0.75)
    want = np.where((px > x[-1]) | (py > y[-1]), 0.75, want)
    assert np.all(np.abs(got.astype(np.float64) - want) <= 2 * np.spacing(np.abs(want)))
    if ny > 1 and nx > 1:
        dn = d.copy()
        dn[7, 12] = np.nan
        g, _ = A.interp_ref(dn, x, y, [x[11], x[12]], [y[7], y[6]])
        assert np.all(np.isnan(g))                      # weight-0 corners carry the NaN, as scipy's sum does
        assert np.all(np.isnan(scipy_interp(dn, x, y, np.array([x[11], x[12]]), np.array([y[7], y[6]]), 0.0)))


def test_interp_defects():
    """'lt' and 'skip_zero' both lose the NaN of a weight-0 corner at a node"""
    rng = np.random.default_rng(4)
    x, y = np.linspace(0, 5, 6), np.linspace(0, 3, 4)
    d = rng.uniform(size=(4, 6))
    d[1, 3] = np.nan
    px, py = np.array([x[2]]), np.array([y[1]])
    assert np.isnan(A.interp_model(d, x, y, px, py))
    for defect in ('lt', 'skip_zero'):
        assert np.isfinite(A.interp_model(d, x, y, px, py, defect=defect)), defect


# ---- statistics and crossings against numpy / the estimate_size loop -------------------------------------------------
def test_azstats_match_numpy():
    rng = np.random.default_rng(5)
    for n in (1, 2, 7, 256, 257):
        v = rng.standard_normal(n)
        r = A.azstats_ref(v)
        assert r['count'] == n
        for k, f in (('mean', np.mean), ('var', np.var), ('median', np.median), ('min', np.min), ('max', np.max)):
            assert abs(float(r[k]) - f(v)) <= 4 * np.spacing(np.abs(v).max()), (n, k)
    v = np.array([np.nan, 3.0, 1.0, np.nan, 2.0, 2.0])
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        assert float(A.azstats_ref(v)['median']) == np.nanmedian(v) == 2.0
        assert np.isnan(A.azstats_ref(np.full(4, np.nan))['median'])


def estimate_size_loop(polar, r, hm, criteria):
    """the reference's estimate_size loop, restated from its definition (without the final raise)"""
    crossings = []
    for row, mask in zip(polar, polar > hm):
        idx = np.flatnonzero(mask[:-1] != mask[1:])
        if idx.size == 0:
            continue
        i = int(idx[0] if criteria == 'first' else idx[-1])
        y0, y1 = row[i], row[i + 1]
        frac = 0 if y1 == y0 else (hm - y0) / (y1 - y0)
        crossings.append(r[i] + frac * (r[i + 1] - r[i]))
    return len(crossings), (np.mean(np.asarray(crossings)) if crossings else np.nan)


@pytest.mark.parametrize('nx', A.RADIAL_NX[:3])
def test_crossings_match_the_loop(nx):
    d, x, y, rmax = A.radial_case(nx)
    vals, maj, _ = A.lattice_ref(d, x, y, rmax)
    rho, _ = A.lattice_axes(nx, d.shape[0], rmax)
    v64 = vals.astype(np.float64)
    for met, rel in A.METRICS.values():
        t = np.float64(met) * v64.max() if rel else met
        for last in (0, 1):
            c, m, _, _ = A.crossings_ref(vals, maj, rho, t, last)
            c2, m2 = estimate_size_loop(v64, rho, t, 'last' if last else 'first')
            assert c == c2 and abs(float(m) - m2) <= 1e-12 * rmax


def test_nan_crossing_keeps_the_row():
    """the 64^2 Gaussian with a NaN patch: the loop gives NaN for both criteria, and so does the reference here"""
    x = np.arange(64) - 32.0
    d = np.exp(-(x[None, :] ** 2 + x[:, None] ** 2) / (2 * 8.0 ** 2))
    d[30:35, 44:47] = np.nan
    rmax = A.rmax_of(x, x)
    vals, maj, _ = A.lattice_ref(d, x, x, rmax)
    rho, _ = A.lattice_axes(64, 64, rmax)
    for last in (0, 1):
        c, m, _, _ = A.crossings_ref(vals, maj, rho, 0.3, last)
        assert c == 64 and np.isnan(m)
        assert np.isnan(estimate_size_loop(vals.astype(np.float64), rho, 0.3, 'last' if last else 'first')[1])
        c3, m3 = A.crossings_model(vals, rho, 0.3, last, 'nan_drop')
        assert c3 == 58 and abs(m3 - 12.4204) < 1e-4


# ---- every GPU case is unambiguous -----------------------------------------------------------------------------------
def test_gpu_cases_are_unambiguous():
    for ny in A.POLAR_N:
        for nx in A.POLAR_N:
            d, x, y, rmax, rows, cols = A.polar_case(ny, nx)
            assert not A.lattice_ref(d, x, y, rmax, rows=rows)[2].any(), (ny, nx)
            assert not A.lattice_ref(d, x, y, rmax, cols=cols)[2].any(), (ny, nx)
    for ny in A.AZ_NY:
        for kind in ('smooth', 'offset', 'nan', 'signs'):
            if ny >= 4097 and kind == 'signs':
                continue
            d, x, y, rmax, cols = A.az_case(ny, kind)
            assert not A.lattice_ref(d, x, y, rmax, cols=cols)[2].any(), (ny, kind)
    for nx in A.CROSS_NX:
        for variant in A.RAY_VARIANTS:
            d, x, y, rmax, t = A.ray_case(nx, variant)
            vals, maj, amb = A.lattice_ref(d, x, y, rmax)
            assert not amb.any()
            rho, _ = A.lattice_axes(nx, 2, rmax)
            ex = A.lattice_points(nx, 2, rmax)[2]
            for metric, relative in ((t, False), (0.5, True))[:1 if variant == 'never' else 2]:
                level, extra = A.crossing_level(vals, maj, metric, relative)
                for last in (0, 1):
                    assert not A.crossings_ref(vals, maj, rho, level, last, extra, exact=ex)[3].any(), (nx, variant)
    for nx in A.RADIAL_NX:
        for nan in (False, True):
            d, x, y, rmax = A.radial_case(nx, nan=nan)
            vals, maj, amb = A.lattice_ref(d, x, y, rmax)
            assert not amb.any()
            rho, _ = A.lattice_axes(nx, d.shape[0], rmax)
            for met, rel in A.METRICS.values():
                t, extra = A.crossing_level(vals, maj, met, rel)
                for last in (0, 1):
                    assert not A.crossings_ref(vals, maj, rho, t, last, extra)[3].any(), (nx, met, last)


# ---- defect models against the ceilings ------------------------------------------------------------------------------
def az_fig(col, maj, defect, stat):
    r, sc = A.azstats_ref(col), A.azstats_scales(col, maj)
    got = A.azstats_model(col.astype(np.float64), defect)
    if np.isnan(got[stat]) != np.isnan(float(r[stat])):
        return np.inf
    return float(abs(LD(got[stat]) - r[stat]) / (LD(A.EPS) * sc[stat]))


@pytest.mark.parametrize('defect,kind,stat,ceil', [('one_pass', 'offset', 'var', 'var'),
                                                   ('upper_median', 'smooth', 'median', 'order'),
                                                   ('nan_rank', 'nan', 'median', 'order'),
                                                   ('f32_sums', 'smooth', 'mean', 'mean')])
def test_az_defects(defect, kind, stat, ceil):
    d, x, y, rmax, cols = A.az_case(512, kind)
    vals, maj, _ = A.lattice_ref(d, x, y, rmax, cols=cols)
    faithful = max(az_fig(vals[:, i], maj[:, i], None, stat) for i in range(len(cols))
                   if A.azstats_ref(vals[:, i])['count'] > 0)
    assert faithful < CEIL[ceil]
    worst = max(az_fig(vals[:, i], maj[:, i], defect, stat) for i in range(len(cols))
                if A.azstats_ref(vals[:, i])['count'] > 0)
    margin(defect, worst, CEIL[ceil])


@pytest.mark.parametrize('defect,variant', [('drop_shared', 'before'), ('swap', 'ring'), ('nan_drop', 'nan')])
def test_crossing_defects(defect, variant):
    nx = 4097
    d, x, y, rmax, t = A.ray_case(nx, variant)
    vals, maj, _ = A.lattice_ref(d, x, y, rmax)
    rho, _ = A.lattice_axes(nx, 2, rmax)
    worst = 0.0
    for last in (0, 1):
        c, m, _, _ = A.crossings_ref(vals, maj, rho, t, last)
        assert A.crossing_fig(*A.crossings_model(vals, rho, t, last), c, m, rmax) < CEIL['cross']
        worst = max(worst, A.crossing_fig(*A.crossings_model(vals, rho, t, last, defect), c, m, rmax))
    margin(defect, worst, CEIL['cross'])


def test_bessel_fixture_vs_scipy():
    z = load_golden(A.BESSEL_FIXTURE)
    assert np.max(np.abs(z['j0'] - sps.j0(z['u']))) < 1e-15
    assert np.max(np.abs(z['j1'] - sps.j1(z['u']))) < 1e-15
    assert z['u'].min() <= 1e-12 and z['u'].max() >= 1e4
    s = z['s']
    assert 1.0 in s and np.nextafter(1.0, 2.0) in s and all((1 - 2.0 ** -k) in s for k in range(1, 53))


@pytest.mark.parametrize('defect,band', [('threshold', (1e-8, 1e-3)), ('asymptotic', (14, 1e5))])
def test_jinc_defects(defect, band):
    z = load_golden(A.BESSEL_FIXTURE)
    sc = A.analytic_scales(z)
    sel = (z['u'] > band[0]) & (z['u'] < band[1])
    ref = z['airy_e'][sel].astype(LD)
    assert A.analytic_fig(A.jinc_model(z['u'][sel]), ref, sc['efield'][sel]) < CEIL['efield']
    margin(defect, A.analytic_fig(A.jinc_model(z['u'][sel], defect), ref, sc['efield'][sel]), CEIL['efield'])
    if defect == 'asymptotic':
        r2 = z['ee'][sel].astype(LD)
        assert A.analytic_fig(A.ee_model(z['u'][sel]), r2, sc['ee'][sel]) < CEIL['ee']
        margin('ee ' + defect, A.analytic_fig(A.ee_model(z['u'][sel], defect), r2, sc['ee'][sel]), CEIL['ee'])


def test_core_model():
    z = load_golden(A.BESSEL_FIXTURE)
    sc = A.analytic_scales(z)
    assert A.analytic_fig(A.core_model(z['s']), z['core'].astype(LD), sc['core']) < CEIL['core']
