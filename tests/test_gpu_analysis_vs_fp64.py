"""GPU: the PSF / MTF analysis kernels of csrc/analysis.cu held to the long-double references of
tests/analysis_reference.py past every grid-stride sweep, chunk edge and the shared-memory row limit.

- pb_interp2d_linear, points: f32 / f64 / c64 / c128 data, a window of a larger array (ld > nx), single-row and
  single-column axes, non-uniform axes, nodes, both ends, one ulp outside each end, a NaN corner of weight 0; 1, the
  grid cap +-1 and 3x the cap points.  Polar: ny, nx in {1, 2, 255, 256, 257, 4097}.
- pb_azimuthal_stats: ny from 1 to the 28672-row limit, each mask bit alone and all together in one launch, smooth,
  offset (1e6 + 1e-3 noise), NaN, signed and subnormal data; 28673 rows, unknown bits and an empty mask refused or
  skipped with no launch.
- pb_polar_crossings: crossings on either side of a chunk edge, first and last in different chunks, exact ties, rows
  that never cross, NaN crossings, the four metrics with first and last; estimate_size's NaN result.
- pb_analytic_radial: every kind against the 60-digit fixture, f32 / f64 inputs and outputs, counts past the grid cap.

fp64 figures are |got - ref| over the reference's error scale (eps times its majorant); float32 outputs are in ulps of
the float32-rounded reference.  Bounds are 1.5x the figures measured on an H100 (`MEASURED`, recorded with
PB_TEST_MEASUREMENTS) and never above the ceilings tests/test_host_analysis_reference.py shows every modelled defect
exceeds by 10x or more.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import analysis_reference as A
from accuracy import Ledger
from conftest import load_golden
from gpu_fixtures import pb, dev, host, launches, sm_count  # noqa: F401

pytestmark = pytest.mark.gpu

LD = A.LDBL
NPR = {32: np.float32, 64: np.float64}

# ceilings, shown by the host test to sit 10x or more below every modelled defect.  fp64 figures are in units of eps
# times the reference's majorant, float32 ones in ulps of the rounded reference.
CEIL = {'interp64': 16.0, 'ulps32': 1.0, 'mean': 16.0, 'var': 64.0, 'order': 16.0, 'cross': 1e-12,
        'efield': 1e5, 'airy': 2e5, 'ee': 1e5, 'core': 64.0}

# ---- measured figures (NVIDIA H100 80GB HBM3, 700 W power limit, 1980 MHz SM clock); bounds are 1.5x these, capped
# at the ceiling --------------------------------------------------------------------------------------------------
# CUDA's fp64 j0 / j1 past u = 14 measure 9640 eps of |f| + |u f'| (2 jinc) and 13400 ((2 jinc)^2), at the zeros of
# J1; a jinc threshold moved to 1e-4 gives 5.6e6 and a J1 of the asymptotic form alone 1.4e13.
MEASURED = {
    '32/az_max': 0.496,
    '32/az_mean': 0.484,
    '32/az_median': 0.457,
    '32/az_min': 0.489,
    '32/az_var': 0.498,
    '32/cross_radial': 5.59e-17,
    '32/cross_ray': 6e-17,
    '32/interp_points': 0.5,
    '32/interp_polar': 0.5,
    '64/airy_ft_small': 0.565,
    '64/airy_large': 13400.0,
    '64/airy_small': 1.75,
    '64/az_max': 0.119,
    '64/az_mean': 0.00834,
    '64/az_median': 0.0834,
    '64/az_min': 0.124,
    '64/az_var': 41.5,
    '64/cross_nan': 4.99e-17,
    '64/cross_radial': 7.95e-17,
    '64/cross_ray': 6e-17,
    '64/difflim_small': 0.565,
    '64/ee_large': 138.0,
    '64/ee_small': 1.86,
    '64/efield_large': 9640.0,
    '64/efield_small': 1.27,
    '64/interp_points': 0.0326,
    '64/interp_polar': 0.208,
    '64/interp_sweep': 0.0731,
    '64/normalized_small': 0.565,
}



def ceiling(name):
    """the CEIL entry of a figure: crossings in rmax at both precisions, other float32 figures in ulps, fp64 ones by
    the quantity"""
    prec, fig = name.split('/')
    if fig.startswith('cross_'):
        return CEIL['cross']
    if prec == '32':
        return CEIL['ulps32']
    if fig.startswith('interp_'):
        return CEIL['interp64']
    if fig.startswith('az_'):
        return CEIL.get(fig[3:], CEIL['order'])
    return CEIL[KINDS[fig.rsplit('_', 1)[0]][2]]


# the worst figure of each name over the whole file: a name collects every test that reaches it
LEDGER = Ledger(MEASURED, ceiling)
check = LEDGER.check


def fig64(got, ref, maj):
    """max |got - ref| / (eps maj); NaN must match NaN; where maj is 0 the values must be equal"""
    got = np.asarray(got, np.float64)
    nan = np.isnan(ref.astype(np.float64))
    assert np.array_equal(np.isnan(got), nan)
    d = np.abs(got[~nan].astype(LD) - ref[~nan])
    s = A.EPS * maj[~nan]
    assert np.all(d[s == 0] == 0)
    return float(np.max(d[s > 0] / s[s > 0])) if np.any(s > 0) else 0.0


def ulps32(got, ref):
    got = np.asarray(got, np.float32)
    nan = np.isnan(ref.astype(np.float64))
    assert np.array_equal(np.isnan(got), nan)
    r32 = ref[~nan].astype(np.float32)
    sp = np.spacing(np.abs(r32)).astype(LD)
    return float(np.max(np.abs(got[~nan].astype(LD) - ref[~nan]) / sp)) if r32.size else 0.0


def figure(name, prec, got, ref, maj):
    check(f'{prec}/{name}', fig64(got, ref, maj) if prec == 64 else ulps32(got, ref))


# ---- pb_interp2d_linear, points --------------------------------------------------------------------------------------
def point_set(x, y, nan_at):
    """nodes, both ends, one ulp outside each end, interior points and the node before a NaN sample (weight-0 NaN)"""
    rng = np.random.default_rng(1)
    px = [x, [x[0], x[-1], np.nextafter(x[0], -np.inf), np.nextafter(x[-1], np.inf)], rng.uniform(x[0], x[-1], 300)]
    py = [np.resize(y, x.size), [y[0], y[-1], y[0], y[-1]], rng.uniform(y[0], y[-1], 300)]
    px.append([x[0], x[-1]])
    py.append([np.nextafter(y[0], -np.inf), np.nextafter(y[-1], np.inf)])
    if nan_at is not None:
        r, c = nan_at
        px.append([x[max(c - 1, 0)], x[c], x[max(c - 1, 0)]])
        py.append([y[r], y[max(r - 1, 0)], y[max(r - 1, 0)]])
    return np.concatenate(px).astype(np.float64), np.concatenate(py).astype(np.float64)


@pytest.mark.parametrize('shape', ('window', 'row', 'column'))
@pytest.mark.parametrize('dtype', ('float32', 'float64', 'complex64', 'complex128'))
def test_interp_points(pb, dtype, shape):
    rng = np.random.default_rng(3)
    big = rng.standard_normal((41, 67)) + 1j * rng.standard_normal((41, 67))
    big = (big if dtype.startswith('complex') else big.real).astype(dtype)
    ny, nx = {'window': (29, 43), 'row': (1, 43), 'column': (29, 1)}[shape]
    r0, c0 = 5, 11
    x = np.cumsum(rng.uniform(0.3, 1.7, nx)) - 9.0 if nx > 1 else np.array([0.25])
    y = np.cumsum(rng.uniform(0.3, 1.7, ny)) - 7.0 if ny > 1 else np.array([-0.5])
    nan_at = (7, 12) if shape == 'window' else None
    if nan_at:
        big[r0 + nan_at[0], c0 + nan_at[1]] = np.nan
    sub = big[r0:r0 + ny, c0:c0 + nx]
    px, py = point_set(x, y, nan_at)
    bt = dev(big)
    view = bt[r0:r0 + ny, c0:c0 + nx]
    out, k = launches(pb, lambda: pb._ops.interp2d_linear(view, dev(x), dev(y), dev(px), dev(py), fill=0.75,
                                                          ld=big.shape[1]))
    assert k == A.INTERP_LAUNCHES
    got = host(out)
    prec = 32 if dtype in ('float32', 'complex64') else 64
    parts = (('re', np.real), ('im', np.imag)) if dtype.startswith('complex') else (('re', np.real),)
    for part, f in parts:
        ref, maj = A.interp_ref(f(sub), x, y, px, py, 0.75 if part == 're' else 0.0)
        figure('interp_points', prec, f(got), ref, maj)
    if nan_at:
        assert np.isnan(got[-3].real) and np.isnan(got[-2].real)


@pytest.mark.parametrize('which', range(5))
def test_interp_points_sweep(pb, which):
    """1, the grid cap - 1, the cap, the cap + 1 and 3x the cap points: every grid-stride sweep writes its points"""
    count = A.sweep_counts(sm_count())[which]
    rng = np.random.default_rng(which)
    x, y = np.linspace(-2.0, 3.0, 57), np.linspace(-1.0, 2.5, 31)
    d = rng.standard_normal((31, 57))
    px, py = rng.uniform(-2.5, 3.5, count), rng.uniform(-1.5, 3.0, count)
    out, k = launches(pb, lambda: pb._ops.interp2d_linear(dev(d), dev(x), dev(y), dev(px), dev(py), fill=-3.0))
    assert k == A.INTERP_LAUNCHES
    ref, maj = A.interp_ref(d, x, y, px, py, -3.0)
    check('64/interp_sweep', fig64(host(out), ref, maj))


# ---- pb_interp2d_linear, polar ---------------------------------------------------------------------------------------
@pytest.mark.parametrize('nx', A.POLAR_N)
@pytest.mark.parametrize('ny', A.POLAR_N)
def test_interp_polar(pb, ny, nx):
    d, x, y, rmax, rows, cols = A.polar_case(ny, nx)
    for prec in (64, 32):
        dd = d.astype(NPR[prec])
        out, k = launches(pb, lambda: pb._ops.interp2d_linear(dev(dd), dev(x), dev(y), rmax=rmax))
        assert k == A.INTERP_LAUNCHES
        got = host(out)
        for sel in ({'rows': rows}, {'cols': cols}):
            ref, maj, amb = A.lattice_ref(dd, x, y, rmax, **sel)
            assert not amb.any()
            g = got[rows] if 'rows' in sel else got[:, cols]
            figure('interp_polar', prec, g, ref, maj)


# ---- pb_azimuthal_stats ----------------------------------------------------------------------------------------------
ROW = {'count': 0, 'mean': 1, 'var': 2, 'min': 3, 'max': 4, 'median': 5}
BIT = {'count': 1, 'mean': 2, 'var': 4, 'min': 8, 'max': 16, 'median': 32}


def az_check(prec, kind, got, vals, maj, cols):
    for c_i, j in enumerate(cols):
        col, mj = vals[:, c_i], maj[:, c_i]
        r = A.azstats_ref(col)
        assert got[0, j] == r['count'], (j, got[0, j], r['count'])
        sc = A.azstats_scales(col, mj)
        for s in ('mean', 'var', 'min', 'max', 'median'):
            g = got[ROW[s], j]
            if r['count'] == 0:
                assert np.isnan(g), (s, j)
                continue
            if prec == 64:
                check(f'64/az_{s}', float(abs(LD(g) - r[s]) / (LD(A.EPS) * sc[s])))
            else:                             # ulps of the rounded reference, at least the fp64 error scale
                sp = LD(np.spacing(np.abs(np.float32(r[s])))) + LD(A.EPS) * sc[s]
                check(f'32/az_{s}', float(abs(LD(np.float32(g)) - r[s]) / sp))


@pytest.mark.parametrize('kind', ('smooth', 'offset', 'nan', 'signs'))
@pytest.mark.parametrize('ny', A.AZ_NY)
def test_azimuthal_stats(pb, ny, kind):
    if ny >= 4097 and kind in ('signs',):
        pytest.skip('the signed case runs up to 513 rows')
    d, x, y, rmax, cols = A.az_case(ny, kind)
    vals = maj = None
    for prec in (64, 32):
        if prec == 32 and kind in ('offset', 'signs'):
            continue                              # float32 has neither the resolution nor the range of these cases
        dd = d.astype(NPR[prec])
        out, k = launches(pb, lambda: pb._ops.azimuthal_stats(dev(dd), dev(x), dev(y), rmax, 63))
        assert k == A.AZ_LAUNCHES
        vals, maj, amb = A.lattice_ref(dd, x, y, rmax, cols=cols)
        assert not amb.any()
        az_check(prec, kind, host(out).astype(np.float64), vals, maj, cols)
    if kind == 'nan':
        counts = np.array([A.azstats_ref(vals[:, i])['count'] for i in range(len(cols))])
        assert (counts % 2 == 0).any() and (counts % 2 == 1).any() or ny == 1


@pytest.mark.parametrize('ny', (257, 4097))
def test_azimuthal_mask_bits(pb, ny):
    """each statistic alone is one launch and the same bits as with every statistic; other rows stay NaN"""
    d, x, y, rmax, _ = A.az_case(ny, 'nan')
    args = (dev(d), dev(x), dev(y), rmax)
    full = host(pb._ops.azimuthal_stats(*args, 63))
    for s, b in BIT.items():
        out, k = launches(pb, lambda: pb._ops.azimuthal_stats(*args, b))
        assert k == 1
        out = host(out)
        assert np.array_equal(out[ROW[s]], full[ROW[s]], equal_nan=True), s
        others = [r for r in range(6) if r != ROW[s]]
        assert np.all(np.isnan(out[others]))
    for m in (BIT['mean'] | BIT['median'], BIT['var'] | BIT['min'] | BIT['count']):
        out, k = launches(pb, lambda: pb._ops.azimuthal_stats(*args, m))
        assert k == 1
        rows = [ROW[s] for s, b in BIT.items() if m & b]
        assert np.array_equal(host(out)[rows], full[rows], equal_nan=True)


def test_azimuthal_refusals(pb):
    nx = 4
    big = torch.zeros((A.AZ_MAX_NY + 1, nx), dtype=torch.float64, device='cuda')
    x, y = dev(np.arange(nx, dtype=np.float64)), dev(np.arange(A.AZ_MAX_NY + 1, dtype=np.float64))
    torch.cuda.synchronize()
    c0 = pb._ops.launch_count()
    with pytest.raises(ValueError):
        pb._ops.azimuthal_stats(big, x, y, 10.0, 63)
    out = torch.empty((6, nx), dtype=torch.float64, device='cuda')
    h = pb._capi.handle_for(torch.cuda.current_device(), torch.cuda.current_stream().cuda_stream)
    vp = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    rc = pb._capi.lib.pb_azimuthal_stats(h.ptr, 1, vp(big), A.AZ_MAX_NY + 1, nx, vp(x), vp(y), 10.0, 63, vp(out),
                                         C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == -1                                   # PB_ERR_INVALID
    small = big[:8]
    with pytest.raises(ValueError):
        pb._ops.azimuthal_stats(small, x, y[:8], 10.0, 64)
    res = pb._ops.azimuthal_stats(small, x, y[:8], 10.0, 0)
    torch.cuda.synchronize()
    assert pb._ops.launch_count() == c0
    assert torch.isnan(res).all()


# ---- pb_polar_crossings ----------------------------------------------------------------------------------------------
def crossing_call(pb, d, x, y, rmax, metric, relative, last):
    return launches(pb, lambda: pb._ops.polar_crossings(dev(d), dev(x), dev(y), rmax, metric, relative, last))


@pytest.mark.parametrize('variant', A.RAY_VARIANTS)
@pytest.mark.parametrize('nx', A.CROSS_NX)
def test_crossings_on_chunk_edges(pb, nx, variant):
    d, x, y, rmax, t = A.ray_case(nx, variant)
    vals, maj, amb = A.lattice_ref(d, x, y, rmax)
    assert not amb.any()
    exact = A.lattice_points(nx, 2, rmax)[2]
    rho, _ = A.lattice_axes(nx, 2, rmax)
    for prec in (64, 32):
        for last in (0, 1):
            for metric, relative in ((t, False), (0.5, True))[:1 if variant == 'never' else 2]:
                level, extra = A.crossing_level(vals, maj, metric, relative)
                count, mean, _, flagged = A.crossings_ref(vals, maj, rho, level, last, extra, exact=exact)
                assert not flagged.any()
                (c, m), k = crossing_call(pb, d.astype(NPR[prec]), x, y, rmax, metric, relative, last)
                assert k == A.crossing_launches(relative)
                check(f'{prec}/cross_ray', A.crossing_fig(c, m, count, mean, rmax))


@pytest.mark.parametrize('metric', tuple(A.METRICS))
@pytest.mark.parametrize('nx', A.RADIAL_NX)
def test_crossings_radial(pb, nx, metric):
    d, x, y, rmax = A.radial_case(nx)
    met, rel = A.METRICS[metric]
    rho, _ = A.lattice_axes(nx, d.shape[0], rmax)
    for prec in (64, 32):
        dd = d.astype(NPR[prec])
        vals, maj, amb = A.lattice_ref(dd, x, y, rmax)
        assert not amb.any()
        t, extra = A.crossing_level(vals, maj, met, rel)
        for last in (0, 1):
            count, mean, _, flagged = A.crossings_ref(vals, maj, rho, t, last, extra)
            assert not flagged.any() and count > 0
            (c, m), k = crossing_call(pb, dd, x, y, rmax, met, rel, last)
            assert k == A.crossing_launches(rel)
            check(f'{prec}/cross_radial', A.crossing_fig(c, m, count, mean, rmax))


@pytest.mark.parametrize('nx', A.RADIAL_NX)
def test_crossings_nan(pb, nx):
    """a NaN beside a crossing makes the mean NaN and still counts; a relative level is NaN, so nothing crosses"""
    d, x, y, rmax = A.radial_case(nx, nan=True)
    vals, maj, amb = A.lattice_ref(d, x, y, rmax)
    assert not amb.any()
    rho, _ = A.lattice_axes(nx, d.shape[0], rmax)
    for last in (0, 1):
        count, mean, _, flagged = A.crossings_ref(vals, maj, rho, 0.2, last)
        assert not flagged.any()
        (c, m), _ = crossing_call(pb, d, x, y, rmax, 0.2, False, last)
        check('64/cross_nan', A.crossing_fig(c, m, count, mean, rmax))
        (c, m), _ = crossing_call(pb, d, x, y, rmax, 0.5, True, last)
        assert c == 0 and np.isnan(m)


def test_estimate_size_keeps_nan_crossings(pb):
    """a 64^2 Gaussian (sigma 8) with a NaN patch: rays whose crossing touches the patch give NaN radii, and the
    reference's np.mean of its crossing list is NaN for both criteria"""
    x = np.arange(64) - 32.0
    d = np.exp(-(x[None, :] ** 2 + x[:, None] ** 2) / (2 * 8.0 ** 2))
    d[30:35, 44:47] = np.nan
    for crit in ('first', 'last'):
        assert np.isnan(pb.psf.estimate_size(dev(d), 0.3, dx=1.0, criteria=crit))
    with pytest.raises(ValueError, match='metric does not cross the sampled data'):
        pb.psf.estimate_size(dev(d), 'fwhm', dx=1.0)


def test_repeated_crossings_are_bit_identical(pb):
    d, x, y, rmax = A.radial_case(4097)
    a = pb._ops.polar_crossings(dev(d), dev(x), dev(y), rmax, 0.5, True, True)
    b = pb._ops.polar_crossings(dev(d), dev(x), dev(y), rmax, 0.5, True, True)
    assert a == b


# ---- pb_analytic_radial ----------------------------------------------------------------------------------------------
KINDS = {'airy': (0, 'u', 'airy', np.pi, 1.0), 'efield': (1, 'u', 'efield', np.pi, 1.0),
         'airy_ft': (2, 's', 'core', 1.0, 1.0), 'difflim': (3, 's', 'core', 1000.0, 1.0),
         'normalized': (4, 's', 'core', 1.0, 1.0), 'ee': (5, 'u', 'ee', 1.0, np.pi)}


@pytest.mark.parametrize('name', tuple(KINDS))
def test_analytic_vs_fixture(pb, name):
    kind, arg, ref_key, a, b = KINDS[name]
    z = load_golden(A.BESSEL_FIXTURE)
    sc = A.analytic_scales(z)
    ref = {'airy': z['airy_e'].astype(LD) ** 2, 'efield': z['airy_e'], 'ee': z['ee'], 'core': z['core']}[ref_key]
    xs = z[arg]
    cap = A.sweep(sm_count())
    reps = -(-(3 * cap + 1) // xs.size)
    xt = np.tile(xs, reps)
    out, k = launches(pb, lambda: pb._ops.analytic_radial(kind, dev(xt), a, b, torch.float64))
    assert k == A.ANALYTIC_LAUNCHES
    got = host(out).reshape(reps, -1)
    assert np.all(got == got[0])
    band = xs < 14 if arg == 'u' else np.ones(xs.size, bool)
    for tag, sel in (('small', band), ('large', ~band)):
        if sel.any():
            check(f'64/{name}_{tag}', A.analytic_fig(got[0][sel], np.asarray(ref, LD)[sel], sc[ref_key][sel]))
    # float32 outputs are the fp64 values rounded once; float32 inputs are the fp64 route at those inputs
    o32 = host(pb._ops.analytic_radial(kind, dev(xs), a, b, torch.float32))
    assert np.array_equal(o32, got[0].astype(np.float32), equal_nan=True)
    x32 = xs.astype(np.float32)
    i32 = host(pb._ops.analytic_radial(kind, dev(x32), a, b, torch.float64))
    i64 = host(pb._ops.analytic_radial(kind, dev(x32.astype(np.float64)), a, b, torch.float64))
    assert np.array_equal(i32, i64, equal_nan=True)


def test_zz_every_figure_has_a_measurement():
    """a figure this session reached that has no MEASURED entry is held to the bare ceiling, a bound nobody measured"""
    if os.environ.get('PB_TEST_MEASUREMENTS'):
        pytest.skip('recording figures')
    assert not LEDGER.missing(), f'no MEASURED entry (record them with PB_TEST_MEASUREMENTS): {LEDGER.missing()}'
