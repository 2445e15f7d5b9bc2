"""GPU: the wavefront-sensing kernels of csrc/wfs.cu and csrc/shack_hartmann.cu held to the high-precision references of
tests/sensing_reference.py past every chunk, vector route and per-launch split.

- pb_overlap: n on both sides of the 4096-pixel chunk and of 256 chunks (stage 2's strided loop), P on both sides of
  the 8-mode group and of the 256-pointer launch; packed and pointer-list, real and complex modes, supplied and computed
  intensity sums, SRI's c, and fields far from unit magnitude.  |eta_got - eta_ref| over the Cauchy-Schwarz majorant.
- pb_lp_modes: the 40-digit Bessel fixture (orders 0-60, through x = l and down to 1e-90), relative to each mode's
  peak; 1, 64, 65 and 129 plans; the core / cladding choice at r = a (1 +- k ulp) under both rules; the azimuth.
- pb_psi: both routes for every frame type; int64 sums past 2^53 bit for bit; 65 frames refused.
- pb_subaperture_centroids: both routes on the same data give the same bits; lenslets straddling chunk boundaries;
  614 / 615 / 1075 lenslet columns and 1076 refused; NaN and empty subapertures.
- pb_sh_reconstruct: M, K and F across the tree, the strided loop and the 65535-frame grid limit.
- pb_lenslet_screen at 2048^2 with 64^2 lenslets against a numpy restatement of the reference's loop.
- pb_wfs_combine and pb_grating against their references; the rectangle grating bit for bit.

Bounds are 1.5x the figures measured on an H100 (`MEASURED`, recorded with PB_TEST_MEASUREMENTS) and never above the
ceilings tests/test_host_sensing_reference.py shows every modelled defect exceeds by 10x or more.
"""
import math
import os

import numpy as np
import pytest
import torch

import scipy.special as sps

import sensing_reference as S
from accuracy import Ledger
from conftest import load_golden
from gpu_fixtures import pb, crand, dev, host, launches, routes_of  # noqa: F401

pytestmark = pytest.mark.gpu

PRECS = (32, 64)
RT = {32: torch.float32, 64: torch.float64}
CT = {32: torch.complex64, 64: torch.complex128}
NPR = {32: np.float32, 64: np.float64}
NPC = {32: np.complex64, 64: np.complex128}
TORCH_OF = {'float32': torch.float32, 'float64': torch.float64, 'uint16': torch.uint16, 'int32': torch.int32}
ELEM = {'float32': 0, 'float64': 1, 'uint16': 5, 'int32': 7}

# ceilings, shown by the host test to sit 10x or more below every modelled defect
CEIL = {'overlap': 1e-13, 'lp': 1e-9, 'psi': 1e-13, 'psi_phase64': 1e-12, 'psi_phase32': 1e-6,
        'centroid64': 1e-12, 'centroid32': 1e-6, 'flux64': 1e-13, 'flux32': 1e-6, 'recon': 1e-13,
        'screen64': 1e-13, 'screen32': 1e-6, 'combine64': 1e-14, 'combine32': 1e-6, 'grating_sin64': 1e-14,
        'grating_sin32': 1e-6}

# ---- measured figures (H100 80GB HBM3, 700 W power limit, 1980 MHz SM clock); bounds are 1.5x these, capped at the
# ceiling ------------------------------------------------------------------------------------------------------------
MEASURED = {
    '32/combine': 5.61e-08,
    '32/grating_sin': 2.98e-08,
    '32/lenslet_screen': 2.98e-08,
    '32/overlap_c_ulps': 0.484,
    '32/overlap_scaled_ulps': 0.413,
    '32/overlap_ulps': 0.5,
    '64/combine': 3.59e-16,
    '64/grating_sin': 8.64e-16,
    '64/lenslet_screen': 1.27e-16,
    '64/lp_fixture': 1.31e-10,
    '64/overlap': 4.44e-16,
    '64/overlap_c': 2.78e-16,
    '64/overlap_scaled': 1.25e-16,
    '64/reconstruct': 2.04e-16,
    'float32/centroid': 2.98e-08,
    'float32/flux': 5.57e-08,
    'float32/psi_phase': 1.19e-07,
    'float64/centroid': 7.31e-14,
    'float64/flux': 4.68e-16,
    'float64/psi_phase': 1.38e-15,
    'float64/psi_sums': 6.01e-16,
    'int32/centroid': 2.07e-08,
    'int32/psi_phase': 9.4e-16,
    'int32/psi_sums': 8.37e-16,
    'uint16/centroid': 2.07e-08,
    'uint16/psi_phase': 9.54e-16,
    'uint16/psi_sums': 6.63e-16,
}



def ceiling(name):
    """the CEIL entry of a figure: per quantity, and per output precision where the quantity has two"""
    tag, fig = name.split('/')
    if fig.endswith('_ulps'):                 # float32 outputs in ulps of the rounded reference
        return 1.0
    key = {'overlap_c': 'overlap', 'overlap_scaled': 'overlap', 'lp_fixture': 'lp', 'psi_sums': 'psi',
           'reconstruct': 'recon', 'lenslet_screen': 'screen'}.get(fig, fig)
    if key in CEIL:
        return CEIL[key]
    # integer frames give float32 centroids and fluxes, and fp64 phases
    f32 = tag in ('32', 'float32') or (tag in ('uint16', 'int32') and fig != 'psi_phase')
    return CEIL[key + ('32' if f32 else '64')]


# the worst figure of each name over the whole file
LEDGER = Ledger(MEASURED, ceiling)
check = LEDGER.check


def wrap(a):
    return a - 2 * np.pi * np.round(a / (2 * np.pi))


# ---- pb_overlap --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('variant', ('packed', 'ptrs_real', 'supplied'))
@pytest.mark.parametrize('n,P', S.overlap_cases())
@pytest.mark.parametrize('prec', PRECS)
def test_overlap(pb, prec, n, P, variant):
    E = crand(n, 1, NPC[prec])
    rng = np.random.default_rng(2)
    if variant == 'ptrs_real':
        modes = rng.standard_normal((P, n)).astype(NPR[prec])
    else:
        modes = crand((P, n), 2, NPC[prec])
    modes[:, ::3] += (E[::3] * 0.5).real if variant == 'ptrs_real' else E[::3] * 0.5    # eta above the noise
    eta_ref, maj, ip, ie = S.overlap_ref(E, modes)
    Ed, Md = dev(E), dev(modes)
    ipd = dev(ip.astype(np.float64)) if variant == 'supplied' else None
    ied = dev(np.array([ie], np.float64)) if variant == 'supplied' else None
    arg = list(Md) if variant == 'ptrs_real' else Md
    (eta, c), k = launches(pb, lambda: pb._ops.overlap(Ed, arg, ipd, ied, want_c=True))
    assert k == S.overlap_launches(P)
    c_ref = S.coupling_c_ref(eta_ref[0], ie)
    overlap_figures(prec, 'overlap', host(eta), eta_ref, maj)
    overlap_figures(prec, 'overlap_c', host(c).reshape(1), np.array([c_ref]), np.array([c_ref / math.sqrt(eta_ref[0])]))


def overlap_figures(prec, name, got, ref, maj):
    """fp64 outputs: |got - ref| over the majorant; float32 outputs: |got - ref| in ulps of the float32-rounded
    reference (the fp64 sums are rounded once, so this stays below 1)"""
    if prec == 64:
        check(f'64/{name}', S.overlap_fig(got, ref, maj))
    else:
        r32 = ref.astype(np.float32)
        check(f'32/{name}_ulps', np.max(np.abs(got.astype(S.LDBL) - ref) / np.spacing(np.abs(r32))))


@pytest.mark.parametrize('scale', ('tiny', 'huge'))
@pytest.mark.parametrize('prec', PRECS)
def test_overlap_scale(pb, prec, scale):
    """fields scaled by 1e-150 / 1e150 (complex128) and 1e-30 / 1e30 (complex64): the fp64 sums neither under- nor
    overflow"""
    f = {64: {'tiny': 1e-150, 'huge': 1e150}, 32: {'tiny': 1e-30, 'huge': 1e30}}[prec][scale]
    n, P = 3 * S.OVERLAP_CHUNK + 5, 9
    E = crand(n, 3, NPC[prec], f)
    modes = crand((P, n), 4, NPC[prec], f)
    modes[:, ::2] += E[::2]
    eta_ref, maj, ip, ie = S.overlap_ref(E, modes)
    eta, _ = pb._ops.overlap(dev(E), dev(modes))
    overlap_figures(prec, 'overlap_scaled', host(eta), eta_ref, maj)


# ---- pb_lp_modes ---------------------------------------------------------------------------------------------------
def bessel_groups():
    """the fixture rows grouped into modes: one plan row per (kind, l, arg), the radius grid is every row's rho"""
    z = load_golden(S.BESSEL_FIXTURE)
    keys = np.stack((z['kind'], z['l'], z['arg']), axis=1)
    uniq, inv = np.unique(keys, axis=0, return_inverse=True)
    return z, uniq, inv.reshape(-1)


@pytest.mark.parametrize('prec', PRECS)
def test_lp_bessel_fixture(pb, prec):
    z, uniq, inv = bessel_groups()
    plan = np.array([[l, l, (a if k == 0 else 1.0), (a if k == 1 else 1.0), 0, 0] for k, l, a in uniq])
    r = z['rho'].astype(NPR[prec])
    rd = dev(r)
    out, k = launches(pb, lambda: pb._ops.lp_modes(rd, None, 1.0, plan))
    assert k == S.lp_launches(len(plan))
    got = host(out)[inv, np.arange(len(inv))]
    if prec == 64:
        ref = z['val']
        peak = np.zeros(len(uniq))
        np.maximum.at(peak, inv, np.abs(ref))
        check('64/lp_fixture', np.max(np.abs(got - ref) / peak[inv]))
    else:
        # the same fp64 arithmetic on the float32 radii, rounded once: the fp64 route at those radii, rounded
        o64 = host(pb._ops.lp_modes(dev(r.astype(np.float64)), None, 1.0, plan))[inv, np.arange(len(inv))]
        assert np.array_equal(got, o64.astype(np.float32), equal_nan=True)
    assert np.all(np.isfinite(got))


def test_lp_tiny_arguments(pb):
    """below x = 1e-20 J_l is (x/2)^l / l! (the next term is 1e-40 of it); Miller's recurrence there would outrun its
    1e-100 rescaling and overflow to NaN for x < ~2 m 1e-100"""
    ls = (2, 3, 5, 20, 60)
    xs = np.array([0.0, 1e-100, 1.1e-100, 1e-99, 1e-98, 1e-90, 1e-60, 1e-30, 1e-21, 1e-20 * (1 - 2.0 ** -52), 1e-19])
    plan = np.array([[l, l, 1.0, 1.0, 0, 0] for l in ls])
    got = host(pb._ops.lp_modes(dev(xs), None, 1.0, plan))
    for p, l in enumerate(ls):
        lead = np.array([(S.LDBL(x) / 2) ** l / S.LDBL(math.factorial(l)) for x in xs])
        ref = (lead / S.LDBL(sps.jv(l, 1.0))).astype(np.float64)
        assert np.all(np.isfinite(got[p])), (l, got[p])
        assert np.all(np.abs(got[p] - ref) <= 64 * np.spacing(np.abs(ref)) + np.nextafter(0.0, 1.0) * 4), (l, got[p], ref)


@pytest.mark.parametrize('rule', (0, 1))
@pytest.mark.parametrize('prec', PRECS)
def test_lp_boundary_and_azimuth(pb, prec, rule):
    """r = a (1 + k ulp): the core is r <= a (LP rule) or r * (1/a) < 1 (SMF rule), decided in fp64 on the stored r.
    With ld != l the two branches give different values at rho = 1, so a wrong choice shows."""
    a = 1.7
    dt = NPR[prec]
    base = dt(a)
    r = np.array([np.nextafter(base, dt(np.inf) if k > 0 else dt(0)) if k else base for k in (-3, -2, -1, 0, 1, 2, 3)],
                 dtype=dt)
    for _ in range(2):
        r = np.concatenate((r, [np.nextafter(r[-1], dt(np.inf))]))
    U, Wv = 1.0, 1.5
    plan = np.array([[0, 1, U, Wv, rule, 0]])
    got = host(pb._ops.lp_modes(dev(r), None, a, plan))[0]
    rd = r.astype(np.float64)
    rho = rd / a if rule == 0 else rd * (1.0 / a)
    core = rd <= a if rule == 0 else rho < 1.0
    jv = sps.jv(0, U * rho) / sps.jv(1, U)
    kv = sps.kv(0, Wv * rho) / sps.kv(1, Wv)
    ref = np.where(core, jv, kv)
    assert np.all(np.abs(got - ref) <= 1e-6 * np.abs(ref)), (got, ref, core)
    # azimuth: cos(l t) and sin(l t) on an angle grid, against the plain mode times the factor in fp64
    t = np.linspace(-np.pi, np.pi, 1001).astype(dt)
    rr = np.full_like(t, dt(0.8))
    plan = np.array([[3, 3, 2.4, 1.0, rule, az] for az in (0, 1, 2)])
    o = host(pb._ops.lp_modes(dev(rr), dev(t), a, plan)).astype(np.float64)
    plain = o[0].astype(np.float64)
    td = t.astype(np.float64)
    tol = 4 * np.spacing(dt(1)) * np.abs(plain).max()
    assert np.max(np.abs(o[1] - plain * np.cos(3 * td))) <= tol
    assert np.max(np.abs(o[2] - plain * np.sin(3 * td))) <= tol


@pytest.mark.parametrize('P', S.LP_P)
@pytest.mark.parametrize('prec', PRECS)
def test_lp_launch_split(pb, prec, P):
    """P plans in ceil(P / 64) launches: plane p is the same mode evaluated alone"""
    r = np.linspace(0, 3, 4099).astype(NPR[prec])
    orders = np.arange(P) % 13
    plan = np.array([[l, l, 2.0 + 0.01 * p, 1.0 + 0.02 * p, p % 2, 0] for p, l in enumerate(orders)])
    rd = dev(r)
    out, k = launches(pb, lambda: pb._ops.lp_modes(rd, None, 1.3, plan))
    assert k == S.lp_launches(P)
    out = host(out)
    for p in sorted({0, P // 2, S.LP_MAX - 1, S.LP_MAX, P - 1} & set(range(P))):
        one = host(pb._ops.lp_modes(rd, None, 1.3, plan[p:p + 1]))[0]
        assert np.array_equal(out[p], one), p


# ---- pb_psi ----------------------------------------------------------------------------------------------------------
def psi_frames(N, n, dtype, seed):
    rng = np.random.default_rng(seed)
    ph = rng.uniform(-np.pi, np.pi, n)
    if dtype in ('float32', 'float64'):
        g, s, c = S.fringes(N, n, ph, dtype)
        return g, s, c
    hi = 60000 if dtype == 'uint16' else 2 ** 31 - 1
    g, s, c = S.fringes(N, n, ph, np.float64, amp=0.45 * hi, bias=0.5 * hi)
    return np.clip(np.rint(g), 0, hi).astype(dtype), s, c


def psi_call(pb, g, s, c, num_dt, phase_dt, offset, as_list):
    N, n = g.shape
    if offset:                        # a 1-D buffer sliced by one element: every frame misaligned
        buf = torch.zeros(N * n + 1, dtype=TORCH_OF[g.dtype.name], device='cuda')
        buf[1:] = dev(g.reshape(-1))
        frames = buf[1:].view(N, n)
    else:
        frames = dev(g)
    arg = list(frames) if as_list else frames
    codes = {(v, i): pb._capi.route_code(pb._capi.ROUTE_PSI, v, i) for v in (1, 2, 4, 8) for i in (0, 1)}
    res, r = routes_of(lambda: pb._ops.psi(arg, s, c, num_dt, phase_dt), codes)
    return [host(t) for t in res], r


@pytest.mark.parametrize('route', ('vec', 'odd_n', 'offset'))
@pytest.mark.parametrize('N', S.PSI_FRAMES)
@pytest.mark.parametrize('dtype', S.PSI_TYPES)
def test_psi(pb, dtype, N, route):
    n = 3 * 4096 + (1 if route == 'odd_n' else 0)
    g, s, c = psi_frames(N, n, dtype, 5 + N)
    flt = dtype in ('float32', 'float64')
    num_dt = TORCH_OF[dtype] if flt else torch.float64
    phase_dt = TORCH_OF[dtype] if flt else torch.float64
    (num, den, ph), r = psi_call(pb, g, s, c, num_dt, phase_dt, route == 'offset', N % 2 == 1)
    V = S.psi_route(n, dtype, aligned=route != 'offset')
    assert r == {(V, 0): 1, 'all': 1}, r
    rn, rc, an, ac = S.psi_ref(g, s, c)
    if dtype == 'float32':
        for got, ref in ((num, rn), (den, rc)):
            r32 = ref.astype(np.float32)
            assert np.all(np.abs(got.astype(np.float64) - r32) <= np.spacing(np.abs(r32))), 'float32 sums'
    else:
        check(f'{dtype}/psi_sums', max(np.max(np.abs(num - rn) / np.maximum(an, 1e-300)),
                                       np.max(np.abs(den - rc) / np.maximum(ac, 1e-300))))
    pref = np.arctan2(rn, rc)
    check(f'{dtype}/psi_phase', np.max(np.abs(wrap(ph.astype(S.LDBL) - pref))))


@pytest.mark.parametrize('route', ('vec', 'odd_n', 'offset'))
@pytest.mark.parametrize('dtype', ('uint16', 'int32'))
def test_psi_int64_exact(pb, dtype, route):
    """integer frames and integer weights: the int64 sums are exact, also past 2^53 where fp64 would round"""
    N = S.PSI_MAX
    n = 4096 + (1 if route == 'odd_n' else 0)
    rng = np.random.default_rng(9)
    hi = 65535 if dtype == 'uint16' else 2 ** 31 - 1
    g = (hi - rng.integers(0, 1000, (N, n))).astype(dtype)
    big = 2 ** 40 if dtype == 'uint16' else 2 ** 26
    s = (rng.integers(-1, 2, N) * big + rng.integers(-999, 1000, N) * 2 + 1).astype(np.float64)
    c = (rng.integers(0, 2, N) * big + rng.integers(-999, 1000, N) * 2 + 1).astype(np.float64)
    (num, den, ph), r = psi_call(pb, g, s, c, torch.int64, torch.float64, route == 'offset', False)
    V = S.psi_route(n, dtype, aligned=route != 'offset')
    assert r == {(V, 1): 1, 'all': 1}, r
    en, ec = S.psi_int_ref(g, s, c)
    assert max(np.abs(en).max(), np.abs(ec).max()) > 2 ** 53
    assert np.array_equal(num, en) and np.array_equal(den, ec)
    check(f'{dtype}/psi_phase', np.max(np.abs(wrap(ph.astype(S.LDBL) - np.arctan2(en.astype(S.LDBL), ec.astype(S.LDBL))))))


def test_psi_refuses_65_frames(pb):
    g = dev(np.ones((S.PSI_MAX + 1, 64), np.float32))
    torch.cuda.synchronize()
    c0 = pb._ops.launch_count()
    with pytest.raises(ValueError):
        pb._ops.psi(g, np.zeros(S.PSI_MAX + 1), np.ones(S.PSI_MAX + 1), torch.float32, torch.float32)
    assert pb._ops.launch_count() == c0


# ---- pb_subaperture_centroids --------------------------------------------------------------------------------------
def centroid_setup(W, dtype, pitch=24, rows=2, F=2, seed=11):
    H = rows * pitch
    xv = np.arange(W, dtype=np.float64) - W // 2
    yv = np.arange(H, dtype=np.float64) - H // 2 + 0.5
    ncols = -(-W // pitch) + 1
    xc, yc = S.centres(pitch, ncols), S.centres(pitch, rows)
    rng = np.random.default_rng(seed)
    if dtype in ('float32', 'float64'):
        fr = rng.uniform(0, 1, (F, H, W)).astype(dtype)
    else:
        hi = 65535 if dtype == 'uint16' else 2 ** 30
        fr = rng.integers(0, hi, (F, H, W)).astype(dtype)
    return fr, xv, yv, xc, yc, ncols, rows


def centroid_call(pb, fr, xv, yv, pitch, n, threshold, offset):
    F, H, W = fr.shape
    if offset:
        buf = torch.zeros(F * H * W + 1, dtype=TORCH_OF[fr.dtype.name], device='cuda')
        buf[1:] = dev(fr.reshape(-1))
        frames = buf[1:].view(F, H, W)
    else:
        frames = dev(fr)
    plan = pb.shack_hartmann.CentroidPlan(xv, yv, pitch, n)
    codes = {v: pb._capi.route_code(pb._capi.ROUTE_CENTROID, v, ELEM[fr.dtype.name]) for v in (1, 4)}
    (disp, flux), r = routes_of(lambda: plan(frames, threshold), codes)
    return host(disp), host(flux), r


@pytest.mark.parametrize('offset', (False, True))
@pytest.mark.parametrize('threshold', (0.0, 0.3))
@pytest.mark.parametrize('W', S.CENTROID_W)
@pytest.mark.parametrize('dtype', S.CENTROID_TYPES)
def test_centroids(pb, dtype, W, threshold, offset):
    pitch = 24
    fr, xv, yv, xc, yc, ncols, rows = centroid_setup(W, dtype, pitch)
    disp, flux, r = centroid_call(pb, fr, xv, yv, pitch, (rows, ncols), threshold, offset)
    V = S.centroid_route(W, ncols, aligned=not offset)
    assert r == {V: 1, 'all': 1}, r
    if W > S.THREADS * V:             # some lenslet straddles a chunk boundary of this route
        own = S.owners(xv, xc, pitch)
        assert any(len(set(np.flatnonzero(own == i) // (S.THREADS * V))) > 1 for i in range(ncols))
    dref, fref, scale = S.centroid_ref(fr, xv, yv, xc, yc, pitch, threshold)
    assert np.array_equal(np.isnan(disp), np.isnan(dref.astype(np.float64)))
    check(f'{dtype}/centroid', S.centroid_fig(disp, dref, scale))
    if dtype in ('uint16', 'int32'):
        assert np.array_equal(flux, fref.astype(np.float64).astype(np.float32))
    else:
        ok = fref > 0
        check(f'{dtype}/flux', np.max(np.abs(flux[ok] - fref[ok]) / fref[ok]))
    if not offset and V == S.CENTROID_VEC:
        # the same data through the one-column route gives the same bits
        d1, f1, r1 = centroid_call(pb, fr, xv, yv, pitch, (rows, ncols), threshold, True)
        assert r1 == {1: 1, 'all': 1}
        assert np.array_equal(d1, disp, equal_nan=True) and np.array_equal(f1, flux, equal_nan=True)


@pytest.mark.parametrize('ncols', S.CENTROID_NCOLS)
def test_centroid_lenslet_columns(pb, ncols):
    """614 columns take V = 4, 615 and 1075 V = 1, 1076 are refused; lenslets past the grid own nothing (NaN)"""
    pitch, W = 2, 2048
    fr, xv, yv, xc, yc, _, rows = centroid_setup(W, 'float32', pitch, rows=2, F=1)
    xc = S.centres(pitch, ncols)
    V = S.centroid_route(W, ncols)
    if V is None:
        with pytest.raises(RuntimeError):
            centroid_call(pb, fr, xv, yv, pitch, (rows, ncols), 0.0, False)
        return
    disp, flux, r = centroid_call(pb, fr, xv, yv, pitch, (rows, ncols), 0.0, False)
    assert r == {V: 1, 'all': 1}, r
    dref, fref, scale = S.centroid_ref(fr, xv, yv, xc, yc, pitch)
    assert np.array_equal(np.isnan(disp), np.isnan(dref.astype(np.float64)))
    check('float32/centroid', S.centroid_fig(disp, dref, scale))


@pytest.mark.parametrize('dtype', ('float32', 'float64'))
def test_centroid_nan_and_empty(pb, dtype):
    """a NaN pixel poisons its own subaperture only; an all-zero subaperture has NaN displacement and zero flux"""
    pitch, W = 24, 1025
    fr, xv, yv, xc, yc, ncols, rows = centroid_setup(W, dtype, pitch)
    d0, f0, _ = centroid_call(pb, fr, xv, yv, pitch, (rows, ncols), 0.0, False)
    own, rown = S.owners(xv, xc, pitch), S.owners(yv, yc, pitch)
    bad = fr.copy()
    i_nan, i_zero = 21, 22
    c_nan = np.flatnonzero(own == i_nan)[5]
    bad[0, np.flatnonzero(rown == 0)[3], c_nan] = np.nan
    bad[1][np.ix_(rown == 0, own == i_zero)] = 0
    d1, f1, _ = centroid_call(pb, bad, xv, yv, pitch, (rows, ncols), 0.0, False)
    hit = np.zeros_like(np.isnan(d0))
    hit[0, :, 0, i_nan] = True
    hit[1, :, 0, i_zero] = True
    assert np.all(np.isnan(d1[hit]))
    assert np.isnan(f1[0, 0, i_nan]) and f1[1, 0, i_zero] == 0
    assert np.array_equal(d1[~hit], d0[~hit], equal_nan=True)
    fh = np.zeros(f0.shape, bool)
    fh[0, 0, i_nan] = fh[1, 0, i_zero] = True
    assert np.array_equal(f1[~fh], f0[~fh])


# ---- pb_sh_reconstruct ---------------------------------------------------------------------------------------------
RECON_CASES = [(M, K, 16) for M in S.RECON_M for K in S.RECON_K] + [(M, 10, 1) for M in S.RECON_M] +     [(1, 1, S.GRID_Y_MAX), (257, 10, S.GRID_Y_MAX)]


@pytest.mark.parametrize('M,K,F', RECON_CASES)
@pytest.mark.parametrize('prec', PRECS)
def test_reconstruct(pb, prec, M, K, F):
    frame = (2, 64, 64)
    rng = np.random.default_rng(M * 7 + K)
    idx = rng.permutation(8192)[:M].astype(np.int32)
    ref = rng.standard_normal(M) * 0.1
    R = rng.standard_normal((K, M))
    sl = rng.standard_normal((F,) + frame).astype(NPR[prec])
    out, k = launches(pb, lambda: pb._ops.sh_reconstruct(dev(sl), dev(idx), dev(ref), dev(R), frame))
    assert k == 1
    want, mag = S.reconstruct_ref(sl, idx, ref, R)
    got = host(out).astype(S.LDBL)
    if prec == 64:
        check('64/reconstruct', np.max(np.abs(got - want) / mag))
    else:
        w32 = want.astype(np.float32)
        assert np.all(np.abs(got - w32) <= np.spacing(np.abs(w32)) + 1e-13 * mag)


@pytest.mark.parametrize('prec', PRECS)
def test_reconstruct_nan_and_limit(pb, prec):
    frame = (2, 8, 8)
    rng = np.random.default_rng(3)
    idx = rng.permutation(128)[:100].astype(np.int32)
    R = rng.standard_normal((7, 100))
    sl = rng.standard_normal((4,) + frame).astype(NPR[prec])
    args = (dev(idx), None, dev(R), frame)
    o0 = host(pb._ops.sh_reconstruct(dev(sl), *args))
    bad = sl.copy()
    bad[2].reshape(-1)[idx[37]] = np.nan
    o1 = host(pb._ops.sh_reconstruct(dev(bad), *args))
    assert np.all(np.isnan(o1[2]))
    keep = [0, 1, 3]
    assert np.array_equal(o1[keep], o0[keep])
    big = torch.zeros((S.GRID_Y_MAX + 1,) + frame, dtype=RT[prec], device='cuda')
    torch.cuda.synchronize()
    c0 = pb._ops.launch_count()
    with pytest.raises(RuntimeError):
        pb._ops.sh_reconstruct(big, *args)
    assert pb._ops.launch_count() == c0


# ---- pb_lenslet_screen ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('grid', ('general', 'edges_on_samples'))
@pytest.mark.parametrize('aperture', ('rectangle', 'circle'))
@pytest.mark.parametrize('prec', PRECS)
def test_lenslet_screen(pb, prec, aperture, grid):
    N, n, pitch, efl, wvl = 2048, 64, 1.0, 20.0, 0.6328
    dx = 1 / 32 if grid == 'edges_on_samples' else 1.0 / 31.37
    dt = NPR[prec]
    v = ((np.arange(N) - N // 2) * dx).astype(dt)
    x, y = np.meshgrid(v, v)
    pb.config.precision = prec
    try:
        ap = pb.shack_hartmann.rectangle if aperture == 'rectangle' else pb.geometry.circle
        out, k = launches(pb, lambda: pb.shack_hartmann.shack_hartmann(pitch, n, efl, wvl, dev(x), dev(y),
                                                                          aperture=ap))
    finally:
        pb.config.precision = 64
    assert k == 1
    total = S.lenslet_phase(x, y, pitch, (n, n), efl, aperture, dt)
    kphase = (-1j * 2 * np.pi / (wvl / 1e3)).imag
    cr, ci = S.lenslet_field_ref(total, kphase)
    got = host(out)
    fig = max(np.max(np.abs(got.real - cr)), np.max(np.abs(got.imag - ci)))
    check(f'{prec}/lenslet_screen', fig)
    assert np.count_nonzero(total) > N * N // 2


# ---- pb_wfs_combine and pb_grating -----------------------------------------------------------------------------------
@pytest.mark.parametrize('real_out', (False, True))
@pytest.mark.parametrize('two', (False, True))
@pytest.mark.parametrize('prec', PRECS)
def test_combine(pb, prec, two, real_out):
    n = 1024 * 1024 + 3
    a, b = crand(n, 21, NPC[prec]), crand(n, 22, NPC[prec])
    al, be = 0.3 - 1.7j, -2.1 + 0.4j
    sa = np.array(1.25, NPR[prec])
    out, k = launches(pb, lambda: pb._ops.wfs_combine(dev(a), al, dev(b) if two else None, be, alpha_scale=dev(sa),
                                                      real_out=real_out))
    assert k == 1
    ref = S.combine_ref(a, al * S.LDBL(sa), b if two else None, be, real_out)
    got = host(out)
    fig = np.max(np.abs(got.astype(np.clongdouble) - ref)) / np.max(np.abs(ref))
    check(f'{prec}/combine', fig)


@pytest.mark.parametrize('period', (0.37, -0.37, 2.0))
@pytest.mark.parametrize('prec', PRECS)
def test_grating_rectangle_exact(pb, prec, period):
    dt = NPR[prec]
    rng = np.random.default_rng(4)
    special = np.array([0.0, -0.0, period, -period, 3 * period, -7 * period, 1e16, -1e16, 1e16 + 2, -2.5, 1e-300,
                        -1e-300, 0.5 * period, np.nextafter(period, 0), np.nextafter(-period, 0)])
    x = np.concatenate((special, rng.uniform(-50, 50, 100000))).astype(dt)
    params = (period, 0.5 * abs(period) * np.sign(period), 1.0, 0.25, 0.6, 1e-9)
    shift = 0.0125
    for E in (None, crand(x.size, 5, NPC[prec])):
        got = host(pb._ops.grating(1, dev(x), params, shift, None if E is None else dev(E)))
        g = S.grating_rect_ref(x, shift, *params)
        if E is None:
            assert np.array_equal(got, g.astype(dt))
        else:
            want = (E.real.astype(np.float64) * g).astype(dt) + 1j * (E.imag.astype(np.float64) * g).astype(dt)
            assert np.array_equal(got, want.astype(NPC[prec]))


@pytest.mark.parametrize('prec', PRECS)
def test_grating_sin(pb, prec):
    x = np.random.default_rng(6).uniform(-3, 3, 1 << 20).astype(NPR[prec])
    got = host(pb._ops.grating(0, dev(x), (41.3,), 0.002))
    ref = S.grating_sin_ref(x, 0.002, 41.3)
    check(f'{prec}/grating_sin', np.max(np.abs(got - ref)))


def test_zz_every_figure_has_a_measurement():
    """a figure this session reached that has no MEASURED entry is held to the bare ceiling, a bound nobody measured"""
    if os.environ.get('PB_TEST_MEASUREMENTS'):
        pytest.skip('recording figures')
    assert not LEDGER.missing(), f'no MEASURED entry (record them with PB_TEST_MEASUREMENTS): {LEDGER.missing()}'
