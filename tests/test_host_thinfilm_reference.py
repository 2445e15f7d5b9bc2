"""CPU: the references of tests/thinfilm_reference.py against closed forms, against mpmath at 50 digits (the sweep and
central differences of it), against the committed fixtures of the reference package (tests/golden/thinfilm*.npz and
coating_design*.npz) within their own fp64 agreement, the launch rules the GPU suite's sweep cases rely on, and every
defect model against the GPU test's ceilings: each faithful fp64 model stays under its ceiling and each defect lands
10x or more above."""
import numpy as np
import pytest

import coating_design_oracle as D
import thinfilm_oracle as O
import thinfilm_reference as T
from accuracy import LDBL, sweep
from conftest import load_golden
from test_gpu_thinfilm_vs_fp64 import CEIL, STACKS, GRID_W, GRID_TH


def samples(name, model=False, wvl=GRID_W, theta=GRID_TH):
    n, d, sub, amb = STACKS[name]
    return T.Samples(wvl, theta, amb, sub, np.asarray(n, complex), np.asarray(d, float), model=model)


def resolve(ns, w):
    """the reference's _resolve of every layer index at w, as one (layers, *w shape) table"""
    vals = [n.nk(w) if callable(getattr(n, 'nk', None)) else n(w) if callable(n) else n for n in ns]
    tab = np.empty((len(vals),) + (np.broadcast_shapes(*[np.shape(v) for v in vals]) if vals else ()), complex)
    for j, v in enumerate(vals):
        tab[j] = v
    return tab


def rel(a, b, floor=0.0):
    a, b = np.asarray(a).astype(np.complex128), np.asarray(b)
    den = max(float(np.abs(b).max()) if b.size else 0.0, floor)
    return float(np.abs(a - b).max()) / (den or 1.0) if b.size else 0.0


# ---- launch rules --------------------------------------------------------------------------------------------------
def test_launch_rules_at_132_sms():
    s256, s128 = sweep(132, 256), sweep(132, 128)
    assert (s256, s128) == (540672, 270336)
    c256, c128 = T.straddle_counts(132, 256), T.straddle_counts(132, 128)
    assert c256 == (1, 31, 32, 33, s256 - 1, s256, s256 + 1, 2 * s256 + 33)
    assert c128[4:] == (s128 - 1, s128, s128 + 1, 2 * s128 + 33)
    for threads, counts in ((256, c256), (128, c128)):
        # one and two (and three) grid sweeps
        assert [T.visits(c, 132, threads) for c in counts] == [1, 1, 1, 1, 1, 1, 2, 3]
        W = 132 * 16 * threads // 32
        slots = [T.warp_slots(c, 132, threads) for c in counts]
        # the warp edges: one slot, then two from 33 on; nw < W below a full grid and nw = W from it on
        assert [nw for _, nw in slots[:4]] == [1, 1, 1, 2]
        assert all(nw < w for w, nw in slots[:4]) and all((w, nw) == (W, W) for w, nw in slots[5:])
        assert slots[4] == (W, W)                  # sweep - 1 still fills the last warp's slot
    assert [T.cm_threads(1), T.cm_threads(2)] == [256, 128]
    assert [T.cpad(c) for c in (1, 31, 32, 33)] == [32, 32, 32, 64]


def test_slot_sum_is_the_plain_sum():
    c = np.random.default_rng(0).standard_normal((2, 2 * sweep(4) + 33))
    assert np.allclose(T.slot_sum(c, 4, 256), c.sum(-1), rtol=0, atol=1e-10)


# ---- closed forms --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('pol', (T.POL_S, T.POL_P))
def test_single_interface_is_fresnel(pol):
    th = np.radians([0.0, 20.0, 50.0])
    n0, ns = 1.2, 1.52
    c0 = np.cos(th.astype(LDBL))
    cs = np.sqrt(1 - (LDBL(n0) / LDBL(ns) * np.sin(th.astype(LDBL))) ** 2)
    S = T.Samples(0.55, th, n0, ns, np.zeros(0, complex), np.zeros(0))
    f = T.forward(S, pol)
    if pol == T.POL_S:
        want = (n0 * c0 - ns * cs) / (n0 * c0 + ns * cs)
    else:
        want = (n0 / c0 - ns / cs) / (n0 / c0 + ns / cs)
    assert np.max(np.abs(f['r'] - want)) < 1e-18
    # multilayer_stack_rt needs a layer: a zero-thickness one is the bare interface (its own sign convention for p)
    S1 = T.Samples(0.55, th, n0, ns, np.array([1.9 + 0j]), np.array([0.0]))
    g = T.forward(S1, pol, T.THINFILM)
    want = ((n0 * c0 - ns * cs) / (n0 * c0 + ns * cs) if pol == T.POL_S
            else (n0 * cs - ns * c0) / (n0 * cs + ns * c0))
    assert np.max(np.abs(g['r'] - want)) < 1e-18


def test_quarter_wave_ar_layer():
    n1 = np.sqrt(1.52)
    S = T.Samples(0.55, 0.0, 1.0, 1.52, np.array([n1 + 0j]), np.array([0.55 / 4 / n1]))
    assert float(T.forward(S, T.POL_S)['R'][0]) < 1e-30


def test_zero_thickness_layer_is_the_identity():
    n, d = [1.38, 2.05, 1.5 + 0.2j], [0.1, 0.08, 0.05]
    a = T.Samples(GRID_W, GRID_TH, 1.0, 1.52, np.array(n, complex), np.array(d))
    b = T.Samples(GRID_W, GRID_TH, 1.0, 1.52, np.array(n[:1] + [1.9] + n[1:], complex), np.array(d[:1] + [0.0] + d[1:]))
    for pol in (T.POL_S, T.POL_P):
        fa, fb = T.forward(a, pol), T.forward(b, pol)
        assert np.array_equal(fa['r'], fb['r']) and np.array_equal(fa['t'], fb['t'])
        assert np.array_equal(fb['E'][1], fb['E'][2])


@pytest.mark.parametrize('pol', (T.POL_S, T.POL_P))
def test_energy_balance_and_tir(pol):
    f = T.forward(samples('absorb'), pol)
    tot = f['R'] + f['T'] + f['A'].sum(0)
    assert float(np.max(np.abs(tot - 1))) < 1e-17 and float(f['A'][1].min()) > 0
    S = T.Samples(0.55, np.radians([40.0, 60.0, 85.0]), 1.7, 1.0, np.array([1.38, 2.05], complex), np.array([0.1, 0.08]))
    assert float(np.max(np.abs(np.abs(T.forward(S, pol)['r']) - 1))) < 1e-17


def test_thinfilm_and_coatings_modes():
    th = np.radians([10.0, 30.0, 50.0])
    S = T.Samples(0.55, th, 1.2, 1.52, np.array([1.38, 2.05 + 0.1j]), np.array([0.1, 0.08]))
    cs = T.cos_snell(S.n0, S.nsub, S.sin0, S.C)
    for pol in (T.POL_S, T.POL_P):
        a, b = T.forward(S, pol, T.THINFILM), T.forward(S, pol)
        assert np.max(np.abs(a['r'] / b['r'] - 1)) < 1e-18
        ratio = S.cos0 / cs if pol == T.POL_P else 1
        assert np.max(np.abs(a['t'] / b['t'] / ratio - 1)) < 1e-18


# ---- mpmath ---------------------------------------------------------------------------------------------------------
MP_CASES = {'gap': ([1.38, 1.0], [0.1, 4.0], 1.7, 1.7), 'ag2um': ([1.46, 0.05 + 3.9j], [0.08, 2.0], 1.52, 1.0),
            'absorb': ([1.38, 1.5 + 0.2j, 2.05], [0.1, 0.05, 0.08], 1.52, 1.0)}
MP_W, MP_TH = np.linspace(0.45, 0.7, 4)[:, None], np.radians([0.0, 30.0, 60.0])[None, :]


def mp_rt(mp, n, d, sub, amb, w, th, pol):
    """r, t, R of one sample at the working precision (the coatings admittance form)"""
    s0, c0 = mp.sin(th), mp.cos(th)

    def cos_snell(n):
        s = amb / n * s0
        c = mp.sqrt(1 - s * s)
        return -c if mp.im(s) == 0 and mp.re(s) > 1 else c

    adm = lambda n, c: n / c if pol == T.POL_P else n * c
    cs = cos_snell(sub)
    v0, v1 = mp.mpc(1), adm(sub, cs)
    for k in range(len(n) - 1, -1, -1):
        c = cos_snell(n[k])
        b, e = 2 * mp.pi * n[k] * d[k] * c / w, adm(n[k], c)
        v0, v1 = mp.cos(b) * v0 - 1j * mp.sin(b) / e * v1, -1j * e * mp.sin(b) * v0 + mp.cos(b) * v1
    e0 = adm(amb, c0)
    r, t = (e0 * v0 - v1) / (e0 * v0 + v1), 2 * e0 / (e0 * v0 + v1)
    return r, t, abs(r) ** 2, mp.re(adm(sub, cs)) / mp.re(e0) * abs(t) ** 2


@pytest.mark.parametrize('name', MP_CASES)
@pytest.mark.parametrize('pol', (T.POL_S, T.POL_P))
def test_sweep_and_tangents_against_mpmath(name, pol):
    mpmath = pytest.importorskip('mpmath')
    mp = mpmath.mp
    mp.dps = 50
    n, d, sub, amb = MP_CASES[name]
    S = T.Samples(MP_W, MP_TH, amb, sub, np.asarray(n, complex), np.asarray(d, float))
    f = T.forward(S, pol)
    N = len(n)
    cR = np.ones(len(S), LDBL)
    _, gR, mR = T.functional(S, pol, (cR, None, None, None), kinds=3)
    _, gT, mT = T.functional(S, pol, (None, cR, None, None), kinds=3)
    w, th = np.broadcast_arrays(MP_W, MP_TH)
    h = mp.mpf('1e-18')
    for i, (wi, ti) in enumerate(zip(w.ravel(), th.ravel())):
        args = [mp.mpc(complex(x)) for x in n], [mp.mpf(float(x)) for x in d], mp.mpc(sub), mp.mpc(amb)
        r, t, R, Tt = mp_rt(mp, *args, mp.mpf(float(wi)), mp.mpf(float(ti)), pol)
        for got, want in ((f['r'][i], r), (f['t'][i], t)):
            err = abs(mp.mpc(complex(np.complex128(got))) + mp.mpc(complex(np.complex128(got - np.complex128(got))))
                      - want) / abs(want)
            # about 100 long-double ulps: the gap's |Im beta| reaches 77
            assert err < 3e-17, (name, pol, i, float(err))
        for p in range(2 * N):
            plus, minus = [list(a) for a in args[:2]], [list(a) for a in args[:2]]
            j = p % N
            if p < N:
                plus[1][j] += h
                minus[1][j] -= h
            else:
                plus[0][j] += h
                minus[0][j] -= h
            rp = mp_rt(mp, plus[0], plus[1], *args[2:], mp.mpf(float(wi)), mp.mpf(float(ti)), pol)
            rm = mp_rt(mp, minus[0], minus[1], *args[2:], mp.mpf(float(wi)), mp.mpf(float(ti)), pol)
            for g, m, q in ((gR, mR, 2), (gT, mT, 3)):
                fd = (rp[q] - rm[q]) / (2 * h)
                if float(m[p, i]) < 1e-25:
                    # an opaque or evanescent layer's far side: below what 50 digits resolve over h
                    assert abs(float(g[p, i])) < 1e-25 and abs(fd) < 1e-25
                    continue
                err = abs(float(g[p, i]) - fd) / float(m[p, i])
                assert err < 1e-15, (name, pol, i, p, q, float(err))


# ---- the committed fixtures -----------------------------------------------------------------------------------------
def test_thinfilm_fixtures():
    g = load_golden('thinfilm.npz')
    bad = {}
    for sname, (n, d, sub, amb) in O.stacks().items():
        tab = resolve(n, O.GRID_WVL)
        w = O.GRID_WVL if len(n) else np.ones(())
        for pol in O.POLS:
            ip = T.POL_P if pol == 'p' else T.POL_S
            S = T.Samples(w, O.GRID_THETA, amb, sub, tab, np.asarray(d, float))
            f, k, sh = T.forward(S, ip), f'{sname}_{pol}', S.shape
            figs = {q: rel(f[q].reshape(sh), g[f'{k}_{q}']) for q in ('r', 't', 'R', 'T')}
            figs.update({q: rel(f[q].reshape((-1,) + sh), g[f'{k}_{q}']) for q in ('E', 'H')})
            figs['A'] = rel(f['A'].reshape((-1,) + sh), g[f'{k}_A'], 1.0)
            for seed, kw in (O.seeds(k, sh, S.N).items() if S.N else ()):
                sd = [None if x not in kw else np.asarray(kw[x]).reshape(kw[x].shape[:kw[x].ndim - len(sh)] + (-1,))
                      for x in ('dR', 'dT', 'dA', 'dEsq')]
                gs = T.stack_grad(S, ip, 3, sd)[0].sum(-1)
                figs[f'gth_{seed}'] = rel(gs[:S.N], g[f'{k}_gth_{seed}'], 1.0) / 100
                figs[f'gix_{seed}'] = rel(gs[S.N:], g[f'{k}_gix_{seed}'], 1.0) / 100
            bad.update({f'{k}_{q}': v for q, v in figs.items() if not v < 1e-12})
    for name, (idx, th, wv, pol, sub, aoi, amb) in O.ml_cases().items():
        idx, th = np.asarray(idx, complex), np.asarray(th, float)
        aoi = np.asarray(aoi, float)
        if idx.ndim > 1 and aoi.size > 1:
            aoi = aoi.reshape(idx.shape[1:])
        S = T.Samples(wv, aoi, amb, sub, idx, th, theta_scale=np.pi / 180)
        f = T.forward(S, T.POL_P if pol == 'p' else T.POL_S, T.THINFILM)
        for q in 'rt':
            ref = g[f'{name}_{q}']
            v = rel(f[q].reshape(ref.shape), ref)
            if name.startswith('ml_gap'):
                v = float(np.max(np.abs(f[q].reshape(ref.shape).astype(complex) - ref) / np.abs(ref))) / 100
            if not v < 1e-12:
                bad[f'{name}_{q}'] = v
    assert not bad, bad


def test_coating_design_fixtures():
    g = load_golden('coating_design.npz')
    quant = {'R': (T.Q_R, {}), 'T': (T.Q_T, {}), 'A0': (T.Q_ABS, dict(b0=0)), 'Am1': (T.Q_ABS, dict(b0=-1)),
             'E1': (T.Q_ESQ, dict(b0=1)), 'Em1': (T.Q_ESQ, dict(b0=-1)), 'Pall': (T.Q_PEAK, dict(blist=None)),
             'Pdup': (T.Q_PEAK, dict(blist=[0, -1, 1, 1])), 'Ptie': (T.Q_PEAK, dict(blist=[1, 1])),
             'L0': (T.Q_LAYER, dict(b0=0, b1=1)), 'Lm1': (T.Q_LAYER, dict(b0=-1, b1=0))}
    pols = {'s': T.POL_S, 'p': T.POL_P, 'avg': T.POL_AVG}
    bad, seen = {}, 0
    for sname, (n, d, sub, amb) in D.stacks().items():
        N = len(n)
        for gname, (wvl, theta, target, weight) in D.grids().items():
            if gname != 'mesh' and sname != 'qw':
                continue
            S = T.Samples(wvl, theta, amb, sub, resolve(n, np.asarray(wvl, float)), np.asarray(d, float))
            for pol in D.POLS:
                for tname, (q, kw) in quant.items():
                    kw = {k: (v % (N if q == T.Q_ABS else N + 1) if isinstance(v, int) else v) for k, v in kw.items()}
                    if q == T.Q_PEAK:
                        kw['blist'] = list(range(N + 1)) if kw['blist'] is None else [b % (N + 1) for b in kw['blist']]
                    k = f'{sname}_{gname}_{pol}_{tname}'
                    m = T.merit(S, q, pols[pol], target, weight, kinds=3, **kw)
                    gs = m['der'].sum(-1)
                    figs = {'value': rel(m['val'].sum(), g[k + '_value']), 'res': rel(m['resid'], g[k + '_res']),
                            'gth': rel(gs[:N], g[k + '_gth'], 1.0) / 100, 'gix': rel(gs[N:], g[k + '_gix'], 1.0) / 100}
                    seen += 4
                    bad.update({f'{k}_{f}': v for f, v in figs.items() if not v < 1e-12})
        wvl, theta, target, weight = D.grids()['mesh']
        S = T.Samples(wvl, theta, amb, sub, resolve(n, np.asarray(wvl, float)), np.asarray(d, float))
        Z = np.concatenate([[0.0], np.cumsum(np.asarray(d, float))])
        zpart, zl = T.depth_runs(Z, D.depths(type('st', (), {'thicknesses': np.asarray(d, float)})), N)
        for pol in D.POLS:
            for qn, q in (('R', T.Q_R), ('T', T.Q_T)):
                for nname, nm in (('c', 1.38), ('d', O.cauchy)):
                    nn = nm(np.asarray(wvl, float)) if callable(nm) else nm
                    k = f'needle_{sname}_{pol}_{qn}_{nname}'
                    v = rel(T.needle(S, q, pols[pol], target, weight, nn, zpart, zl)[0].sum(-1), g[k], 1.0) / 100
                    seen += 1
                    if not v < 1e-12:
                        bad[k] = v
    assert seen == sum(1 for k in g if not k.endswith(('_gth_value', '_gix_value')))
    assert not bad, bad


# ---- defect models --------------------------------------------------------------------------------------------------
def grad_fig(name, pol, kinds, which, defect=None):
    """the fp64 model's seeded gradient over the long-double reference's majorant"""
    from test_gpu_thinfilm_vs_fp64 import seeds_of
    S, M = samples(name), samples(name, model=True)
    sd = seeds_of(S, which, 1)
    c, m = T.stack_grad(S, pol, kinds, sd)
    cm, _ = T.stack_grad(M, pol, kinds, sd, defect=defect)
    return T.over_majorant(cm.sum(-1), c.sum(-1), m.sum(-1))


def fwd_fig(name, pol, key, defect=None):
    S, M = samples(name), samples(name, model=True)
    with np.errstate(all='ignore'):
        f, fm = T.forward(S, pol), T.forward(M, pol, defect=defect)
    if key in ('E', 'H'):
        return T.rel_boundaries(fm[key], f[key]) if np.all(np.isfinite(fm[key])) else np.inf
    return T.rel_per_sample(fm[key], f[key]) if np.all(np.isfinite(fm[key])) else np.inf


def assert_defect(faithful, defective, ceil):
    assert faithful < ceil, (faithful, ceil)
    assert not defective < 10 * ceil, (defective, ceil)


def test_defect_beta_in_float32():
    assert_defect(fwd_fig('hl40', T.POL_S, 'r'), fwd_fig('hl40', T.POL_S, 'r', 'beta32'), CEIL['rt'])
    # float32 outputs: the 0.2 mm layer's float32 phase moves r by thousands of float32 ulps
    S, M = samples('thick'), samples('thick', model=True)
    f, fm = T.forward(S, T.POL_S), T.forward(M, T.POL_S, defect='beta32')
    ok = T.ulps32(T.forward(M, T.POL_S)['r'].astype(np.complex64), f['r'])
    assert_defect(ok, T.ulps32(fm['r'].astype(np.complex64), f['r']), CEIL['ulps'])


def test_defect_float32_field_stage():
    assert_defect(fwd_fig('ag2um', T.POL_S, 'E'), fwd_fig('ag2um', T.POL_S, 'E', 'stage32'), CEIL['field'])


@pytest.mark.parametrize('defect', ('esq_dropped', 'ce_single', 'seed_k'))
def test_defect_field_seed(defect):
    assert_defect(grad_fig('absorb', T.POL_P, 3, 'dEsq'), grad_fig('absorb', T.POL_P, 3, 'dEsq', defect),
                  CEIL['grad'])


@pytest.mark.parametrize('defect', ('no_dcos', 'im_for_re'))
def test_defect_index_gradient(defect):
    assert_defect(grad_fig('absorb', T.POL_S, 2, 'dR'), grad_fig('absorb', T.POL_S, 2, 'dR', defect), CEIL['grad'])


@pytest.mark.parametrize('defect', ('slot_zero', 'slot_twice', 'sweep2_overwrite'))
def test_defect_warp_slots(defect):
    """on 2 sweeps + 33 samples of an 8-SM grid: one slot, or the first pass of every slot, lost or doubled"""
    from test_gpu_thinfilm_vs_fp64 import seeds_of, sweep_samples
    _, S = sweep_samples(2 * sweep(8) + 33)
    c, m = T.stack_grad(S, T.POL_S, 3, seeds_of(S, 'all', 7))
    ref, maj = c.sum(-1), m.sum(-1)
    ok = T.over_majorant(T.slot_sum(c, 8, 256), ref, maj)
    assert_defect(ok, T.over_majorant(T.slot_sum(c, 8, 256, defect), ref, maj), CEIL['grad'])


def test_defect_expm1_with_sign_through_the_gap():
    assert_defect(fwd_fig('gap', T.POL_S, 't'), fwd_fig('gap', T.POL_S, 't', 'expm1_signed'), CEIL['rt'])


def test_defect_peak_seed_to_the_last_maximum():
    S, M = samples('zero'), samples('zero', model=True)
    fig = {}
    for defect in (None, 'peak_last'):
        r = T.merit(S, T.Q_PEAK, T.POL_S, 0.1, 1.0, kinds=3, blist=[1, 2])
        rm = T.merit(M, T.Q_PEAK, T.POL_S, 0.1, 1.0, kinds=3, blist=[1, 2], defect=defect)
        fig[defect] = T.over_majorant(rm['der'].sum(-1), r['der'].sum(-1), r['maj'].sum(-1))
    assert_defect(fig[None], fig['peak_last'], CEIL['merit'])
