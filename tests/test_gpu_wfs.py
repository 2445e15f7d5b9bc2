"""GPU: wavefront sensing on the device (prysm_b200.fibers, .sri, .pdi, .psi) against the reference's fixtures
(tests/golden/wfs*.npz, written by tests/wfs_oracle.py), the Bessel ratios against scipy, the determinism and graph
capture of the coupling reduction and of a whole SRI forward model, the launch count of a PSI reconstruction, and the
drop-in path executed against the unmodified reference."""
import types

import numpy as np
import pytest
import torch
from scipy import special

from conftest import load_golden, rel_linf, within
from gpu_fixtures import pb  # noqa: F401
import reference
import wfs_oracle as O

pytestmark = pytest.mark.gpu

BOUND = {32: 1e-6, 64: 1e-12}
# Camera intensities at fp32 are squared fields after two matrix DFTs per arm, so the transforms' ~5e-7 field error
# doubles.  Measured on an H100 (700 W, 1980 MHz): SRI 1.68e-6 (phase pi/2) and 1.44e-6 (phase 0), ronchi PS/PDI along x
# 1.05e-6, its weak test arm's intensity 1.28e-6.
BOUND_INTENSITY_32 = 3e-6
INTENSITIES = ('sri_I_', 'pdi_ronchi_x_0', 'pdi_ronchi_x_60', 'pdi_ratio_I2')
EXACT = ('pdi_ronchi_x_grating', 'pdi_ronchi_y_grating', 'rect1', 'rect2')


@pytest.fixture(scope='module')
def golden():
    return load_golden('wfs.npz')


def to_numpy(t):
    t = getattr(t, 'data', t)
    return t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)


def engine(pb):
    return types.SimpleNamespace(fibers=pb.fibers, sri=pb.sri, pdi=pb.pdi, psi=pb.psi, Wavefront=pb.Wavefront)


def modes10(golden):
    return {int(l): golden[f'fam_V10_{l}'] for l in golden['fam_V10_keys']}


def wrapped(a, b):
    """max |a - b| modulo 2 pi, so that a branch flip at +-pi is no error."""
    d = np.asarray(a, dtype=np.float64) - np.asarray(b, dtype=np.float64)
    return float(np.abs(np.angle(np.exp(1j * d))).max())


def compare(mine, golden, prec, tag):
    """Every fixture against the engine's outputs: returns {key: (error, bound)} of the failures."""
    bad = {}
    for k in sorted(golden):
        got, want = np.asarray(mine[k]), golden[k]
        assert got.shape == want.shape, k
        if k.startswith(('fam_', 'cnt_')):
            # find_all_modes returns b at config.precision: one float32 rounding at precision 32
            err, bound = float(np.abs(got - want).max()) if got.size else 0.0, (1e-12 if prec == 64 else 2 ** -23)
        elif k.startswith('psi_') and k.endswith('_phase'):
            err, bound = wrapped(got, want), 4 * BOUND[prec]
        elif k.startswith('psi_') and '_u16_' in k:
            assert got.dtype == want.dtype, k             # int64 sums (integer weights), float64 phase
            err, bound = float(np.abs(got - want).max()), 0.5
        elif k in EXACT:
            if prec == 64:
                err, bound = float(np.count_nonzero(got != want)), 0.5
            else:
                continue                                  # counted in test_grating_edges_at_fp32
        else:
            err, bound = rel_linf(got, want), BOUND[prec]
            if prec == 32 and k.startswith(INTENSITIES):
                bound = BOUND_INTENSITY_32
        if err < bound:
            within(f'wfs{prec}_{k}', err, bound)
        else:
            bad[k] = (err, bound)
    return bad


@pytest.mark.parametrize('prec', [32, 64])
def test_every_fixture(pb, golden, prec):
    pb.config.precision = prec
    rdt = np.float32 if prec == 32 else np.float64
    cdt = np.complex64 if prec == 32 else np.complex128

    def asarray(a):
        a = np.asarray(a)
        return pb.asdevice(a if a.dtype.kind in 'iu' else a.astype(cdt if np.iscomplexobj(a) else rdt))
    mine = O.run(engine(pb), O.inputs(), to_numpy=to_numpy, asarray=asarray, modes10=modes10(golden))
    assert sorted(mine) == sorted(golden)
    bad = compare(mine, golden, prec, prec)
    if bad:
        pytest.fail(' '.join(f'{k}: {e:.2e} (bound {b:.0e})' for k, (e, b) in sorted(bad.items())))


def test_grating_edges_at_fp32(pb, golden):
    """At fp32 the grid itself is rounded (the fixtures evaluate the fp64 grid), so a sample within one float32 ulp of
    a ronchi edge may land on the other side.  Count those flips: every one must sit within an ulp of an edge."""
    pb.config.precision = 32
    g = O.inputs()
    px = pb.asdevice(g['pdi_x'].astype(np.float32))
    period = O.PDI['epd'] / O.PDI['grating_rulings']
    inst = pb.pdi.PSPDI(px, px, O.PDI['efl'], O.PDI['epd'], O.PDI['wavelength'], grating_type='ronchi',
                        grating_rulings=O.PDI['grating_rulings'], test_arm_samples=8, pinhole_samples=8)
    got = to_numpy(inst.grating_func(px + 0.5 / 6))
    want = golden['pdi_ronchi_x_grating']
    x = (g['pdi_x'] + 0.5 / 6) % period
    flips = got != want
    near = np.minimum(np.abs(x - period / 2), np.minimum(x, period - x)) <= 2 * np.spacing(np.float32(8.0))
    assert np.all(near[flips]), f'{int(flips.sum())} flips, {int((flips & ~near).sum())} away from an edge'
    within('wfs32_ronchi_edge_flips', flips.sum(), flips.size * 0.02 + 1)


# Bessel ratios against scipy, relative to each mode's peak.  Measured on an H100 (700 W, 1980 MHz): K 6.6e-14 (order 40,
# W = 30); J 1.05e-13 for arguments up to 20 (order 1, U = 20) and 7.8e-12 up to 60 (order 5, U = 60).  The J error is
# that of CUDA's fp64 j0 / j1, whose absolute error grows with the argument, divided by a small J_l(U).
BOUND_K = 1e-13
BOUND_J = {0.5: 1.6e-13, 5.0: 1.6e-13, 20.0: 1.6e-13, 60.0: 1.2e-11}


def test_bessel_ratios_match_scipy(pb):
    """pb_lp_modes' ratios J_l(U rho) / J_l(U) (core) and K_l(W rho) / K_l(W) (cladding) on orders 0-40 and arguments
    1e-3-60 match scipy's jv / kv relative to each mode's peak magnitude (bounds above)."""
    from prysm_b200 import _ops
    from prysm_b200._capi import LP_RULE_LP, LP_NONE
    pb.config.precision = 64
    orders = (0, 1, 2, 3, 5, 8, 13, 20, 30, 40)
    worst = 0.0
    rho_j = torch.linspace(0, 1, 4001, dtype=torch.float64, device='cuda')
    for U in (0.5, 5.0, 20.0, 60.0):
        plan = np.array([[l, l, U, 1.0, LP_RULE_LP, LP_NONE] for l in orders])
        got = to_numpy(_ops.lp_modes(rho_j, None, 1.0, plan))
        x = to_numpy(rho_j) * U
        keep = x >= 1e-3
        for i, l in enumerate(orders):
            want = special.jv(l, x) / special.jv(l, U)
            err = np.abs(got[i][keep] - want[keep]).max() / np.abs(want[keep]).max()
            worst = max(worst, err)
            assert err < BOUND_J[U], (l, U, err)
    for W in (1e-3, 0.05, 0.5, 2.0, 10.0, 30.0):
        rho = torch.from_numpy(np.geomspace(1.0, 60.0 / W, 4001)).cuda()
        plan = np.array([[l, l, 1.0, W, LP_RULE_LP, LP_NONE] for l in orders])
        got = to_numpy(_ops.lp_modes(rho, None, 1.0 - 1e-15, plan))
        x = to_numpy(rho) * W
        for i, l in enumerate(orders):
            want = special.kve(l, x) / special.kve(l, W) * np.exp(W - x)
            err = np.abs(got[i] - want).max() / np.abs(want).max()
            within(f'wfs_bessel_k_{l}_{W}', err, BOUND_K)
    within('wfs_bessel_j_peak_relative', worst, max(BOUND_J.values()))


def test_overlap_is_deterministic_and_replays(pb, golden):
    """pb_overlap sums per-chunk partials in a fixed order: bit-identical across calls and across a graph replay."""
    from prysm_b200 import graphs
    pb.config.precision = 64
    g = O.inputs()
    modes = pb.fibers.compute_LP_modes(10, modes10(golden), O.LP['a'], g['lp_r'], g['lp_t'])
    E = pb.asdevice(g['mm_E'])

    def step(e):
        eta = pb.fibers.multimode_coupling(e, modes)
        return eta[0][0]._base if eta[0][0]._base is not None else torch.stack([v for vs in eta.values() for v in vs])
    a, b = step(E).clone(), step(E).clone()
    assert torch.equal(a, b)
    cap = graphs.capture(step, E)
    c = cap(E).clone()
    assert torch.equal(a, c)
    cap.close()


def test_sri_forward_model_plans_once_and_replays(pb, monkeypatch):
    """The SRI executor is built at construction: a second forward model builds no plan, and the whole forward model
    replays bit-identically from a CUDA graph."""
    from prysm_b200 import graphs, fttools
    pb.config.precision = 32
    g = O.inputs()
    inst = pb.sri.SelfReferencedInterferometer(pb.asdevice(g['sri_x'].astype(np.float32)),
                                               pb.asdevice(g['sri_y'].astype(np.float32)), O.SRI['efl'], O.SRI['epd'],
                                               O.SRI['wavelength'], fiber_a=O.SRI['fiber_a'],
                                               fiber_samples=O.SRI['fiber_samples'])
    pupil = pb.asdevice(g['sri_pupil'].astype(np.complex64))
    first = inst.forward_model(pupil, phase_shift=np.pi / 2).data.clone()

    def no_plan(*a, **k):
        raise AssertionError('forward_model built a plan')
    monkeypatch.setattr(pb.sri, 'prepare_executor', no_plan)
    monkeypatch.setattr(fttools.MDFT, '__init__', no_plan)
    second = inst.forward_model(pupil, phase_shift=np.pi / 2).data
    assert torch.equal(first, second)
    cap = graphs.capture(lambda w: inst.forward_model(w, phase_shift=np.pi / 2).data, pupil)
    assert torch.equal(cap(pupil).clone(), first)
    cap.close()
    pb.config.precision = 64


def test_degroot_is_one_launch(pb):
    from prysm_b200 import _ops
    pb.config.precision = 32
    g = O.inputs()
    f32, u16 = O.psi_frames(g['psi_phase'], pb.psi.ZYGO_THIRTEEN_FRAME.shifts)
    for frames in (f32.astype(np.float32), u16):
        fr = [pb.asdevice(f) for f in frames]
        torch.cuda.synchronize()
        n0 = _ops.launch_count()
        out = pb.psi.degroot_formalism_psi(fr, pb.psi.ZYGO_THIRTEEN_FRAME)
        assert _ops.launch_count() - n0 == 1
        assert out.dtype == (torch.float32 if frames.dtype == np.float32 else torch.float64)
    rd = [pb._richdata.RichData(f, 0.5, 0.6) for f in fr]
    out = pb.psi.degroot_formalism_psi(rd, pb.psi.ZYGO_THIRTEEN_FRAME)
    assert isinstance(out, pb._richdata.RichData) and out.dx == 0.5 and out.wavelength == 0.6
    pb.config.precision = 64


def test_dropin_reference_user_code(pb, golden):
    """The reference's own SRI, PS/PDI, PSI and multimode_coupling code, run through set_backend_to_b200(), gives the
    fixtures (the reference's numpy results) within 1e-6."""
    if not reference.installed():
        pytest.skip('oracle/_ref is not installed')
    from prysm_b200 import mathops
    with reference.loaded(also=('skimage',)):
        m = O.reference_modules()
        try:
            mathops.set_backend_to_b200()
            assert m.sri.SelfReferencedInterferometer is pb.sri.SelfReferencedInterferometer
            assert m.fibers.multimode_coupling is pb.fibers.multimode_coupling
            import warnings
            with warnings.catch_warnings():
                warnings.simplefilter('ignore')
                mine = O.run(m, O.inputs(), to_numpy=to_numpy)
        finally:
            mathops.set_backend_to_defaults()
    for k in ('fam_V10_keys',):
        assert np.array_equal(mine[k], golden[k])
    bad = {}
    for k in sorted(golden):
        if not k.startswith(('mmc', 'lp_', 'smf', 'moi', 'tpf', 'sri', 'pdi', 'rect', 'psi')):
            continue
        got, want = np.asarray(mine[k]), golden[k]
        err = wrapped(got, want) if k.endswith('_phase') else rel_linf(got, want)
        if err < 1e-6:
            within(f'wfs_dropin_{k}', err, 1e-6)
        else:
            bad[k] = err
    if bad:
        pytest.fail(' '.join(f'{k}: {v:.2e}' for k, v in sorted(bad.items())))
