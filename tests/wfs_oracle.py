"""The wavefront-sensing cases the engine is checked on (prysm/x/fibers.py, sri.py, pdi.py, psi.py) and the writer of
tests/golden/wfs*.npz.

    PYTHONDONTWRITEBYTECODE=1 python tests/wfs_oracle.py   (needs the unmodified reference: PRYSM_REFERENCE or oracle/_ref)

The fixtures are the REFERENCE's own outputs at precision 64, from the inputs `inputs()` builds with numpy.
`run(m, g, ...)` computes every case with the modules m.fibers, m.sri, m.pdi, m.psi (and m.Wavefront): the reference's
with numpy arrays, or the engine's (tests/test_gpu_wfs.py).  Every grid spacing is exactly representable in float32, so
a float32 run differs from the fixtures by the engine's rounding, not by the grids'.

Two departures from "call the reference as a user would", both to keep its outputs meaningful:
  - prysm.x.psi imports scikit-image's unwrapper at import time; this writer stubs that one module (unwrap_phase is not
    exercised).
  - the reference casts PSI weights to the frames' dtype, so uint16 frames wrap the negative weights modulo 2^16; the
    uint16 fixtures are the reference's sums of the same frames as int64, which is what the engine computes.
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (ROOT, os.path.join(ROOT, 'oracle')):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import reference  # noqa: E402

V_FIND = (0.5, 2.3, 3.0, 10, 20)
LP = dict(V=10, a=4.0, dx=0.375, shape=(64, 72))          # out to 3a along y
SMF = dict(V=2.3, a=0.975, dx=0.0625, n=96)
TPF = dict(n=64, dx=0.125, fib_n=64, fib_dx=0.09375, efl=16.0, wavelength=0.55, a=0.96)
SRI = dict(n=256, diameter=8.0, efl=16.0, epd=8.0, wavelength=0.55, fiber_a=0.96, fiber_samples=128)
PDI = dict(n=128, diameter=8.0, efl=80.0, epd=8.0, wavelength=0.55, test_arm_offset=16, test_arm_fov=16,
           test_arm_samples=64, pinhole_samples=32, grating_rulings=16)
PSI_SHAPE = (48, 64)
SCHEMES = ('zygo', 'schwider', 'hann7')
WIN = 64


def fftgrid(shape, dx):
    """make_xy_grid(shape, dx=dx) in fp64: fftrange(n) * dx per axis."""
    ny, nx = shape
    x = (np.arange(nx) - nx // 2) * dx
    y = (np.arange(ny) - ny // 2) * dx
    return np.meshgrid(x, y)


def polar(x, y):
    return np.hypot(x, y), np.arctan2(y, x)


def pupil_field(n, dx, seed):
    x, y = fftgrid((n, n), dx)
    r = np.hypot(x, y)
    R = n * dx / 2
    rng = np.random.default_rng(seed)
    c = rng.normal(0, 0.3, 4)
    phase = c[0] * (x / R) + c[1] * (y / R) + c[2] * (2 * (r / R) ** 2 - 1) + c[3] * (x * y) / R ** 2
    return (r <= R).astype(np.float64) * np.exp(1j * phase)


def inputs():
    """Every input array of the cases: fp64 / complex128 / uint16 host arrays."""
    g = {}
    x, y = fftgrid(LP['shape'], LP['dx'])
    g['lp_r'], g['lp_t'] = polar(x, y)
    a = LP['a']
    g['mm_E'] = np.exp(-(g['lp_r'] / (0.9 * a)) ** 2) * np.exp(1j * (0.4 * x / a + 0.3 * (g['lp_r'] / a) ** 2
                                                                      - 0.2 * x * y / a ** 2))
    x, y = fftgrid((SMF['n'], SMF['n']), SMF['dx'])
    g['smf_r'] = np.hypot(x, y)
    g['tpf_pupil'] = pupil_field(TPF['n'], TPF['dx'], 1)
    x, y = fftgrid((TPF['fib_n'], TPF['fib_n']), TPF['fib_dx'])
    g['tpf_r'] = np.hypot(x, y)
    g['sri_x'], g['sri_y'] = fftgrid((SRI['n'], SRI['n']), SRI['diameter'] / SRI['n'])
    g['sri_pupil'] = pupil_field(SRI['n'], SRI['diameter'] / SRI['n'], 2)
    g['pdi_x'], g['pdi_y'] = fftgrid((PDI['n'], PDI['n']), PDI['diameter'] / PDI['n'])
    g['pdi_pupil'] = pupil_field(PDI['n'], PDI['diameter'] / PDI['n'], 3)
    g['rect_x1'] = np.concatenate((np.linspace(-20, 20, 401), np.arange(-6, 7) * 2 * np.pi))
    g['rect_x2'] = np.arange(-40, 41) * 0.25
    yy, xx = np.mgrid[:PSI_SHAPE[0], :PSI_SHAPE[1]]
    g['psi_phase'] = 2.5 * ((xx - 30) / 32) ** 2 - 1.5 * ((yy - 20) / 24) + 0.8 * ((xx - 30) / 32) * ((yy - 20) / 24)
    return g


def psi_frames(phase, shifts):
    """Frames 2 + cos(phase + shift_k), float64, and the same rounded to counts of 1/1000 as uint16."""
    f = np.stack([2.0 + np.cos(phase + s) for s in np.asarray(shifts, dtype=np.float64)])
    return f, np.round(f * 1000).astype(np.uint16)


def schemes(psi):
    return {'zygo': psi.ZYGO_THIRTEEN_FRAME, 'schwider': psi.SCHWIDER, 'hann7': psi.design_scheme(7, window='hann')}


def window(a, w=WIN):
    cy, cx = a.shape[0] // 2, a.shape[1] // 2
    return a[cy - w // 2:cy + w // 2, cx - w // 2:cx + w // 2]


def _np(v):
    return np.asarray(getattr(v, 'data', v))


def run(m, g, to_numpy=_np, asarray=np.asarray, modes10=None, reference=False):
    """Every case through the modules of m.  modes10: the V = 10 mode dict compute_LP_modes and multimode_coupling use
    (default: m.fibers.find_all_modes(10)).  reference: the uint16 PSI frames go in as int64 (see the module doc)."""
    fib, sri, pdi, psi = m.fibers, m.sri, m.pdi, m.psi
    out = {}
    for V in V_FIND:
        fam = fib.find_all_modes(V)
        out[f'fam_V{V}_keys'] = np.asarray(list(fam), dtype=np.int64)
        for l, b in fam.items():
            out[f'fam_V{V}_{l}'] = np.asarray(b, dtype=np.float64)
        cnt = fib.find_all_modes(V, count_only=True)
        out[f'cnt_V{V}'] = np.asarray([[l, c] for l, c in cnt.items()], dtype=np.int64)
    md = modes10 if modes10 is not None else fib.find_all_modes(LP['V'])
    lp = fib.compute_LP_modes(LP['V'], md, LP['a'], asarray(g['lp_r']), asarray(g['lp_t']))
    flat = [mode for ms in lp.values() for mode in ms]
    out['lp_V10'] = np.stack([to_numpy(mode) for mode in flat])
    for b in (0.5, 0.3):
        out[f'smf_b{b}'] = to_numpy(fib.smf_mode_field(SMF['V'], SMF['a'], b, asarray(g['smf_r'])))
    E1, E2 = flat[2], asarray(g['mm_E'])
    out['moi_plain'] = np.float64(to_numpy(fib.mode_overlap_integral(E1, E2)))
    e1 = to_numpy(E1)
    out['moi_pre'] = np.float64(to_numpy(fib.mode_overlap_integral(E1, E2, E2conj=asarray(g['mm_E'].conj()),
                                                                   I1sum=float((e1 * e1).sum()),
                                                                   I2sum=float((np.abs(g['mm_E']) ** 2).sum()))))
    mm = fib.multimode_coupling(E2, lp)
    out['mmc_V10'] = np.asarray([float(to_numpy(v)) for vs in mm.values() for v in vs])

    # SRI: to_photonic_fiber_and_back on its own, then the instrument
    Efib = fib.smf_mode_field(2.3, TPF['a'], 0.5, asarray(g['tpf_r']))
    ef = to_numpy(Efib)
    wf = m.Wavefront(asarray(g['tpf_pupil']), TPF['wavelength'], TPF['dx'])
    nxt, at_fpm, emitted, coupling = sri.to_photonic_fiber_and_back(
        wf, TPF['efl'], Efib, TPF['fib_dx'], float((ef * ef).sum()), shift=(0.2, -0.1), phase_shift=0.7,
        return_more=True)
    out.update(tpf_next=to_numpy(nxt), tpf_at_fpm=to_numpy(at_fpm), tpf_emitted=to_numpy(emitted),
               tpf_coupling=np.float64(to_numpy(coupling)))
    inst = sri.SelfReferencedInterferometer(asarray(g['sri_x']), asarray(g['sri_y']), SRI['efl'], SRI['epd'],
                                            SRI['wavelength'], fiber_a=SRI['fiber_a'],
                                            fiber_samples=SRI['fiber_samples'])
    pupil = asarray(g['sri_pupil'])
    for tag, ps in (('0', 0), ('90', np.pi / 2)):
        out[f'sri_I_{tag}'] = to_numpy(inst.forward_model(pupil, phase_shift=ps))
    dbg = inst.forward_model(pupil, phase_shift=np.pi / 2, debug=True)['at_camera']
    out['sri_dbg_ref'] = window(to_numpy(dbg['ref']))
    out['sri_dbg_test'] = window(to_numpy(dbg['test']))

    # PS/PDI
    pupil = asarray(g['pdi_pupil'])
    px, py = asarray(g['pdi_x']), asarray(g['pdi_y'])
    common = {k: PDI[k] for k in ('test_arm_offset', 'test_arm_fov', 'test_arm_samples', 'pinhole_samples',
                                  'grating_rulings')}
    for gt in ('sin_amp', 'ronchi'):
        for ax in ('x', 'y'):
            inst = pdi.PSPDI(px, py, PDI['efl'], PDI['epd'], PDI['wavelength'], test_arm_transmissivity=0.7,
                             grating_type=gt, grating_axis=ax, **common)
            for tag, ps in (('0', 0), ('60', np.pi / 3)):
                out[f'pdi_{gt}_{ax}_{tag}'] = to_numpy(inst.forward_model(pupil, phase_shift=ps))
            out[f'pdi_{gt}_{ax}_test_beam'] = to_numpy(inst.test_beam)
            out[f'pdi_{gt}_{ax}_grating'] = to_numpy(inst.grating_func(px + 0.5 / 6))
    inst = pdi.PSPDI(px, py, PDI['efl'], PDI['epd'], PDI['wavelength'], test_arm_transmissivity=0.7,
                     grating_type='ronchi', grating_axis='x', **common)
    d = inst.forward_model(pupil, phase_shift=np.pi / 3, debug=True)
    out.update(pdi_dbg_total=to_numpy(d['total_field']), pdi_dbg_ref=to_numpy(d['at_camera']['ref']),
               pdi_dbg_test=to_numpy(d['at_camera']['test']), pdi_dbg_ref_at=to_numpy(d['at_fpm']['ref'][0]),
               pdi_dbg_ref_after=to_numpy(d['at_fpm']['ref'][1]), pdi_dbg_test_at=to_numpy(d['at_fpm']['test'][0]),
               pdi_dbg_test_after=to_numpy(d['at_fpm']['test'][1]))
    ratio, I1, I2 = pdi.evaluate_test_ref_arm_matching(d)
    out.update(pdi_ratio=np.float64(to_numpy(ratio)), pdi_ratio_I1=to_numpy(I1), pdi_ratio_I2=to_numpy(I2))
    out['rect1'] = to_numpy(pdi.rectangle_pulse(asarray(g['rect_x1'])))
    out['rect2'] = to_numpy(pdi.rectangle_pulse(asarray(g['rect_x2']), duty=0.3, amplitude=0.7, offset=0.2,
                                                period=0.5))

    # PSI
    for name, sch in schemes(psi).items():
        f64, u16 = psi_frames(g['psi_phase'], sch.shifts)
        for kind, frames in (('f64', f64), ('u16', u16)):
            if kind == 'u16' and name == 'hann7':
                continue
            if reference and kind == 'u16':
                frames = frames.astype(np.int64)
            fr = [asarray(f) for f in frames]
            num, den = psi.psi_accumulate(fr, sch)
            out[f'psi_{name}_{kind}_num'] = to_numpy(num)
            out[f'psi_{name}_{kind}_den'] = to_numpy(den)
            out[f'psi_{name}_{kind}_phase'] = to_numpy(psi.degroot_formalism_psi(fr, sch))
    return out


def reference_modules():
    """Call inside reference.loaded(also=('skimage',)): the skimage stub goes with the reference's modules."""
    if 'skimage.restoration._unwrap_2d' not in sys.modules:      # prysm.x.psi imports it; unwrap_phase is not used
        stub = types.ModuleType('skimage.restoration._unwrap_2d')
        stub.unwrap_2d = None
        for mod in (types.ModuleType('skimage'), types.ModuleType('skimage.restoration'), stub):
            sys.modules.setdefault(mod.__name__, mod)
    from prysm.conf import config
    from prysm.x import fibers, sri, pdi, psi
    from prysm.propagation import Wavefront
    config.precision = 64
    return types.SimpleNamespace(fibers=fibers, sri=sri, pdi=pdi, psi=psi, Wavefront=Wavefront)


def reference_outputs():
    import warnings
    with reference.loaded(also=('skimage',)), warnings.catch_warnings():
        m = reference_modules()
        warnings.simplefilter('ignore')
        return run(m, inputs(), reference=True)


def main():
    """Write tests/golden/wfs*.npz from the unmodified reference."""
    with reference.loaded():
        from make_golden import save      # imports the reference
        save('wfs.npz', reference_outputs())


if __name__ == '__main__':
    main()
