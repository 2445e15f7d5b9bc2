"""GPU parity of the SURVEY.md 8(f) rows: adjoint twins of the elementwise steps and the otf reductions, and the
Lyot-coronagraph compositions (to_fpm_and_back, babinet, multi-resolution vortex) -- the CUDA path through the
C ABI against the reference's golden outputs (tests/golden/coronagraph.npz) and the CPU oracle.

Tolerances (relative L-inf): complex128 vs the reference's fp64 golden 1e-12; complex64 vs the fp64 oracle on the
same inputs 1e-6 per transform (compositions chain two transforms and a product: 3e-6).
"""
import numpy as np
import pytest
import torch

import prysm_oracle as O
from conftest import rel_linf, load_golden
from gpu_fixtures import pb, host  # noqa: F401

pytestmark = pytest.mark.gpu
HeNe = 0.6328
TOL64 = 1e-12


@pytest.fixture(scope='module')
def gold():
    return load_golden('coronagraph.npz')


def setprec(pb, prec):
    pb.config.precision = prec
    return (np.float64, np.complex128, TOL64) if prec == 64 else (np.float32, np.complex64, 2e-6)


# ------------------------------------------------------------------------------------------
# elementwise adjoints + otf adjoints
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize('prec', [64, 32])
def test_wavefront_adjoint_twins(pb, gold, prec):
    rdt, cdt, tol = setprec(pb, prec)
    g = gold
    WF = pb.propagation.Wavefront
    amp, opd = g['ea_amp'].astype(rdt), g['ea_opd'].astype(rdt)
    wf = WF.from_amp_and_phase(amp, opd, 0.55, 0.1)
    bar = WF(g['ea_bar'].astype(cdt), 0.55, 0.1)
    ibar = g['ea_ibar'].astype(rdt)
    out = wf.intensity_adjoint(ibar)
    assert isinstance(out, WF) and out.space == 'pupil' and out.dx == 0.1
    assert rel_linf(host(out.data), g['ea_intensity_adjoint']) < tol
    ph = wf.from_amp_and_phase_adjoint_phase(bar)
    assert ph.is_complex() and float(ph.real.abs().max()) == 0.0            # the reference's imaginary-valued result
    assert rel_linf(host(ph), g['ea_phase']) < tol
    assert rel_linf(host(wf.phase_screen_adjoint_phase(bar)), g['ea_phase']) < tol
    a1 = wf.from_amp_and_phase_adjoint_amp(bar)
    assert not a1.is_complex() and float(a1[2, 3]) == 0.0                   # zero amplitude -> zero gradient
    assert rel_linf(host(a1), g['ea_amp_nophase']) < tol
    assert rel_linf(host(wf.from_amp_and_phase_adjoint_amp(bar, phase=opd)), g['ea_amp_phase']) < tol
    x, y = np.meshgrid(O.fftrange(24) * 0.1, O.fftrange(18) * 0.1)
    got = WF.thin_lens_adjoint(250.0, 0.55, x.astype(rdt), y.astype(rdt), bar)
    assert got == pytest.approx(float(g['ea_lens_adjoint']), rel=1e-11 if prec == 64 else 2e-5)
    modes = g['ma_modes'].astype(rdt)
    got = pb.polynomials.sum_of_2d_modes_adjoint(modes, ibar)
    assert got.shape == (5,) and rel_linf(got, g['ma_out']) < tol
    gotc = pb.polynomials.sum_of_2d_modes_adjoint(modes, ph)                # complex gradient -> complex projection
    assert rel_linf(gotc, np.tensordot(g['ma_modes'], g['ea_phase'])) < tol
    # components
    f = wf.data
    assert rel_linf(host(wf.real.data), host(f).real) == 0 and rel_linf(host(wf.imag.data), host(f).imag) == 0
    assert np.abs(host(wf.phase.data) - np.angle(host(f))).max() < (1e-14 if prec == 64 else 1e-6)


@pytest.mark.parametrize('prec', [64, 32])
def test_otf_adjoints(pb, gold, prec):
    rdt, cdt, tol = setprec(pb, prec)
    g = gold
    otf = pb.otf
    psf = g['oa_psf'].astype(rdt)
    rb, cb = g['oa_rbar'].astype(rdt), g['oa_cbar'].astype(cdt)
    _, D = otf.mtf_from_psf(psf, 1.5, return_more=True)
    tol_ee = tol * 5 if prec == 32 else tol
    # the ptf adjoint divides by |D|^2: the fp32 rounding of the forward transform's small samples is amplified
    # (the reference at config.precision=32 shows the same spread against its own fp64 result)
    for fn, bar, key, amp in ((otf.mtf_from_psf_adjoint, rb, 'oa_mtf', 3), (otf.ptf_from_psf_adjoint, rb, 'oa_ptf', 3 if prec == 64 else 30),
                              (otf.otf_from_psf_adjoint, cb, 'oa_otf', 3)):
        a = fn(bar, data=D)
        b = fn(bar, psf=psf, dx=1.5)                 # recomputes the forward transform
        assert not a.is_complex()
        assert rel_linf(host(a), g[key]) < tol * amp, key
        assert rel_linf(host(b), g[key]) < tol * amp, key
    ee = otf.encircled_energy_adjoint([0.3, -1.2], dx=1.5, radius=[2.0, 7.5], data=D)
    assert rel_linf(host(ee), g['oa_ee']) < tol_ee
    ee1 = otf.encircled_energy_adjoint(0.3, psf=psf, dx=1.5, radius=2.0)
    ref1 = O.encircled_energy_adjoint(0.3, O.transform_psf(g['oa_psf'], 1.5)[0], 1.5, 2.0)
    assert rel_linf(host(ee1), ref1) < tol_ee
    with pytest.raises(ValueError):
        otf.encircled_energy_adjoint(0.3, radius=2.0, data=D)


# ------------------------------------------------------------------------------------------
# single-executor compositions
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize('prec', [64, 32])
@pytest.mark.parametrize('kind', ['mdft', 'czt'])
@pytest.mark.parametrize('fname', ['real', 'cplx'])
def test_to_fpm_and_back_and_babinet_vs_golden(pb, gold, prec, kind, fname):
    rdt, cdt, tol = setprec(pb, prec)
    tol = tol if prec == 64 else 3e-6
    g = gold
    P = pb.propagation
    pdx, fdx, wvl, efl = (float(v) for v in g['co_params'])
    w, gb = g['co_w'].astype(cdt), g['co_g'].astype(cdt)
    lyot = g['co_lyot'].astype(rdt)
    fpm = g[f'co_fpm_{fname}'].astype(rdt if fname == 'real' else cdt)
    ex = P.prepare_executor(pdx, w.shape, fdx, fpm.shape, wvl, efl, kind=kind)
    t = f'co_{kind}_{fname}_'
    nxt, at, after = P.to_fpm_and_back(w, fpm, ex, return_more=True)
    assert rel_linf(host(nxt), g[t + 'next']) < tol and rel_linf(host(at), g[t + 'at_fpm']) < tol
    assert rel_linf(host(after), g[t + 'after_fpm']) < tol
    assert rel_linf(host(P.to_fpm_and_back(w, fpm, ex)), g[t + 'next']) < tol
    Ea, Eb, it, fb = P.to_fpm_and_back_adjoint(gb, fpm, ex, return_more=True, return_fpm_grad=True, field_at_fpm=at)
    for u, nm in ((Ea, 'Eabar'), (Eb, 'Ebbar'), (it, 'inter'), (fb, 'fpm_bar')):
        assert rel_linf(host(u), g[t + nm]) < tol, nm
    assert fb.is_complex() == (fname == 'cplx')
    Ea2, fb2 = P.to_fpm_and_back_adjoint(gb, fpm, ex, return_fpm_grad=True, field_at_fpm=at)
    assert torch.equal(Ea2, Ea) and torch.equal(fb2, fb)
    assert torch.equal(P.to_fpm_and_back_adjoint(gb, fpm, ex), Ea)
    with pytest.raises(ValueError, match='requires field_at_fpm'):
        P.to_fpm_and_back_adjoint(gb, fpm, ex, return_fpm_grad=True)
    # babinet
    al, at2, af2, atl = P.babinet(w, lyot, fpm, ex, return_more=True)
    assert rel_linf(host(al), g[t + 'bab_after_lyot']) < tol and rel_linf(host(atl), g[t + 'bab_at_lyot']) < tol
    assert rel_linf(host(at2), g[t + 'bab_at_fpm']) < tol
    assert rel_linf(host(P.babinet(w, lyot, fpm, ex)), g[t + 'bab_after_lyot']) < tol       # fused subtract-and-stop
    assert rel_linf(host(P.babinet(w, None, fpm, ex)), g[t + 'bab_at_lyot']) < tol
    ab, fbb, lb = P.babinet_adjoint(gb, lyot, fpm, ex, field_at_fpm=at2, field_at_lyot=atl, return_fpm_grad=True,
                                    return_lyot_grad=True)
    for u, nm in ((ab, 'bab_abar'), (fbb, 'bab_fpm_bar'), (lb, 'bab_lyot_bar')):
        assert rel_linf(host(u), g[t + nm]) < tol, nm
    assert not lb.is_complex()
    assert torch.equal(P.babinet_adjoint(gb, lyot, fpm, ex), ab)
    with pytest.raises(ValueError, match='requires field_at_lyot'):
        P.babinet_adjoint(gb, lyot, fpm, ex, return_lyot_grad=True)


def test_wavefront_wrappers_and_adjoint_identity(pb):
    """reference tests/test_propagation.py:318-349: Wavefront-typed masks, <A x, y> == <x, A^H y>."""
    pb.config.precision = 64
    P = pb.propagation
    rng = np.random.default_rng(2468)
    x = rng.normal(size=(7, 9)) + 1j * rng.normal(size=(7, 9))
    fpm = rng.normal(size=(8, 11)) + 1j * rng.normal(size=(8, 11))
    y = rng.normal(size=x.shape) + 1j * rng.normal(size=x.shape)
    ex = P.prepare_executor(0.25, x.shape, 0.1, fpm.shape, HeNe, 10.0)
    lhs = np.vdot(host(P.to_fpm_and_back(x, fpm=fpm, executor=ex)), y)
    rhs = np.vdot(x, host(P.to_fpm_and_back_adjoint(y, fpm=fpm, executor=ex)))
    assert lhs == pytest.approx(rhs, abs=1e-12)
    wf = P.Wavefront(x, HeNe, 0.25)
    fpm_wf = P.Wavefront(fpm, HeNe, 0.1, 'psf')
    out, at, after = wf.to_fpm_and_back(fpm_wf, ex, return_more=True)
    assert out.space == 'pupil' and out.dx == 0.25 and at.space == 'psf' and at.dx == ex.focal_dx
    grad = out.to_fpm_and_back_adjoint(fpm=fpm_wf, executor=ex)
    assert grad.data.shape == wf.data.shape
    Ea, fb = out.to_fpm_and_back_adjoint(fpm_wf, ex, return_fpm_grad=True, field_at_fpm=at)
    assert Ea.space == 'pupil' and fb.space == 'psf' and fb.dx == ex.focal_dx
    lyot = P.Wavefront(rng.normal(size=x.shape), HeNe, 0.25)
    res = wf.babinet(lyot, fpm_wf, ex, return_more=True)
    assert [r.space for r in res] == ['pupil', 'psf', 'psf', 'pupil']
    ab, fbb, lb = res[0].babinet_adjoint(lyot, fpm_wf, ex, field_at_fpm=res[1], field_at_lyot=res[3],
                                         return_fpm_grad=True, return_lyot_grad=True)
    assert ab.space == 'pupil' and fbb.space == 'psf' and lb.space == 'pupil'
    # on-device inner product agrees with numpy's vdot (conjugates the second operand here: sum a*conj(b))
    d = pb._ops.dot(pb._ops.asdevice(y), pb._ops.asdevice(x))
    assert d == pytest.approx(np.vdot(x, y), rel=1e-13)


# ------------------------------------------------------------------------------------------
# multi-resolution vortex stack
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize('prec', [64, 32])
@pytest.mark.parametrize('kind', ['mdft', 'czt'])
def test_multiresolution_vs_golden(pb, gold, prec, kind):
    rdt, cdt, tol = setprec(pb, prec)
    g = gold
    P = pb.propagation
    pdx, fdx, wvl, efl = (float(v) for v in g['mr_params'])
    x, y = g['mr_x'].astype(cdt), g['mr_y'].astype(cdt)
    mex = P.prepare_multiresolution(pdx, 64, fdx, 32, wvl, efl, num_levels=3, fine_samples=32, kind=kind)
    assert len(mex) == 3
    wtol = 1e-14 if prec == 64 else 1e-6
    for k in range(3):
        assert rel_linf(host(mex.windows[k]), g[f'mr_win{k}']) < wtol
        assert rel_linf(host(mex.xf[k]), g[f'mr_xf{k}']) < wtol and rel_linf(host(mex.yf[k]), g[f'mr_yf{k}']) < wtol
    fpm = P.vortex_phase_mask(2)
    assert rel_linf(host(fpm(mex.xf[1], mex.yf[1])), g['mr_vortex1']) < (1e-14 if prec == 64 else 1e-6)
    t = f'mr_{kind}_'
    ctol = tol if prec == 64 else 4e-6
    out, at, after = P.to_fpm_and_back_multiresolution(x, fpm, mex, return_more=True)
    assert rel_linf(host(out), g[t + 'out']) < ctol
    assert rel_linf(host(P.to_fpm_and_back_multiresolution(x, fpm, mex)), g[t + 'out']) < ctol
    Ea, Ebs, its, fbs = P.to_fpm_and_back_multiresolution_adjoint(y, fpm, mex, return_more=True, return_fpm_grad=True,
                                                                  field_at_fpm=at)
    assert rel_linf(host(Ea), g[t + 'Eabar']) < ctol
    for k in range(3):
        assert rel_linf(host(at[k]), g[t + f'at{k}']) < ctol and rel_linf(host(after[k]), g[t + f'after{k}']) < ctol
        assert rel_linf(host(Ebs[k]), g[t + f'Ebbar{k}']) < ctol and rel_linf(host(its[k]), g[t + f'inter{k}']) < ctol
        assert rel_linf(host(fbs[k]), g[t + f'fpm_bar{k}']) < ctol
    Ea2, fbs2 = P.to_fpm_and_back_multiresolution_adjoint(y, fpm, mex, return_fpm_grad=True, field_at_fpm=at)
    assert torch.equal(Ea2, Ea) and len(fbs2) == 3
    # <A x, y> == <x, A^H y>, evaluated on the device (reference tests/test_propagation.py:544-556)
    lhs = pb._ops.dot(out, pb._ops.asdevice(y))          # sum out * conj(y)
    rhs = pb._ops.dot(pb._ops.asdevice(x), Ea)           # sum x * conj(A^H y)
    assert lhs == pytest.approx(rhs, rel=1e-10 if prec == 64 else 2e-5)
    # user callables receive device grids and may return device tensors
    out_u = P.to_fpm_and_back_multiresolution(x, lambda xf, yf: torch.exp(2j * torch.atan2(yf, xf)), mex)
    assert rel_linf(host(out_u), g[t + 'out']) < ctol * 2
    with pytest.raises(ValueError, match='requires field_at_fpm'):
        P.to_fpm_and_back_multiresolution_adjoint(y, fpm, mex, return_fpm_grad=True)


def test_multiresolution_wrappers_and_tuple_samples(pb):
    """reference tests/test_propagation.py:577-586, 625-645."""
    pb.config.precision = 64
    P = pb.propagation
    mex = P.prepare_multiresolution(pupil_dx=0.1, pupil_samples=32, focal_dx=2.0, focal_samples=(24, 40), wavelength=HeNe,
                                    efl=10.0, num_levels=2, fine_samples=16)
    assert tuple(mex.xf[0].shape) == (24, 40) and tuple(mex.xf[1].shape) == (16, 16)
    fpm = P.vortex_phase_mask(2)
    rng = np.random.default_rng(11)
    x = rng.random((32, 32)).astype(complex)
    assert tuple(P.to_fpm_and_back_multiresolution(x, fpm, mex).shape) == (32, 32)
    z = rng.standard_normal((16, 16)) + 1j * rng.standard_normal((16, 16))
    wf = P.Wavefront(z, HeNe, 0.25)
    mex = wf.prepare_multiresolution(efl=10.0, focal_dx=4.0, focal_samples=16, num_levels=2, fine_samples=12)
    out, at, after = wf.to_fpm_and_back_multiresolution(fpm, mex, return_more=True)
    assert out.dx == wf.dx and out.space == 'pupil'
    assert at[1].dx == mex.executors[1].focal_dx and at[1].space == 'psf'
    grad, bars = out.to_fpm_and_back_multiresolution_adjoint(fpm, mex, return_fpm_grad=True, field_at_fpm=at)
    assert tuple(grad.data.shape) == (16, 16) and grad.space == 'pupil' and len(bars) == 2
    with pytest.raises(ValueError):
        P.Wavefront(z, HeNe, 1.0, 'psf').prepare_multiresolution(10.0, 4.0, 16, 2)
    with pytest.raises(TypeError):
        P.vortex_phase_mask(2.5)
    P.vortex_phase_mask(np.int64(2))
    # unit-cell round trip is unitary (reference tests/test_propagation.py:566-574)
    n, pdx, efl = 64, 0.1, 50.0
    yy, xx = np.meshgrid(O.fftrange(n) * pdx, O.fftrange(n) * pdx, indexing='ij')
    pupil = (np.hypot(xx, yy) < 2.4).astype(complex)
    fdx, nf = P.unit_cell_focal_grid(pdx, 4.8, HeNe, efl)
    ex = P.prepare_executor(pdx, n, fdx, nf, HeNe, efl)
    rt = host(P.unfocus_dft(P.focus_dft(pupil, ex), ex))
    assert np.abs(rt - pupil).max() < 1e-12


def _grey_circle(radius, npup, dx, ss=16):
    g = (np.arange(npup * ss) - (npup * ss) // 2) * (dx / ss)
    xx, yy = np.meshgrid(g, g)
    fine = (np.hypot(xx, yy) < radius).astype(np.float32)
    return fine.reshape(npup, ss, npup, ss).mean(axis=(1, 3)).astype(np.float64)


@pytest.mark.parametrize('kind', ['mdft', 'czt'])
def test_vortex_dark_hole_below_1e12(pb, kind):
    """The reference's headline coronagraph test (tests/test_propagation.py:463-541): charge-2 vortex, 384^2 pupil,
    6 resolution levels, 0.8 R Lyot stop -> normalised intensity < 1e-12 in the 3-10 lambda/D dark hole (fp64)."""
    pb.config.precision = 64
    P = pb.propagation
    wvl, efl, pdx, npup, nd = HeNe, 100.0, 0.05, 384, 320
    Dap = nd * pdx
    lamD = efl / Dap * wvl
    period = wvl * efl / pdx
    pupil = _grey_circle(Dap / 2, npup, pdx).astype(complex)
    lyot = _grey_circle(0.8 * Dap / 2, npup, pdx)
    nf0 = 2 * nd
    mex = P.prepare_multiresolution(pdx, npup, period / nf0, nf0, wvl, efl, num_levels=6, fine_samples=256, kind=kind)
    nf, fdx = 256, lamD / 4
    final = P.prepare_executor(pdx, npup, fdx, nf, wvl, efl, kind=kind)
    ref_peak = float(P.Wavefront(P.focus_dft(pupil, final), wvl, fdx, 'psf').intensity.data.max())
    lyot_field = P.to_fpm_and_back_multiresolution(pupil, P.vortex_phase_mask(2), mex)
    after = P.Wavefront(lyot_field, wvl, pdx) * lyot
    I = host(P.Wavefront(P.focus_dft(after.data, final), wvl, fdx, 'psf').intensity.data) / ref_peak
    fx = np.arange(-(nf // 2), nf // 2) * fdx
    XF, YF = np.meshgrid(fx, fx)
    rad = np.hypot(XF, YF) / lamD
    assert I[(rad > 3) & (rad < 10)].max() < 1e-12


@pytest.mark.parametrize('shape', [((256, 256), (256, 256)), ((384, 256), (128, 640))])
def test_tensor_core_mdft_adjoint_and_round_trip(pb, shape):
    """complex64 MDFT adjoint on the wgmma tensor cores (the swapped-basis plan) against the fp64 oracle, and the composition
    through it."""
    pb.config.precision = 32
    P = pb.propagation
    (ny, nx), (my, mx) = shape
    rng = np.random.default_rng(ny + mx)
    a = (rng.standard_normal((ny, nx)) + 1j * rng.standard_normal((ny, nx))).astype(np.complex64)
    g = (rng.standard_normal((my, mx)) + 1j * rng.standard_normal((my, mx))).astype(np.complex64)
    fpm = rng.random((my, mx)).astype(np.float32)
    ex = P.prepare_executor(0.05, (ny, nx), 1.1, (my, mx), HeNe, 80.0, kind='mdft')
    assert ex._tc is not None and ex._tc_adj is not None
    exo = O.prepare_executor(0.05, (ny, nx), 1.1, (my, mx), HeNe, 80.0, kind='mdft')
    assert rel_linf(host(ex.adjoint(g)), exo.adjoint(g.astype(np.complex128))) < 1e-6
    assert rel_linf(host(ex(a)), exo(a.astype(np.complex128))) < 1e-6
    ref = O.to_fpm_and_back(a.astype(np.complex128), fpm.astype(np.float64), exo)
    assert rel_linf(host(P.to_fpm_and_back(a, fpm, ex)), ref) < 3e-6
    pb.config.precision = 64


@pytest.mark.parametrize('prec', [64, 32])
def test_measured_fpm_resampling(pb, gold, prec):
    """prepare_measured_fpm at order=1 against the reference (scipy.ndimage.map_coordinates) and inside the
    multi-resolution stack."""
    rdt, cdt, tol = setprec(pb, prec)
    g = gold
    P = pb.propagation
    mm, qx, qy = g['mf_map'].astype(cdt), g['mf_qx'].astype(rdt), g['mf_qy'].astype(rdt)
    # fp32 coordinates move the sample points by ~1e-6 of a pixel: compare at 1e-5 of the map's scale
    ftol = 1e-12 if prec == 64 else 2e-5
    assert rel_linf(host(P.prepare_measured_fpm(mm, 0.4, center=(0.3, -0.2), charge=2)(qx, qy)), g['mf_vortex']) < ftol
    assert rel_linf(host(P.prepare_measured_fpm(mm, 0.4, center=(0.3, -0.2), fill=0.25)(qx, qy)), g['mf_scalar']) < ftol
    assert rel_linf(host(P.prepare_measured_fpm(mm, 0.4)(qx, qy)), g['mf_default']) < ftol
    with pytest.raises(NotImplementedError):
        P.prepare_measured_fpm(mm, 0.4, order=3)
    # reference tests/test_propagation.py:648-676: exact on its own grid, ideal vortex beyond, scalar fill
    x, y = O.make_xy_grid(129, dx=0.4)
    meas = np.exp(1j * 2 * np.arctan2(y, x))
    f = P.prepare_measured_fpm(meas.astype(cdt), 0.4, charge=2)
    assert np.abs(host(f(x.astype(rdt), y.astype(rdt))) - meas).max() < (1e-12 if prec == 64 else 2e-5)
    far = np.full((1, 1), 1e5, dtype=rdt)
    assert np.abs(host(f(far, far)) - np.exp(1j * 2 * np.arctan2(1e5, 1e5))).max() < (1e-12 if prec == 64 else 1e-6)
    assert complex(host(P.prepare_measured_fpm(np.ones((65, 65), dtype=cdt), 1.0, fill=0.0)(np.full((1, 1), 1e3, dtype=rdt),
                                                                                             np.full((1, 1), 1e3, dtype=rdt)))[0, 0]) == 0
    # a measured copy of the ideal vortex drives the multi-resolution stack to the ideal-mask result where it is sampled
    pb.config.precision = 64
    mex = P.prepare_multiresolution(0.1, 64, 2.0, 32, HeNe, 10.0, num_levels=2, fine_samples=32)
    xm, ym = O.make_xy_grid(1025, dx=0.05)
    measured = P.prepare_measured_fpm(np.exp(1j * 2 * np.arctan2(ym, xm)), 0.05, charge=2)
    rng = np.random.default_rng(3)
    w = rng.standard_normal((64, 64)) + 1j * rng.standard_normal((64, 64))
    a = host(P.to_fpm_and_back_multiresolution(w, measured, mex))
    b = host(P.to_fpm_and_back_multiresolution(w, P.vortex_phase_mask(2), mex))
    assert rel_linf(a, b) < 1e-10         # the level grids fall on samples of the 0.05 um map: interpolation is exact
    mo = O.prepare_multiresolution(0.1, 64, 2.0, 32, HeNe, 10.0, num_levels=2, fine_samples=32)
    ref = O.to_fpm_and_back_multiresolution(w, O.prepare_measured_fpm(np.exp(1j * 2 * np.arctan2(ym, xm)), 0.05, charge=2), mo)
    assert rel_linf(a, ref) < 1e-11
