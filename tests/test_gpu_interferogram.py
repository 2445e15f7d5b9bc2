"""GPU: interferometric metrology on the device -- the NaN-aware statistics, masked least squares (lstsq, fit_plane,
fit_sphere, the remove_* methods, pvr), crop, spike_clip, the PSD and its windows, bandlimited_rms, TIS, the four
filters and slope -- against the reference's fixtures (tests/golden/interferogram*.npz, written by
tests/interferogram_oracle.py) at precision 64 and 32; repeatability and launch counts; the metrology chain behind
set_backend_to_b200() on a reference Interferogram holding a CUDA tensor; and pvr and psd at 2048^2 against the
reference run on the host."""
import warnings

import numpy as np
import pytest
import torch

from conftest import load_golden, within
from gpu_fixtures import pb, launches  # noqa: F401
import interferogram_oracle as O
import reference

pytestmark = pytest.mark.gpu

# max|engine - reference| / max|reference| over the finite samples of each key of a group, with the NaN pattern
# identical.  Measured on an H100 80GB HBM3 at a 700 W power limit; each bound is the measured figure x 1.5.  fp64:
# scalar 2.2e-15 (rect_mean), fit 1.1e-13 (circ_pvr), array 1.8e-16 (circ_slope_r), spectral 1.3e-13 (rect_filter_bp).
# fp32 (the fixture maps rounded once): scalar 1.6e-7 (circ_blr_wl), fit 1.8e-7 (circ_remove_power), array 1.2e-6
# (circ_slope_y), spectral 1.3e-6 (rect_filter_hp).
BOUNDS = {
    64: {'scalar': 3.4e-15, 'fit': 1.7e-13, 'array': 2.8e-16, 'spectral': 2.1e-13},
    32: {'scalar': 2.5e-7, 'fit': 2.8e-7, 'array': 1.8e-6, 'spectral': 2e-6},
}
# the chain behind the backend at 1000^2, fp64 against the host reference: 7.4e-15 (the radial PSD)
BOUND_DROPIN = 1.2e-14
# the re-bound free functions on CUDA tensors against the host reference, fp64: 3.6e-13 (designfilt2d 'br' at 255^2,
# the |FFT| of the windowed jinc; ideal_lpf_iir2d itself 1.7e-14)
BOUND_DISPATCH = 5.4e-13
# 2048^2 fp64 against the host reference: pvr 1.9e-14, psd 1.3e-15
BOUND_2048 = {'pvr': 3e-14, 'psd': 2e-15}
# the fp64 pvr coefficients of the circ map (37 Fringe terms, cond(A) = 4.5): 3.2e-15 relative, so squaring cond(A) in
# the normal equations costs nothing measurable here
BOUND_LSTSQ_PVR_FP64 = 4.8e-15


def group(key):
    if key.endswith(('_data', '_modes', '_in')):
        return None
    if any(t in key for t in ('_psd_', '_filter_', '_window', '_hann2d', '_designfilt', '_lpf')):
        return 'spectral'
    if any(t in key for t in ('remove_', 'fit_', 'lstsq', 'pvr')):
        return 'fit'
    if any(t in key for t in ('_crop', '_clip', '_slope', '_mask', '_recenter', '_latcal', '_strip', '_pad')):
        return 'array'
    return 'scalar'


@pytest.fixture(scope='module')
def golden():
    return load_golden('interferogram.npz')


def rel_err(got, want, key):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert got.shape == want.shape, (key, got.shape, want.shape)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), key
    if nan.all():
        return 0.0
    den = np.abs(want[~nan]).max()
    return float(np.abs(got[~nan] - want[~nan]).max() / (den if den > 0 else 1.0))


def engine_outputs(pb, prec):
    pb.config.precision = prec
    rdt = torch.float64 if prec == 64 else torch.float32
    try:
        return O.run(pb.interferogram, pb.util, pb.polynomials.lstsq,
                     prep=lambda a: torch.from_numpy(np.ascontiguousarray(a)).to('cuda', rdt))
    finally:
        pb.config.precision = 64


@pytest.mark.parametrize('prec', [64, 32])
def test_every_fixture(pb, golden, prec):
    got = engine_outputs(pb, prec)
    worst = {}
    for k, want in golden.items():
        g = group(k)
        if g is None:
            continue
        e = rel_err(got[k], want, k)
        if e >= worst.get(g, (-1, ''))[0]:
            worst[g] = (e, k)
    for g, (e, k) in worst.items():
        within(f'interferogram_{g}_fp{prec} ({k})', e, BOUNDS[prec][g])


def test_lstsq_and_pvr_against_the_condition_number(pb, golden):
    """The normal equations square cond(A): the fp64 pvr coefficient error, next to cond of its Fringe Zernike basis
    (pvr takes Fringe indices 1 to 37)."""
    from prysm_b200 import _ops
    d = torch.from_numpy(golden['circ_data']).cuda()
    i = pb.interferogram.Interferogram(d.clone(), dx=O.DX)
    r, t = i.r, i.t
    rn = r / O.PVR_RADIUS
    nms = [pb.polynomials.fringe_to_nm(j) for j in range(1, 38)]
    basis = _ops.zernike_seq(nms, rn, t, norm=False, polar=True)
    keep = (rn <= 1) & torch.isfinite(d)
    A = basis.reshape(len(nms), -1)[:, keep.reshape(-1)].T.cpu().numpy()
    data = torch.where(rn > 1, torch.nan, d)
    got = pb.polynomials.lstsq(basis, data)
    want = np.linalg.lstsq(A, d.reshape(-1)[keep.reshape(-1)].cpu().numpy(), rcond=None)[0]
    cond = np.linalg.cond(A)
    within(f'interferogram_pvr_coefs_fp64 (cond(A) = {cond:.1f})',
           np.abs(got - want).max() / np.abs(want).max(), BOUND_LSTSQ_PVR_FP64)


def test_repeat_calls_are_bit_identical(pb, golden):
    d = torch.from_numpy(golden['spiky_data']).cuda()
    a = pb.util.nan_stats(d)
    b = pb.util.nan_stats(d)
    assert np.array_equal(a, b)
    m = torch.from_numpy(golden['lstsq_modes']).cuda()
    ld = torch.from_numpy(golden['lstsq_data']).cuda()
    assert np.array_equal(pb.polynomials.lstsq(m, ld), pb.polynomials.lstsq(m, ld))
    f = torch.nan_to_num(d)
    assert torch.equal(pb.interferogram.psd(f, O.DX)[2], pb.interferogram.psd(f, O.DX)[2])


def test_launch_counts(pb, golden):
    d = torch.from_numpy(golden['circ_data']).cuda()
    _, n = launches(pb, lambda: pb.util.nan_stats(d))
    assert n == 2
    m = torch.from_numpy(golden['lstsq_modes']).cuda()
    ld = torch.from_numpy(golden['lstsq_data']).cuda()
    _, n = launches(pb, lambda: pb.polynomials.lstsq(m, ld))
    assert n == 1
    f = torch.nan_to_num(d)
    _, n1 = launches(pb, lambda: pb.interferogram.psd(f, O.DX, 'hann'))
    _, n2 = launches(pb, lambda: pb.interferogram.psd(f, O.DX, 'hann'))
    _, na = launches(pb, lambda: pb.interferogram.psd(f, O.DX))
    # the window prologue, the transform's launches, the epilogue; the automatic choice adds the corner test
    assert n1 == n2 and na == n1 + 1
    _, nt = launches(pb, lambda: pb._ops.fft2(f))
    assert n1 == nt + 2


def _chain(ifg, util_mod, I, data, dx):
    i = I(data, dx=dx)
    i.remove_piston().remove_tiptilt().remove_power().spike_clip(3).crop().fill(0)
    p = i.psd()
    rho, azavg = p.slices().azavg
    return {'data': i.data, 'azavg': azavg, 'rho': rho, 'blr': i.bandlimited_rms(flow=1.0, fhigh=5.0),
            'tis': i.total_integrated_scatter(10.6, np.array([0.0, 45.0])), 'pv': i.pv, 'rms': i.rms}


def _map(n, seed):
    rng = np.random.default_rng(seed)
    y, x = (np.mgrid[:n, :n] - n // 2) / (n // 2)
    d = 40 * x - 25 * y + 1.5 * (x * x + y * y) + rng.standard_normal((n, n))
    d[np.hypot(x, y) > 0.95] = np.nan
    d[rng.random((n, n)) < 0.0005] = 200.0
    return d


def test_metrology_chain_behind_the_backend(pb):
    if not reference.installed():
        pytest.skip('reference prysm not installed')
    d = _map(1000, 3)
    dx = 0.05
    with reference.loaded(), warnings.catch_warnings():
        warnings.simplefilter('ignore')
        from prysm.conf import config
        from prysm import interferogram as pifg, util as putil
        config.precision = 64
        want = _chain(pifg, putil, pifg.Interferogram, d.copy(), dx)
        try:
            pb.mathops.set_backend_to_b200()
            got = _chain(pifg, putil, pifg.Interferogram, torch.from_numpy(d.copy()).cuda(), dx)
            assert isinstance(got['data'], torch.Tensor) and got['data'].is_cuda
            # a host Interferogram behind the backend gives the reference's bits
            host = _chain(pifg, putil, pifg.Interferogram, d.copy(), dx)
        finally:
            pb.mathops.set_backend_to_defaults()
    for k, v in want.items():
        assert np.array_equal(np.asarray(host[k]), np.asarray(v), equal_nan=True), k
        g = got[k]
        g = g.detach().cpu().numpy() if isinstance(g, torch.Tensor) else g
        within(f'interferogram_dropin_fp64 {k}', rel_err(g, v, k), BOUND_DROPIN)


def _free_calls(pifg, putil, ppoly, golden, dev):
    """the re-bound free functions on the circ fixture, with every array argument put through dev"""
    d = golden['circ_data']
    f = np.nan_to_num(d)
    x, y = np.meshgrid((np.arange(255) - 127) * O.DX, (np.arange(255) - 127) * O.DX)
    ux = np.fft.fftshift(np.fft.fftfreq(255, O.DX))
    r = np.hypot(ux[None, :], ux[:, None])
    psd = pifg.psd(dev(f), O.DX)[2]
    return {'psd': psd, 'welch': pifg.make_window(dev(f), O.DX, 'welch'),
            'blr': pifg.bandlimited_rms(dev(r), psd, **O.BAND),
            'rms': putil.rms(dev(d)), 'std': pifg.std(dev(d)),
            'lstsq': ppoly.lstsq(dev(golden['lstsq_modes']), dev(golden['lstsq_data'])),
            'plane': pifg.fit_plane(dev(x), dev(y), dev(d)), 'sphere': pifg.fit_sphere(dev(d))[1],
            'welch_r': pifg.window_2d_welch(dev(r), 8), 'lpf': pifg.ideal_lpf_iir2d(dev(r), O.DX, 0.3),
            'H': pifg.designfilt2d(dev(r), O.DX, (0.8, 2.5), 'br')}


def test_free_functions_dispatch_behind_the_backend(pb, golden):
    """After the switch a CUDA tensor runs the engine and gives a CUDA tensor; numpy gives the reference's bits."""
    if not reference.installed():
        pytest.skip('reference prysm not installed')
    with reference.loaded(), warnings.catch_warnings():
        warnings.simplefilter('ignore')
        from prysm.conf import config
        from prysm import interferogram as pifg, util as putil, polynomials as ppoly
        config.precision = 64
        want = _free_calls(pifg, putil, ppoly, golden, lambda a: a)
        try:
            pb.mathops.set_backend_to_b200()
            got = _free_calls(pifg, putil, ppoly, golden, lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda())
            host = _free_calls(pifg, putil, ppoly, golden, lambda a: a)
        finally:
            pb.mathops.set_backend_to_defaults()
    errs = {}
    for k, v in want.items():
        np.testing.assert_array_equal(host[k], v, err_msg=k)
        g = got[k]
        if np.ndim(v) and k != 'lstsq':
            assert isinstance(g, torch.Tensor) and g.is_cuda, k
        errs[k] = rel_err(g.detach().cpu().numpy() if isinstance(g, torch.Tensor) else g, v, k)
    k = max(errs, key=errs.get)
    within(f'interferogram_dispatch_fp64 ({k})', errs[k], BOUND_DISPATCH)


def test_2048_pvr_and_psd_match_the_host_reference(pb):
    if not reference.installed():
        pytest.skip('reference prysm not installed')
    d = _map(2048, 9)
    dx = 0.025
    with reference.loaded(), warnings.catch_warnings():
        warnings.simplefilter('ignore')
        from prysm.conf import config
        from prysm import interferogram as pifg
        config.precision = 64
        want = {'pvr': pifg.Interferogram(d.copy(), dx=dx).pvr(),
                'psd': pifg.psd(np.nan_to_num(d), dx)[2]}
    i = pb.interferogram.Interferogram(torch.from_numpy(d.copy()).cuda(), dx=dx)
    got = {'pvr': i.pvr(), 'psd': pb.interferogram.psd(torch.from_numpy(np.nan_to_num(d)).cuda(), dx)[2].cpu().numpy()}
    for k in want:
        within(f'interferogram_2048_fp64 {k}', rel_err(got[k], want[k], k), BOUND_2048[k])
