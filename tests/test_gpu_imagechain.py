"""GPU parity of the SURVEY.md 8(f) rank-4 row -- image-chain consumers of the path's FFTs (conv,
apply_transfer_functions, fourier_resample) -- against the reference's golden outputs (tests/golden/imagechain.npz)
and the CPU oracle.  Tolerances (relative L-inf): fp64 1e-12 vs the reference's fp64 golden; fp32 2e-6 vs the same
(two transforms and a product)."""
import numpy as np
import pytest
import torch

import prysm_oracle as O
from conftest import rel_linf, load_golden
from gpu_fixtures import pb, host  # noqa: F401

pytestmark = pytest.mark.gpu
ZOOMS = (0.5, 2, (2, 1.5))


@pytest.fixture(scope='module')
def gold():
    return load_golden('imagechain.npz')


def setprec(pb, prec):
    pb.config.precision = prec
    return (np.float64, np.complex128, 1e-12) if prec == 64 else (np.float32, np.complex64, 2e-6)


@pytest.mark.parametrize('prec', [64, 32])
def test_conv(pb, gold, prec):
    rdt, cdt, tol = setprec(pb, prec)
    g = gold
    conv = pb.convolution.conv
    out = conv(g['obj'].astype(rdt), g['psf'].astype(rdt))                 # packed: one forward, one inverse transform
    assert not out.is_complex() and rel_linf(host(out), g['conv_real']) < tol
    outc = conv(g['obj_c'].astype(cdt), g['psf'].astype(rdt))
    assert outc.is_complex() and rel_linf(host(outc), g['conv_cplx']) < tol
    assert rel_linf(host(conv(g['odd_obj'].astype(rdt), g['odd_psf'].astype(rdt))), g['conv_odd']) < tol
    obj = np.arange(25, dtype=rdt).reshape(5, 5)                           # reference tests/test_convolution.py:10-17, 50-58
    d = np.zeros_like(obj)
    d[2, 2] = 1
    assert np.allclose(host(conv(obj, d)), obj, atol=1e-12 if prec == 64 else 1e-5)
    objc = (np.arange(25).reshape(5, 5) * (1 + 1j)).astype(cdt)
    assert np.allclose(host(conv(objc, d.astype(cdt))), objc, atol=1e-12 if prec == 64 else 1e-5)
    with pytest.raises(ValueError):
        conv(obj, np.zeros((4, 5), dtype=rdt))


def test_conv_packed_at_size(pb):
    """1024^2 real x real (tuned FFT engine) against the oracle."""
    pb.config.precision = 32
    rng = np.random.default_rng(8)
    o = rng.random((1024, 1024)).astype(np.float32)
    h = np.exp(-((np.indices((1024, 1024)) - 512) ** 2).sum(axis=0) / 50.0).astype(np.float32)
    h /= h.sum()
    ref = O.conv(o.astype(np.float64), h.astype(np.float64))
    assert rel_linf(host(pb.convolution.conv(o, h)), ref) < 1e-6


@pytest.mark.parametrize('prec', [64, 32])
@pytest.mark.parametrize('shift', [False, True])
def test_apply_transfer_functions(pb, gold, prec, shift):
    rdt, cdt, tol = setprec(pb, prec)
    g = gold
    s = int(shift)
    atf = pb.convolution.apply_transfer_functions
    ob, obc = g['obj'].astype(rdt), g['obj_c'].astype(cdt)
    tf1, tf2 = g['tf1'].astype(rdt), g['tf2'].astype(cdt)
    out = atf(ob, 0.5, [tf1, tf2], shift=shift)
    assert not out.is_complex() and rel_linf(host(out), g[f'atf_shift{s}']) < tol
    outc = atf(obc, 0.5, [tf1], shift=shift)
    assert outc.is_complex() and rel_linf(host(outc), g[f'atf_c_shift{s}']) < tol
    seen = {}

    def gaussian(fx, fy, fr, ft):
        seen.update(fx=fx, fy=fy, fr=fr, ft=ft)
        return torch.exp(-(fr / 0.7) ** 2)
    out = atf(ob, 0.5, [gaussian], shift=shift)
    assert tuple(seen['fx'].shape) == (1, 30) and tuple(seen['fy'].shape) == (36, 1) and tuple(seen['fr'].shape) == (36, 30)
    gtol = 1e-14 if prec == 64 else 1e-6
    for nm in ('fx', 'fy', 'fr'):
        assert rel_linf(host(seen[nm]), g[f'grid_{nm}_shift{s}']) < gtol
    # ft wraps at +-pi on the negative real axis in either precision: compare on the unit circle
    assert np.abs(np.exp(1j * host(seen['ft'])) - np.exp(1j * g[f'grid_ft_shift{s}'])).max() < (1e-14 if prec == 64 else 1e-6)
    assert rel_linf(host(out), g[f'atf_callable_shift{s}']) < tol
    ident = atf(np.arange(16, dtype=rdt).reshape(4, 4), 1, [np.ones((4, 4), dtype=rdt)], shift=shift)
    assert np.allclose(host(ident), np.arange(16).reshape(4, 4), atol=1e-12 if prec == 64 else 1e-5)

    def not_a_tf(wavelength):
        return 1
    with pytest.raises(ValueError):
        atf(ob, 1, [not_a_tf])


@pytest.mark.parametrize('prec', [64, 32])
def test_fourier_resample(pb, gold, prec):
    rdt, cdt, tol = setprec(pb, prec)
    g = gold
    fr = pb.fttools.fourier_resample
    for i, z in enumerate(ZOOMS):
        out = fr(g['obj'].astype(rdt), z)
        assert tuple(out.shape) == g[f'resample{i}'].shape and not out.is_complex()
        assert rel_linf(host(out), g[f'resample{i}']) < tol
    outc = fr(g['obj_c'].astype(cdt), 2)
    assert outc.is_complex() and rel_linf(host(outc), g['resample_c']) < tol
    a = torch.ones((8, 8), device='cuda', dtype=torch.float64 if prec == 64 else torch.float32)
    assert fr(a, 1) is a
    assert np.allclose(host(fr(a, (2, 3))), 1, atol=1e-12 if prec == 64 else 1e-5)      # tests/test_fttools.py:229-235
    with pytest.raises(ValueError):
        fr(a, -1)
    with pytest.raises(ValueError):
        fr(a, 0.01)


@pytest.mark.parametrize('prec', [64, 32])
def test_detector_sampling(pb, gold, prec):
    rdt, cdt, tol = setprec(pb, prec)
    g = gold
    D = pb.detector
    ob = g['obj'].astype(rdt)
    tol = 1e-14 if prec == 64 else 1e-6
    for i, fac in enumerate((2, 3, (2, 3), (4, 6))):
        assert rel_linf(host(D.bindown(ob, fac, 'avg')), g[f'bin{i}_avg']) < tol
        assert rel_linf(host(D.bindown(ob, fac, 'sum')), g[f'bin{i}_sum']) < tol
        assert rel_linf(host(D.tile(g['psf'][:6, :5].astype(rdt), fac, 'sum')), g[f'tile{i}_sum']) < tol
    fx, fy = O.transfer_function_grids(g['obj'].shape, 2.0, False, rdt)[:2]
    assert rel_linf(host(D.pixel_ft(fx, fy, 3.0, 2.5)), g['pixel_ft']) < tol * 5
    assert rel_linf(host(D.olpf_ft(fx, fy, 0.7, 0.9)), g['olpf_ft']) < tol * 5
    with pytest.raises(ValueError, match='mode must be average or sum'):
        D.bindown(ob, 2, 'median')
    with pytest.raises(ValueError):
        D.bindown(ob, 5)                                   # 36 x 30 is not a multiple of 5 on both axes
    with pytest.raises(ValueError, match='scaling must be average or sum'):
        D.tile(ob, 2, 'max')
    # the image chain end to end on the device: blur by pixel and OLPF transfer functions, bin to detector pixels
    blurred = pb.convolution.apply_transfer_functions(ob, 2.0, [lambda fx, fy: D.pixel_ft(fx, fy, 3.0, 2.5),
                                                                 lambda fx, fy: D.olpf_ft(fx, fy, 0.7, 0.9)])
    ref = O.apply_transfer_functions(g['obj'], [g['pixel_ft'], g['olpf_ft']])
    assert rel_linf(host(D.bindown(blurred, (2, 3))), O.bindown(ref, (2, 3))) < (1e-12 if prec == 64 else 3e-6)
