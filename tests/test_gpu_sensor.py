"""GPU: image sensors on the device (prysm_b200.detector, prysm_b200.bayer).  Every bayer function and the deterministic
detector cases against the reference's fixtures (tests/golden/sensor*.npz, written by tests/sensor_oracle.py); the
random part of Detector.expose against exact distributions (chi-square, moments), for independence and for
reproducibility under numpy's global seed; and the reference's own user code through the drop-in switch."""
import math

import numpy as np
import pytest
import torch
from scipy import stats

from conftest import load_golden, rel_linf
from gpu_fixtures import pb  # noqa: F401
import reference
import sensor_oracle as O

pytestmark = pytest.mark.gpu

ROUNDED = ('malvar_', 'superres_', 'wbpre_1', 'wbpost_1')      # fp64 sums or descaled gains: 1e-12, not bit-exact


@pytest.fixture(scope='module')
def golden():
    return load_golden('sensor.npz')


def to_numpy(t):
    return t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)


def compare(mine, golden, bound, keys=None):
    bad = {}
    for k in sorted(keys or golden):
        got, want = mine[k], golden[k]
        if want.dtype.kind == 'U':
            if str(got) != str(want):
                bad[k] = f'{got} != {want}'
            continue
        got = np.asarray(got)
        if got.shape != want.shape:
            bad[k] = f'shape {got.shape} != {want.shape}'
        elif k.startswith(ROUNDED) or bound > 1e-12:
            err = rel_linf(got, want) if want.size else 0.0
            if not err <= bound:
                bad[k] = f'{err:.2e}'
        elif got.dtype != want.dtype or not np.array_equal(got, want):
            bad[k] = f'{got.dtype} vs {want.dtype}, {np.count_nonzero(got != want)} differ'
    return bad


def test_every_fixture_at_fp64_from_device_tensors(pb, golden):
    pb.config.precision = 64
    np.random.seed(0)
    mine = O.run(pb.detector, pb.bayer, O.inputs(), to_numpy=to_numpy, asarray=pb.asdevice)
    assert sorted(mine) == sorted(golden)
    bad = compare(mine, golden, 1e-12)
    assert not bad, bad


def test_every_fixture_at_fp64_from_numpy_arrays(pb, golden):
    """The same cases with host arrays in: the white balances then scale the caller's numpy array in place."""
    pb.config.precision = 64
    mine = O.run(pb.detector, pb.bayer, O.inputs(), to_numpy=to_numpy)
    bad = compare(mine, golden, 1e-12)
    assert not bad, bad


def test_demosaic_and_superresolution_at_fp32(pb, golden):
    pb.config.precision = 32
    try:
        g = {k: (v.astype(np.float32) if v.dtype == np.float64 else v) for k, v in O.inputs().items()}
        mine = O.run(pb.detector, pb.bayer, g, to_numpy=to_numpy, asarray=pb.asdevice)
    finally:
        pb.config.precision = 64
    keys = [k for k in golden if k.startswith(('malvar_', 'superres_')) and golden[k].dtype.kind == 'f']
    for k in keys:
        assert np.asarray(mine[k]).dtype == np.float32, k
    bad = compare(mine, golden, 1e-6, keys)
    assert not bad, bad


def test_white_balance_scales_a_device_tensor_where_it_is(pb, golden):
    g = O.inputs()
    for safe in (False, True):
        t = pb.asdevice(g['mosaic_f64_64x96'])
        ptr = t.data_ptr()
        pb.bayer.wb_prescale(t, *O.WB_GAINS, cfa='BGGR', safe=safe, saturation=(900, 1000, 1000, 800))
        assert t.data_ptr() == ptr
        np.testing.assert_allclose(to_numpy(t), golden[f'wbpre_{int(safe)}_BGGR_64x96'], rtol=1e-12, atol=0)
        t = pb.asdevice(g['rgb_64x96'])
        pb.bayer.wb_postscale(t, 1.7, 1.0, 1.4, safe=safe, saturation=(1000, 900, 1000))
        np.testing.assert_allclose(to_numpy(t), golden[f'wbpost_{int(safe)}_64x96'], rtol=1e-12, atol=0)


def test_decomposite_returns_views(pb):
    img = pb.asdevice(np.arange(48.0).reshape(6, 8))
    r, g1, g2, b = pb.bayer.decomposite_bayer(img, 'rggb')
    assert r.data_ptr() == img.data_ptr() and g1.data_ptr() == img.data_ptr() + 8
    img[1, 1] = -1
    assert float(b[0, 0]) == -1


def test_one_launch_per_bayer_call(pb):
    from prysm_b200 import _ops
    img = pb.asdevice(np.random.default_rng(1).random((64, 96)))
    planes = [pb.asdevice(np.random.default_rng(i).random((64, 96))) for i in range(4)]
    for fn in (lambda: pb.bayer.demosaic_malvar(img), lambda: pb.bayer.composite_bayer(*planes),
               lambda: pb.bayer.recomposite_bayer(*planes), lambda: pb.bayer.demosaic_deinterlace(img)):
        before = _ops.launch_count()
        fn()
        assert _ops.launch_count() - before == 1


# ---- Detector.expose -------------------------------------------------------------------------------------------------
def test_expose_dtype_by_bits(pb):
    for bits, dt in ((8, torch.uint8), (12, torch.uint16), (16, torch.uint16), (32, torch.uint32)):
        img = pb.detector.Detector(0, 0, 10, 60_000, 2, bits, 1).expose(np.zeros((3, 4)))
        assert img.dtype == dt and img.shape == (3, 4)
        assert np.array_equal(to_numpy(img).astype(np.int64), np.full((3, 4), 5))


def test_expose_errors_carry_the_reference_messages(pb):
    D = pb.detector.Detector
    with pytest.raises(ValueError, match="numpy's random functionality is inadequate for > 32 unsigned bits"):
        D(0, 0, 0, 1e9, 1, 33, 1).expose(np.ones((2, 3)))
    for bad in (-1.0, np.nan):
        a = np.ones((4, 5))
        a[2, 3] = bad
        with pytest.raises(ValueError, match=r'^lam < 0 or lam is NaN$'):
            D(0, 0, 0, 1e9, 1, 12, 1).expose(a)
    with pytest.raises(ValueError, match='^lam value too large$'):
        D(0, 0, 0, 1e9, 1, 12, 1).expose(np.full((2, 2), 1e19))
    with pytest.raises(IndexError, match='out of bounds for axis 0 with size 10'):
        D(0, 0, 100, 1e9, 1, 12, 1, lut=np.arange(10, dtype=np.uint16)).expose(np.zeros((2, 2)))


def test_expose_refuses_graph_capture(pb):
    d = pb.detector.Detector(0, 1, 10, 60_000, 2, 12, 1)
    img = pb.asdevice(np.ones((8, 8)))
    d.expose(img)
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        with pytest.raises(RuntimeError, match='CUDA graph'):
            with torch.cuda.graph(g, stream=s):
                d.expose(img)


def counts_detector(pb, **kw):
    """dark 0, read 0, bias 0, gain 1, 32 bits: DN = k"""
    p = dict(dark_current=0, read_noise=0, bias=0, fwc=1e18, conversion_gain=1, bits=32, exposure_time=1)
    p.update(kw)
    return pb.detector.Detector(**p)


def draw(pb, det, lam, shape=(500, 200), frames=10, dtype=np.float64):
    return to_numpy(det.expose(np.full(shape, lam, dtype=dtype), frames=frames)).astype(np.int64).ravel()


def chi2_p(samples, pmf_support, pmf):
    """p-value of a chi-square test of integer samples against pmf over pmf_support (bins of expected count >= 5; the
    tails beyond merged into one bin each)."""
    n = samples.size
    exp = pmf * n
    keep = exp >= 5
    lo, hi = pmf_support[keep][0], pmf_support[keep][-1]
    sel = (pmf_support >= lo) & (pmf_support <= hi)
    obs_mid = np.bincount(samples[(samples >= lo) & (samples <= hi)] - lo, minlength=hi - lo + 1)
    e_mid = np.zeros(hi - lo + 1)
    e_mid[pmf_support[sel] - lo] = exp[sel]
    obs = np.concatenate([[np.count_nonzero(samples < lo)], obs_mid, [np.count_nonzero(samples > hi)]])
    e = np.concatenate([[exp[pmf_support < lo].sum()], e_mid, [exp[pmf_support > hi].sum()]])
    m = e >= 5
    obs, e = obs[m], e[m]
    e = e * obs.sum() / e.sum()
    chi = ((obs - e) ** 2 / e).sum()
    return stats.chi2.sf(chi, m.sum() - 1)


@pytest.mark.parametrize('lam', (1e-3, 0.5, 3, 9.99, 10, 10.01, 37, 250, 1e4, 2e6))
def test_shot_noise_is_poisson(pb, lam):
    np.random.seed(int(lam * 1000) % 2 ** 31)
    k = draw(pb, counts_detector(pb), lam)
    n = k.size
    assert n == 10 ** 6
    lo = max(0, int(stats.poisson.ppf(1e-12, lam)) - 2)
    hi = int(stats.poisson.isf(1e-12, lam)) + 2
    support = np.arange(lo, hi + 1)
    p = chi2_p(k, support, stats.poisson.pmf(support, lam))
    assert p > 1e-6, (lam, p)
    assert abs(k.mean() - lam) < 6 * math.sqrt(lam / n), (lam, k.mean())
    assert abs(k.var() - lam) < 6 * math.sqrt((lam + 2 * lam * lam) / n), (lam, k.var())


def test_adc_path_gain_and_bias(pb):
    """gain 2.7, bias 100, no read noise: DN = trunc((k + 100) * (1 / 2.7)), k ~ Poisson(37)"""
    np.random.seed(5)
    dn = draw(pb, counts_detector(pb, bias=100, conversion_gain=2.7, bits=12), 37.0)
    ks = np.arange(0, 200)
    codes = np.floor((ks + 100.0) * (1 / 2.7)).astype(np.int64)
    pmf = np.bincount(codes, weights=stats.poisson.pmf(ks, 37.0))
    assert chi2_p(dn, np.arange(pmf.size), pmf) > 1e-6


def test_adc_path_read_noise(pb):
    """sigma 50, lam 0, bias 1000: DN = floor(1000 + 50 z)"""
    np.random.seed(6)
    dn = draw(pb, counts_detector(pb, bias=1000, read_noise=50, bits=16), 0.0)
    d = np.arange(600, 1401)
    pmf = stats.norm.cdf((d + 1 - 1000) / 50) - stats.norm.cdf((d - 1000) / 50)
    assert chi2_p(dn, d, pmf) > 1e-6


def pearson(a, b):
    return float(np.corrcoef(a.astype(np.float64).ravel(), b.astype(np.float64).ravel())[0, 1])


def test_noise_is_independent_across_pixels_frames_and_calls(pb):
    np.random.seed(7)
    d = counts_detector(pb, read_noise=3.0, bias=50)
    a = to_numpy(d.expose(np.full((400, 500), 37.0), frames=4)).astype(np.int64)
    b = to_numpy(d.expose(np.full((400, 500), 37.0), frames=4)).astype(np.int64)
    lim = lambda n: 5 / math.sqrt(n)                                       # noqa: E731
    assert abs(pearson(a[..., :-1], a[..., 1:])) < lim(a[..., 1:].size)
    assert abs(pearson(a[:-1], a[1:])) < lim(a[1:].size)
    assert abs(pearson(a, b)) < lim(a.size)


def test_expose_is_reproducible_under_numpy_seed(pb):
    d = pb.detector.Detector(2.0, 4.0, 100, 60_000, 1.5, 12, 0.5, prnu=np.linspace(0.9, 1.1, 48),
                             dcnu=np.ones((32, 1)))
    img = np.random.default_rng(3).random((32, 48)) * 3000
    np.random.seed(11)
    a1 = to_numpy(d.expose(img, frames=4))
    a2 = to_numpy(d.expose(img, frames=4))
    np.random.seed(11)
    b1 = to_numpy(d.expose(img, frames=4))
    np.random.seed(11)
    c = to_numpy(d.expose(img))
    np.random.seed(12)
    e = to_numpy(d.expose(img, frames=4))
    assert np.array_equal(a1, b1)
    assert not np.array_equal(a1, a2)
    assert np.array_equal(a1[0], c)
    assert not np.array_equal(a1, e)


def test_expose_lut_is_fused_and_matches_apply_lut(pb):
    lut = (np.sqrt(np.arange(4096) * 16.0)).astype(np.float32)
    d = pb.detector.Detector(0, 2.0, 20, 60_000, 1, 12, 1)
    dl = pb.detector.Detector(0, 2.0, 20, 60_000, 1, 12, 1, lut=lut)
    img = np.random.default_rng(4).random((64, 64)) * 3000
    np.random.seed(13)
    raw = d.expose(img, frames=3)
    np.random.seed(13)
    got = dl.expose(img, frames=3)
    assert got.dtype == torch.float32
    assert np.array_equal(to_numpy(got), to_numpy(pb.detector.apply_lut(raw, lut)))


# ---- drop-in ----------------------------------------------------------------------------------------------------------
def _with_reference(fn):
    if not reference.installed():
        pytest.skip('oracle/_ref is not installed')
    from prysm_b200 import mathops
    with reference.loaded():
        try:
            return fn()
        finally:
            mathops.set_backend_to_defaults()


def test_dropin_image_simulation_chain(pb):
    """The reference's Image Simulation chain (siemensstar -> conv -> bindown -> Detector.expose(frames=64)) through
    set_backend_to_b200() has the per-pixel mean and variance of the numpy backend's run."""
    def chain():
        from prysm.conf import config
        config.precision = 64
        from prysm import coordinates, objects, convolution, detector
        from prysm_b200 import mathops

        def run():
            x, y = coordinates.make_xy_grid(256, diameter=2)
            r, t = coordinates.cart_to_polar(x, y)
            star = objects.siemensstar(r, t, 32)
            psf = np.exp(-(np.asarray(r) / 0.02) ** 2)
            img = convolution.conv(star, psf / psf.sum())
            img = detector.bindown(img, 4)
            cam = detector.Detector(10, 4, 100, 20_000, 2.0, 12, 0.01)
            frames = cam.expose(np.asarray(to_numpy(img)) * 3e5, frames=64)
            return to_numpy(frames).astype(np.float64)
        np.random.seed(1)
        ref = run()
        mathops.set_backend_to_b200()
        assert detector.Detector is pb.detector.Detector
        np.random.seed(1)
        mine = run()
        return ref, mine
    ref, mine = _with_reference(chain)
    assert ref.shape == mine.shape == (64, 64, 64)
    m_ref, m_mine = ref.mean(0), mine.mean(0)
    v_ref, v_mine = ref.var(0, ddof=1), mine.var(0, ddof=1)
    se = np.sqrt((v_ref + v_mine) / 64 + 1e-12)
    assert np.all(np.abs(m_mine - m_ref) < 6 * se + 1e-9)
    assert abs(v_mine.mean() / v_ref.mean() - 1) < 0.05


def test_dropin_bayer_chain(pb, golden):
    """composite_bayer then demosaic_malvar, called through the reference's module after the switch, matches the
    reference's numpy result to 1e-6."""
    g = O.inputs()
    planes = [g[f'plane_{p}_64x96'] for p in ('r', 'g1', 'g2', 'b')]

    def chain():
        from prysm.conf import config
        config.precision = 64
        from prysm import bayer
        from prysm_b200 import mathops
        ref = bayer.demosaic_malvar(bayer.composite_bayer(*planes, cfa='bggr'), 'bggr')
        mathops.set_backend_to_b200()
        assert bayer.demosaic_malvar is pb.bayer.demosaic_malvar
        mine = to_numpy(bayer.demosaic_malvar(bayer.composite_bayer(*planes, cfa='bggr'), 'bggr'))
        return ref, mine
    ref, mine = _with_reference(chain)
    assert rel_linf(mine, ref) <= 1e-6
