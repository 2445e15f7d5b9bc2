"""GPU: Shack-Hartmann sensing on the device (prysm_b200.shack_hartmann) -- the lenslet screen against the reference's
fixtures (tests/golden/shack_hartmann*.npz, written by tests/shack_hartmann_oracle.py), spot_centroids against its numpy
statement, the physics of a tilted beam, a calibrated modal loop with its CUDA-graph capture, the drop-in path with
the unmodified reference, and a Detector.expose frame straight into the slopes."""
import numpy as np
import pytest
import torch

from conftest import load_golden, within
from gpu_fixtures import pb  # noqa: F401
import reference
import shack_hartmann_oracle as O

pytestmark = pytest.mark.gpu

# Measured on an H100 SXM (700 W, 1980 MHz); each bound is the measured figure x 1.5.
# fp32 screens against the fp64 fixtures, away from the samples whose mask the float32 grid itself flips: 1.03e-5
# (circle_shift; the others 4.1e-6 to 7.0e-6), mostly the float32 grid's own rounding of rsq.
BOUND_SCREEN_32 = 1.55e-5
# relative error of the spot shift (slopes minus the unaberrated frame's), interior lenslets, tilts up to a quarter
# pitch: 0.142.  The subaperture truncates a shifted spot's sinc^2 tails, pulling its centre of gravity back.
BOUND_TILT = 0.21
# worst coefficient error of the calibrated Noll 2-11 loop at ~50 nm RMS: 0.340 nm
BOUND_LOOP_NM = 0.51


@pytest.fixture(scope='module')
def golden():
    return load_golden('shack_hartmann.npz')


def to_numpy(t):
    t = getattr(t, 'data', t)
    return t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)


def engine_screen(pb, name, dtype=np.float64, aperture=None):
    shape, dx, pitch, n, efl, ap, kw, shift = O.CASES[name]
    x, y = O.grid(shape, dx)
    aperture = aperture or getattr(pb.geometry, ap)
    return pb.shack_hartmann.shack_hartmann(pitch, n, efl, O.WAVELENGTH, x.astype(dtype), y.astype(dtype),
                                            aperture=aperture, aperture_kwargs=kw, shift=shift)


# ---- the screen ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', sorted(O.CASES))
def test_screen_matches_the_reference_fp64(pb, golden, name):
    """Every fixture to 1e-12; the masks are exact (a flipped sample would differ by O(1)), except that a rotated
    rectangle may flip samples whose reference signed distance is within a few ulp of 0."""
    got = to_numpy(engine_screen(pb, name))
    want = golden[f'screen_{name}']
    assert got.dtype == np.complex128 and got.shape == want.shape
    diff = np.abs(got - want)
    bad = diff > 1e-12
    if f'near_{name}' in golden:
        assert not np.any(bad & ~golden[f'near_{name}']), name
    else:
        assert not bad.any(), (name, float(diff.max()), int(bad.sum()))
    # the samples two to four lenslets claim carry the sum of their phases (where the mask is not a rounding decision)
    multi = golden[f'claims_{name}'] >= 2
    if f'near_{name}' in golden:
        multi &= ~golden[f'near_{name}']
    if multi.any():
        assert float(diff[multi].max()) <= 1e-12


@pytest.mark.parametrize('name', sorted(O.CASES))
def test_screen_fp32(pb, golden, name):
    """A float32 grid gives a complex64 screen.  Rounding the grid to float32 moves samples that sit on a lenslet edge
    across it (a phase jump of order one radian); those are found by the fp64 screen of the same rounded grid and left
    out.  Elsewhere the rounded grid moves the phase by ~1e-6 rad, which the bound includes."""
    shape, dx = O.CASES[name][:2]
    got = to_numpy(engine_screen(pb, name, np.float32))
    assert got.dtype == np.complex64
    want = golden[f'screen_{name}']
    xr, yr = (a.astype(np.float32).astype(np.float64) for a in O.grid(shape, dx))
    rounded_grid_64 = to_numpy(_screen_from(pb, name, xr, yr))
    flips = np.abs(rounded_grid_64 - want) > 1e-3
    assert flips.mean() < 0.5, (name, float(flips.mean()))
    within(f'sh_screen_fp32_{name}', np.abs(got - want)[~flips].max(), BOUND_SCREEN_32)


def _screen_from(pb, name, x, y):
    shape, dx, pitch, n, efl, ap, kw, shift = O.CASES[name]
    return pb.shack_hartmann.shack_hartmann(pitch, n, efl, O.WAVELENGTH, x, y, aperture=getattr(pb.geometry, ap),
                                            aperture_kwargs=kw, shift=shift)


def test_screen_is_one_launch(pb):
    shape, dx, pitch, n, efl, *_ = O.CASES['rect_edges']
    x, y = (pb.asdevice(a) for a in O.grid(shape, dx))
    pb.shack_hartmann.shack_hartmann(pitch, n, efl, O.WAVELENGTH, x, y)
    torch.cuda.synchronize()
    before = pb._ops.launch_count()
    pb.shack_hartmann.shack_hartmann(pitch, n, efl, O.WAVELENGTH, x, y)
    assert pb._ops.launch_count() - before == 1


def test_any_other_aperture_takes_the_device_loop(pb, golden):
    """A callable the engine does not recognise runs the reference's loop on device tensors, and agrees."""
    def square(width, x, y):
        return (x.abs() <= width) & (y.abs() <= width)

    got = to_numpy(engine_screen(pb, 'rect_edges', aperture=square))
    assert np.abs(got - golden['screen_rect_edges']).max() <= 1e-12

    def disc(radius, r):
        return r <= radius

    got = to_numpy(engine_screen(pb, 'circle_edges', aperture=disc))
    assert np.abs(got - golden['screen_circle_edges']).max() <= 1e-12


def test_unknown_rectangle_keyword_raises(pb):
    x, y = O.grid((64, 64), 0.01)
    with pytest.raises(TypeError):
        pb.shack_hartmann.shack_hartmann(0.32, 2, 20.0, 0.55, x, y, aperture_kwargs={'hieght': 0.1})


def test_free_space_intensity(pb, golden):
    shape, dx, pitch, n, efl = O.FREE_SPACE
    x, y = O.grid(shape, dx)
    screen = pb.shack_hartmann.shack_hartmann(pitch, n, efl, O.WAVELENGTH, x, y)
    wf = pb.Wavefront(O.pupil(shape, dx), O.WAVELENGTH, dx)
    got = to_numpy((wf * screen).free_space(dz=efl).intensity)
    want = golden['free_space_intensity']
    assert np.abs(got - want).max() / want.max() <= 1e-12


# ---- centroids -----------------------------------------------------------------------------------------------------
CENTROID_CASES = [((256, 256), 0.32, 8, False), ((250, 256), 0.3225, (5, 8), True), ((231, 231), 0.32, 7, True)]


def _frames(shape, F, dtype, pitch, n, shift, seed=3):
    """Random frames with subaperture (0, 1) dark: its displacement is NaN."""
    rng = np.random.default_rng(seed)
    f = rng.gamma(0.5, 300.0, (F, *shape))
    f[rng.random(f.shape) < 0.3] = 0
    x, y = O.grid(shape, 0.01)
    xc, yc = O.centres(pitch, n, shift)
    f[:, (np.abs(x - xc[1]) <= pitch / 2 + 0.01) & (np.abs(y - yc[0]) <= pitch / 2 + 0.01)] = 0
    if dtype in (np.uint16, np.int32):
        f = np.minimum(np.round(f), 65535)
    return f.astype(dtype)


@pytest.mark.parametrize('threshold', (0.0, 0.25))
@pytest.mark.parametrize('shape,pitch,n,shift', CENTROID_CASES)
def test_centroids_fp64_match_the_numpy_statement(pb, shape, pitch, n, shift, threshold):
    x, y = O.grid(shape, 0.01)
    frames = _frames(shape, 3, np.float64, pitch, n, shift)
    disp, flux = pb.shack_hartmann.spot_centroids(frames, x, y, pitch, n, shift=shift, threshold=threshold)
    assert disp.dtype == torch.float64 and flux.dtype == torch.float64
    want_d, want_f = O.centroids_numpy(frames, x, y, pitch, n, shift, threshold)
    got_d, got_f = to_numpy(disp), to_numpy(flux)
    assert got_d.shape == want_d.shape and got_f.shape == want_f.shape
    assert np.array_equal(np.isnan(got_d), np.isnan(want_d))
    assert np.isnan(want_d[:, :, 0, 1]).all()                   # the dark subaperture
    ok = ~np.isnan(want_d)
    assert np.abs(got_d[ok] - want_d[ok]).max() <= 1e-12
    assert np.abs(got_f - want_f).max() <= 1e-12 * np.abs(want_f).max()


@pytest.mark.parametrize('dtype', (np.uint16, np.int32, np.float32))
@pytest.mark.parametrize('threshold', (0.0, 0.25))
def test_centroids_of_integer_and_float32_frames(pb, dtype, threshold):
    """The sums are fp64 and rounded once: integer fluxes are exact, so the float32 output equals the statement's flux
    rounded to float32; the displacements agree to float32 rounding."""
    shape, pitch, n, shift = CENTROID_CASES[1]
    x, y = O.grid(shape, 0.01)
    frames = _frames(shape, 4, dtype, pitch, n, shift)
    disp, flux = pb.shack_hartmann.spot_centroids(frames, x, y, pitch, n, shift=shift, threshold=threshold)
    assert disp.dtype == torch.float32 and flux.dtype == torch.float32
    want_d, want_f = O.centroids_numpy(frames, x, y, pitch, n, shift, threshold)
    got_d = to_numpy(disp)
    if dtype != np.float32:
        assert np.array_equal(to_numpy(flux), want_f.astype(np.float32))
    else:
        assert np.abs(to_numpy(flux) - want_f).max() <= 1e-6 * np.abs(want_f).max()
    assert np.array_equal(np.isnan(got_d), np.isnan(want_d))
    ok = ~np.isnan(want_d)
    assert np.abs(got_d[ok] - want_d[ok]).max() <= 1e-6 * pitch


def test_centroid_stack_is_one_launch_and_bit_identical(pb):
    shape, pitch, n, shift = CENTROID_CASES[0]
    x, y = O.grid(shape, 0.01)
    frames = pb.asdevice(_frames(shape, 16, np.uint16, pitch, n, shift))
    plan = pb.shack_hartmann.CentroidPlan(x, y, pitch, n, shift)
    first = plan(frames, 0.1)
    torch.cuda.synchronize()
    before = pb._ops.launch_count()
    again = plan(frames, 0.1)
    assert pb._ops.launch_count() - before == 1
    for a, b in zip(first, again):
        assert torch.equal(torch.nan_to_num(a, nan=-1.0), torch.nan_to_num(b, nan=-1.0))
    one = plan(frames[5], 0.1)
    assert torch.equal(torch.nan_to_num(one[0]), torch.nan_to_num(first[0][5]))
    # a frame that starts off the vector alignment takes the one-column-per-thread kernel: same sums, same bits
    buf = pb.asdevice(np.concatenate(([0], to_numpy(frames[5]).ravel())).astype(np.uint16))
    odd = plan(buf[1:].view(frames.shape[1:]), 0.1)
    for a, b in zip(odd, (first[0][5], first[1][5])):
        assert torch.equal(torch.nan_to_num(a, nan=-1.0), torch.nan_to_num(b, nan=-1.0))


def test_empty_subapertures_are_nan(pb):
    x, y = O.grid((128, 128), 0.01)
    disp, flux = pb.shack_hartmann.spot_centroids(np.zeros((128, 128)), x, y, 0.32, 4, shift=True)
    assert torch.isnan(disp).all() and (flux == 0).all()


# ---- physics -------------------------------------------------------------------------------------------------------
# 512^2 at dx = 10 um.  The pitch is 31.95 samples so that no lenslet edge falls on a sample: an edge sample takes the
# phase of both lenslets (the reference's screen), a line defect that scatters light between neighbouring spots.
SENSOR = dict(pitch=0.3195, n=16, efl=20.0, wavelength=0.55, shift=True)
INNER = (slice(1, -1), slice(1, -1))     # the outer ring of lenslets also sees the unfocused light beyond the array


def _sensor(pb, **kw):
    x, y = pb.coordinates.make_xy_grid(512, dx=0.01)
    return pb.shack_hartmann.ShackHartmann(x=x, y=y, **{**SENSOR, **kw}), x, y


def test_tilt_moves_every_spot_by_efl_theta(pb):
    """A tilt theta moves each spot by efl theta, measured as the change of the slopes from the unaberrated frame (as
    calibrate measures them), so each subaperture's static offset cancels.  A plain centre of gravity over a
    subaperture still truncates the spot's sinc^2 tails, which pulls a shifted spot toward the lenslet centre: the
    bound is the measured relative error."""
    pb.config.precision = 64
    sh, x, y = _sensor(pb)
    flat = pb.Wavefront.from_amp_and_phase(torch.ones_like(x), torch.zeros_like(x), SENSOR['wavelength'], 0.01)
    s0 = to_numpy(sh.slopes(sh.forward_model(flat)))
    worst = 0.0
    for theta in (5e-4, 1e-3, 2e-3, 4e-3):              # up to a quarter pitch: efl theta = 0.08 mm
        for axis, g in ((0, x), (1, y)):
            wave = pb.Wavefront.from_amp_and_phase(torch.ones_like(x), g * (theta * 1e6), SENSOR['wavelength'], 0.01)
            d = to_numpy(sh.slopes(sh.forward_model(wave))) - s0
            worst = max(worst, float(np.abs(d[axis][INNER] - theta).max() / theta))
            assert np.abs(d[1 - axis][INNER]).max() < 0.01 * theta          # no cross-axis leak
    within('sh_tilt_relative_error', worst, BOUND_TILT)


def _noll_2_11(x, y, R):
    r, t = np.hypot(x, y) / R, np.arctan2(y, x)
    z = [2 * r * np.cos(t), 2 * r * np.sin(t), np.sqrt(3) * (2 * r ** 2 - 1), np.sqrt(6) * r ** 2 * np.sin(2 * t),
         np.sqrt(6) * r ** 2 * np.cos(2 * t), np.sqrt(8) * (3 * r ** 3 - 2 * r) * np.sin(t),
         np.sqrt(8) * (3 * r ** 3 - 2 * r) * np.cos(t), np.sqrt(8) * r ** 3 * np.sin(3 * t),
         np.sqrt(8) * r ** 3 * np.cos(3 * t), np.sqrt(5) * (6 * r ** 4 - 6 * r ** 2 + 1)]
    return np.stack(z), (r <= 1).astype(np.float64)


def test_calibrated_loop_and_its_graph(pb):
    """Calibrate on Noll 2-11 over a circular pupil, then reconstruct a random ~50 nm RMS combination; the loop
    forward_model -> slopes -> reconstruct captures into a CUDA graph whose replays are bit-identical to the eager
    call."""
    pb.config.precision = 64
    sh, x, y = _sensor(pb)
    xh, yh = to_numpy(x), to_numpy(y)
    modes, amp = _noll_2_11(xh, yh, 2.56)
    modes *= amp
    sh.calibrate(modes, 20.0, amp=amp)
    assert sh.valid.sum() > 100 and sh.reconstructor.shape == (10, 2 * sh.valid.sum())
    coefs = np.random.default_rng(5).normal(0, 50 / np.sqrt(10), 10)
    opd = pb.asdevice(np.tensordot(coefs, modes, axes=1))
    ampd = pb.asdevice(amp)

    def loop(o):
        w = pb.Wavefront.from_amp_and_phase(ampd, o, SENSOR['wavelength'], 0.01)
        return sh.reconstruct(sh.slopes(sh.forward_model(w)))

    eager = loop(opd)
    assert eager.shape == (10,) and eager.is_cuda
    within('sh_loop_worst_coefficient_nm', np.abs(to_numpy(eager) - coefs).max(), BOUND_LOOP_NM)
    g = pb.graphs.capture(loop, opd)
    try:
        a = g(opd).clone()
        b = g(opd).clone()
        assert torch.equal(a, b) and torch.equal(a, eager)
    finally:
        g.close()
    # a batch of slopes gives (F, K), and a NaN in a valid subaperture propagates
    s = sh.slopes(sh.forward_model(pb.Wavefront.from_amp_and_phase(ampd, opd, SENSOR['wavelength'], 0.01)))
    batch = torch.stack((s, s))
    j, i = np.argwhere(sh.valid)[0]
    batch[1, 0, j, i] = float('nan')
    out = sh.reconstruct(batch)
    assert out.shape == (2, 10) and torch.equal(out[0], eager) and torch.isnan(out[1]).all()
    # slopes the reconstructor was not built for are refused before anything is launched: the kernel's gather table
    # indexes (2, 16, 16) slope frames and cannot be bound-checked on the device
    other = pb.shack_hartmann.CentroidPlan(x, y, SENSOR['pitch'], 8, True)
    wrong = [s[:, :4, :4].contiguous(), s.reshape(-1), s[None, None], s.to(torch.float16), s.to(torch.int32),
             other(sh.forward_model(pb.Wavefront.from_amp_and_phase(ampd, opd, SENSOR['wavelength'], 0.01)))[0]]
    torch.cuda.synchronize()
    before = pb._ops.launch_count()
    for bad in wrong:
        with pytest.raises(ValueError):
            sh.reconstruct(bad)
    assert pb._ops.launch_count() == before
    with pytest.raises(ValueError):
        pb._ops.sh_reconstruct(s.reshape(1, -1), sh._idx, sh._ref, sh._R, (2, 16, 16))
    assert pb._ops.launch_count() == before


def test_exposed_frame_goes_straight_into_slopes(pb):
    """Detector.expose -> uint16 frame -> slopes, without leaving the device."""
    pb.config.precision = 64
    sh, x, y = _sensor(pb)
    I = sh.forward_model(pb.Wavefront.from_amp_and_phase(torch.ones_like(x), x * 1e3, SENSOR['wavelength'], 0.01))
    aerial = I.data * (2e4 / float(I.data.max()))
    det = pb.detector.Detector(dark_current=0, read_noise=2, bias=50, fwc=40000, conversion_gain=1, bits=16,
                               exposure_time=1)
    np.random.seed(1)
    frame = det.expose(aerial)
    assert frame.dtype == torch.uint16 and frame.is_cuda
    s = to_numpy(sh.slopes(frame))
    clean = to_numpy(sh.slopes(I))
    assert s.dtype == np.float32 and s.shape == (2, 16, 16)
    # the bias and the noise pull a plain centre of gravity toward the lenslet centre, but the tilt of 1e-3 rad reads
    # through on every interior spot
    flat = pb.Wavefront.from_amp_and_phase(torch.ones_like(x), torch.zeros_like(x), SENSOR['wavelength'], 0.01)
    clean0 = to_numpy(sh.slopes(sh.forward_model(flat)))
    assert np.abs((clean[0] - clean0[0])[INNER] / 1e-3 - 1).max() < BOUND_TILT
    assert np.all(s[0][INNER] > 0.2e-3)


# ---- drop-in -------------------------------------------------------------------------------------------------------
def test_dropin_reference_user_code(pb, golden):
    """The reference's own shack_hartmann and Wavefront code, run through set_backend_to_b200(), gives the fixtures
    (the reference's numpy results) within 1e-6."""
    if not reference.installed():
        pytest.skip('oracle/_ref is not installed')
    from prysm_b200 import mathops
    with reference.loaded():
        m = O.reference_modules()
        try:
            mathops.set_backend_to_b200()
            assert m.sh.shack_hartmann is pb.shack_hartmann.shack_hartmann
            import warnings
            with warnings.catch_warnings():
                warnings.simplefilter('ignore')
                mine = O.run(m, to_numpy=to_numpy)
        finally:
            mathops.set_backend_to_defaults()
            pb.config.precision = 64
    for k in sorted(golden):
        if k.startswith('near_'):
            continue
        got, want = np.asarray(mine[k]), golden[k]
        if k.startswith('screen_') and f'near_{k[7:]}' in golden:
            bad = np.abs(got - want) > 1e-6
            assert not np.any(bad & ~golden[f'near_{k[7:]}']), k
            continue
        err = float(np.abs(got - want).max() / max(np.abs(want).max(), 1e-300))
        assert err < 1e-6, (k, err)
