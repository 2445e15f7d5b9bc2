"""Shack-Hartmann sensing on the device (reference prysm/x/shack_hartmann.py), from the lenslet screen to modal
coefficients.

`shack_hartmann` is the reference's function: the complex screen of a lenslet array, in the precision of x, in one
launch (pb_lenslet_screen).  The host does the integer work with numpy in the reference's own dtypes -- the lenslet
centres, each lenslet's window and, per grid column and row, the lenslets whose window covers it -- and the kernel sums
each sample's phase in the reference's order, so the fp64 screen is the reference's bit for bit, edges claimed by two
to four lenslets included.

The measurement side has no reference counterpart:
  - `spot_centroids`: the displacement of every spot from its lenslet centre, and its flux, for one frame or a stack
    (pb_subaperture_centroids, one launch);
  - `ShackHartmann`: the sensor as an object -- forward model, slopes, a calibrated modal reconstructor and the
    reconstruction itself as a batched GEMV on the device (pb_sh_reconstruct), so that a loop of
    forward_model -> slopes -> reconstruct never leaves the device and can be captured in a CUDA graph.
"""
import inspect
from math import ceil

import numpy as np
import torch

from . import _ops
from ._capi import LENSLET_CIRCLE, LENSLET_RECT, LENSLET_RECT_ROTATED, LENSLET_RECT_SWAP
from .conf import config
from .geometry import circle as _circle, rectangle as _rectangle
from .propagation import Wavefront
from .sri import _wave

rectangle = _rectangle


def _n_pair(n):
    """(rows, cols) of lenslets: a scalar n is (n, n), as in the reference."""
    if not hasattr(n, '__iter__'):
        n = (n, n)
    n = tuple(int(v) for v in n)
    if len(n) != 2 or min(n) < 1:
        raise ValueError(f'n must be a positive int or a pair of them, got {n}')
    return n


def lenslet_centres(pitch, n, shift=False):
    """(xc, yc): the lenslet centres of shack_hartmann, in config.precision on the host.  xc has n[1] entries and yc
    n[0] (make_xy_grid takes (rows, cols)); with shift, the parity of n[0] decides the x shift and that of n[1] the
    y shift, as in the reference (shack_hartmann.py:83-89)."""
    n = _n_pair(n)
    yc, xc = (np.arange(-(s // 2), -(s // 2) + s, dtype=config.precision) * pitch for s in n)
    if shift:
        if not n[0] & 1:
            xc += (pitch / 2)
        if not n[1] & 1:
            yc += (pitch / 2)
    return xc, yc


def _host_scalar(v):
    """A 0-d device tensor or a numpy scalar -> the numpy scalar of the same dtype."""
    if isinstance(v, torch.Tensor):
        return v.detach().cpu().numpy()[()]
    return v


def _host_vector(a):
    return np.asarray(_ops.asnumpy(a), dtype=np.float64)


def _windows(centres, dx, spl, c, size):
    """The reference's _local_window along one axis for every lenslet (prysm/segmented.py:102-130): [c + int(centre /
    dx) - spl, + 2 spl), clamped to [0, size].  The quotient has the reference's dtype (numpy's promotion of the
    centres' and dx's types) and int() truncates it."""
    lo = c + np.trunc(centres / dx).astype(np.int64) - spl
    hi = lo + 2 * spl
    return np.clip(lo, 0, size), np.clip(hi, 0, size)


def _candidates(lo, hi, size):
    """Per grid index, the (first, one past last) lenslet whose window [lo, hi) covers it: windows move monotonically
    with the centres, so the set is contiguous."""
    k = np.arange(size)[:, None]
    cov = (lo[None, :] <= k) & (k < hi[None, :])
    idx = np.arange(len(lo))
    first = np.where(cov, idx, len(lo)).min(axis=1)
    last = np.where(cov, idx, -1).max(axis=1) + 1
    count = cov.sum(axis=1)
    if np.any((count > 0) & (last - first != count)):
        raise ValueError('the lenslet windows are not monotone in the lenslet index: pitch must be positive')
    first = np.where(count > 0, first, 0)
    last = np.where(count > 0, last, 0)
    return np.stack((first, last), axis=1).astype(np.int32)


def _aperture_kind(aperture, kw, pitch):
    """(kind, params) of a recognised aperture (the reference's or this package's rectangle / circle), else None."""
    mod, name = getattr(aperture, '__module__', ''), getattr(aperture, '__name__', '')
    is_rect = aperture is _rectangle or (mod == 'prysm.geometry' and name == 'rectangle')
    is_circle = aperture is _circle or (mod == 'prysm.geometry' and name == 'circle')
    width = pitch / 2
    if is_rect:
        extra = set(kw) - {'height', 'angle'}
        if extra:
            raise TypeError(f'rectangle() got an unexpected keyword argument {sorted(extra)[0]!r}')
        height = kw.get('height')
        height = width if height is None else height
        angle = kw.get('angle', 0)
        if angle == 0:
            return LENSLET_RECT, (width, height, 0.0, 0.0)
        if angle == 90:
            return LENSLET_RECT_SWAP, (width, height, 0.0, 0.0)
        return LENSLET_RECT_ROTATED, (width, height, float(np.radians(angle)), 0.0)
    if is_circle:
        if kw:
            raise TypeError(f'circle() got an unexpected keyword argument {sorted(kw)[0]!r}')
        return LENSLET_CIRCLE, (0.0, 0.0, 0.0, (pitch / 2) ** 2)
    return None


class _ScreenPlan:
    """The host half of shack_hartmann for one grid: centres, windows and per-column / per-row candidate lenslets,
    with their device copies."""

    def __init__(self, pitch, n, x, y, shift):
        self.n = _n_pair(n)
        self.xc, self.yc = lenslet_centres(pitch, self.n, shift)
        self.H, self.W = (int(v) for v in x.shape)
        dx = _host_scalar(x[0, 1] - x[0, 0])
        spl = int(pitch / dx + 1)                 # the reference's dtypes: a float32 quotient when x is float32
        cx, cy = ceil(self.W / 2), ceil(self.H / 2)
        self.xlo, self.xhi = _windows(self.xc, dx, spl, cx, self.W)
        self.ylo, self.yhi = _windows(self.yc, dx, spl, cy, self.H)
        cand = np.concatenate((_candidates(self.xlo, self.xhi, self.W).ravel(),
                               _candidates(self.ylo, self.yhi, self.H).ravel()))
        self.cand = _ops.asdevice(cand)
        self.centres = _ops.asdevice(np.concatenate((self.xc, self.yc)).astype(np.float64))


def _prefix_imag(wavelength):
    prefix = -1j * 2 * np.pi / (wavelength / 1e3)
    return prefix.imag


def _screen_any_aperture(plan, pitch, efl, wavelength, x, y, aperture, kw):
    """The reference's loop with `aperture` evaluated on device tensors: correct for any callable that takes (x, y) or
    r keyword arguments and accepts tensors, but one small launch sequence per lenslet -- slow."""
    callxy = {'x', 'y'} <= set(inspect.signature(aperture).parameters)
    total = torch.zeros_like(x)
    for j, yy in enumerate(plan.yc):
        for i, xx in enumerate(plan.xc):
            win = (slice(int(plan.ylo[j]), int(plan.yhi[j])), slice(int(plan.xlo[i]), int(plan.xhi[i])))
            lx = x[win] - float(xx)
            ly = y[win] - float(yy)
            rsq = lx * lx + ly * ly
            phase = rsq / (2 * efl)
            if callxy:
                m = aperture(pitch / 2, x=lx, y=ly, **kw)
            else:
                m = aperture((pitch / 2) ** 2, r=rsq, **kw)
            total[win] += phase * _ops.asdevice(m).to(phase.dtype)
    return _ops.phase_screen(None, total, _prefix_imag(wavelength))


def _real_grids(x, y):
    x = _ops.asdevice(x)
    if x.dtype not in (torch.float32, torch.float64):
        x = x.to(config.real_dtype)
    y = _ops.asdevice(y, x.dtype)
    if x.ndim != 2 or tuple(y.shape) != tuple(x.shape):
        raise ValueError('x and y must be 2-D grids of one shape')
    return x, y


def _screen(plan, pitch, efl, wavelength, x, y, aperture, aperture_kwargs):
    kw = {} if aperture_kwargs is None else dict(aperture_kwargs)
    known = _aperture_kind(aperture, kw, pitch)
    if known is None:
        return _screen_any_aperture(plan, pitch, efl, wavelength, x, y, aperture, kw)
    kind, params = known
    return _ops.lenslet_screen(x, y, plan.centres, plan.cand, kind, params, 2 * efl, _prefix_imag(wavelength),
                               len(plan.xc), len(plan.yc))


_PLANS = {}            # (pitch, n, shift, shape, dx and its dtype, precision, device) -> _ScreenPlan; most recent last
_MAX_PLANS = 8


def _plan_for(pitch, n, x, y, shift):
    """The screen plan of this grid, cached: it depends on the grid only through its shape and spacing."""
    dx = _host_scalar(x[0, 1] - x[0, 0])
    key = (float(pitch), _n_pair(n), bool(shift), tuple(x.shape), float(dx), np.dtype(type(dx)).str,
           np.dtype(config.precision).str, str(x.device))
    plan = _PLANS.pop(key, None)
    if plan is None:
        plan = _ScreenPlan(pitch, n, x, y, shift)
        while len(_PLANS) >= _MAX_PLANS:
            _PLANS.pop(next(iter(_PLANS)))
    _PLANS[key] = plan
    return plan


def shack_hartmann(pitch, n, efl, wavelength, x, y, aperture=rectangle, aperture_kwargs=None, shift=False):
    """The complex screen of a lenslet array (prysm/x/shack_hartmann.py:11-120), a device tensor in the precision of x.

    pitch [mm], n lenslets (an int or (rows, cols)), efl [mm] of each lenslet, wavelength [um], x / y the grids [mm].
    Propagate it with `(wf * screen).free_space(dz=efl)`.

    `aperture` is evaluated natively, in one launch for the whole array, when it is `rectangle` (with `height` and
    `angle`) or `circle`, the reference's or this package's: rectangle(pitch/2, x=lx, y=ly, **kw) or
    circle(pitch^2/4, r=rsq).  Any other callable runs the reference's loop over lenslets with the callable applied to
    device tensors: correct, but one short launch sequence per lenslet, so slow on large arrays.

    The reference's behaviours are kept: a sample on an edge shared by several lenslets takes the phase of each of
    them; `n = (n0, n1)` gives n1 lenslet columns and n0 rows; `shift` moves x by half a pitch when n[0] is even and y
    when n[1] is even."""
    x, y = _real_grids(x, y)
    plan = _plan_for(pitch, n, x, y, shift)
    return _screen(plan, pitch, efl, wavelength, x, y, aperture, aperture_kwargs)


# ---- centroids -----------------------------------------------------------------------------------------------------
def _owners(coords, centres, pitch):
    """Owner lenslet of each coordinate, lowest index first where rounding lets two half-open intervals meet, -1 for
    none; and each lenslet's owned index range [lo, hi)."""
    c = np.asarray(centres, dtype=np.float64)
    lo, hi = c - pitch / 2, c + pitch / 2
    cov = (lo[None, :] <= coords[:, None]) & (coords[:, None] < hi[None, :])
    owner = np.where(cov.any(axis=1), cov.argmax(axis=1), -1)
    rng = np.zeros((2, len(c)), dtype=np.int64)
    for i in range(len(c)):
        where = np.flatnonzero(owner == i)
        if where.size:
            if where[-1] - where[0] + 1 != where.size:
                raise ValueError('the grid coordinates must increase along each axis')
            rng[:, i] = where[0], where[-1] + 1
    return owner, rng


class CentroidPlan:
    """The device tables of spot_centroids for one grid and lenslet array (built once by ShackHartmann)."""

    def __init__(self, x, y, pitch, n, shift=False):
        self.n = _n_pair(n)
        self.xc, self.yc = lenslet_centres(pitch, self.n, shift)
        xv = _host_vector(x[0, :] if getattr(x, 'ndim', 1) == 2 else x)
        yv = _host_vector(y[:, 0] if getattr(y, 'ndim', 1) == 2 else y)
        self.shape = (len(yv), len(xv))
        xo, xr = _owners(xv, self.xc, pitch)
        yo, yr = _owners(yv, self.yc, pitch)
        self.col_owner, self.row_owner = xo, yo
        self.col_range, self.row_range = xr, yr
        self.dtab = _ops.asdevice(np.concatenate((xv, yv, self.xc.astype(np.float64), self.yc.astype(np.float64))))
        self.itab = _ops.asdevice(np.concatenate((xo, xr.ravel(), yr.ravel())).astype(np.int32))

    def __call__(self, frames, threshold=0.0, scale=1.0):
        if not isinstance(frames, (np.ndarray, torch.Tensor)) and hasattr(frames, 'data'):
            frames = frames.data                     # RichData (forward_model's result)
        f = _ops.asdevice(frames)
        if f.ndim not in (2, 3) or tuple(f.shape[-2:]) != self.shape:
            raise ValueError(f'frames must be (H, W) or (F, H, W) with (H, W) = {self.shape}, got {tuple(f.shape)}')
        single = f.ndim == 2
        disp, flux = _ops.subaperture_centroids(f[None] if single else f, self.dtab, self.itab, len(self.xc),
                                                len(self.yc), threshold, scale)
        return (disp[0], flux[0]) if single else (disp, flux)


def spot_centroids(frames, x, y, pitch, n, shift=False, threshold=0.0):
    """Per-subaperture spot displacements and fluxes of one frame (H, W) or a stack (F, H, W), in one launch.

    Definition (an engine extension; the reference has no measurement side):
      - the lenslet centres xc_i, yc_j are those of shack_hartmann(pitch, n, ..., shift=shift), parity quirk included;
      - lenslet (j, i) owns the samples with xc_i - pitch/2 <= x < xc_i + pitch/2 and yc_j - pitch/2 <= y < yc_j +
        pitch/2 (in fp64, x read along the first row of x and y down the first column of y).  The intervals are
        half-open, so no sample has two owners (where rounding lets two meet, the lower index owns); samples no
        lenslet owns are ignored;
      - weights w = max(I - t, 0) with t = threshold * max(I over the subaperture);
      - disp = (sum w x / sum w - xc_i, sum w y / sum w - yc_j) in grid units, shape (..., 2, n_rows, n_cols), NaN where
        sum w = 0; flux = sum I, shape (..., n_rows, n_cols).
    Frames may be float32, float64, uint16 or int32 (Detector.expose output goes in directly).  The sums are fp64 in
    a fixed order (repeated calls are bit-identical); the results are float64 for float64 frames, float32 otherwise.

    This function plans on every call: it reads x and y to the host (a synchronising copy when they are device
    tensors) and uploads the ownership tables before its one launch.  For repeated frames on one grid, build a
    CentroidPlan once (or use ShackHartmann.slopes): its calls neither synchronise nor re-plan, and can be captured in
    a CUDA graph."""
    return CentroidPlan(x, y, pitch, n, shift)(frames, threshold)


# ---- the sensor ----------------------------------------------------------------------------------------------------
class ShackHartmann:
    """A Shack-Hartmann wavefront sensor: lenslet array, spot centroids and a modal reconstructor (an engine extension
    in the style of SelfReferencedInterferometer)."""

    def __init__(self, pitch, n, efl, wavelength, x, y, aperture=rectangle, aperture_kwargs=None, shift=False,
                 threshold=0.0):
        """Same lenslet parameters as shack_hartmann; threshold is spot_centroids'.  The screen plan and the centroid
        tables are built here, once."""
        self.pitch, self.n, self.efl, self.wavelength = pitch, _n_pair(n), efl, wavelength
        self.x, self.y = _real_grids(x, y)
        self.dx = float(self.x[0, 1] - self.x[0, 0])
        self.aperture, self.aperture_kwargs, self.shift, self.threshold = aperture, aperture_kwargs, shift, threshold
        self._plan = _ScreenPlan(pitch, self.n, self.x, self.y, shift)
        self.centroids = CentroidPlan(self.x, self.y, pitch, self.n, shift)
        self._screens = {}
        self.valid = None               # (n_rows, n_cols) bool, set by calibrate
        self.interaction = None         # (2 n_valid, K) fp64 host: d slopes / d coefficient
        self.reconstructor = None       # (K, 2 n_valid) fp64 host: its pseudo-inverse
        self.reference_slopes = None    # (2, n_rows, n_cols) slopes of the unaberrated pupil

    def screen(self, wavelength=None, dtype=None):
        """The complex lenslet screen at `wavelength` (default: the sensor's), built once and cached."""
        wavelength = self.wavelength if wavelength is None else wavelength
        key = (wavelength, dtype)
        if key not in self._screens:
            s = _screen(self._plan, self.pitch, self.efl, wavelength, self.x, self.y, self.aperture,
                        self.aperture_kwargs)
            self._screens[key] = s if dtype is None else s.to(dtype)
        return self._screens[key]

    def forward_model(self, wave):
        """Intensity at the lenslets' focal plane as RichData: (wave * screen).free_space(dz=efl), then |.|^2.  The
        product is fused into the first pass of the angular-spectrum transform."""
        wave = _wave(wave, self.wavelength, self.dx)
        scr = self.screen(wave.wavelength, wave.data.dtype)
        return (wave * scr).free_space(dz=self.efl).intensity

    def slopes(self, frames):
        """spot_centroids(frames, ...) / efl: the spot displacements as angles [rad], (..., 2, n_rows, n_cols)."""
        disp, _ = self.centroids(frames, self.threshold, scale=1.0 / self.efl)
        return disp

    def calibrate(self, modes, amplitude, valid_fraction=0.5, rcond=1e-6, amp=None):
        """Build the modal reconstructor from `modes` (K, H, W) of OPD [nm] on the pupil grid.

        Each mode is pushed through forward_model at +amplitude and -amplitude (amp: the pupil amplitude, default 1
        everywhere) and its interaction column is (slopes(+) - slopes(-)) / (2 amplitude).  The valid subapertures are
        those whose flux in the unaberrated frame reaches valid_fraction of the largest.  The reconstructor is the fp64
        pseudo-inverse (numpy.linalg.pinv, rcond) over the valid subapertures, computed once on the host; the
        unaberrated slopes are kept as the reference that reconstruct subtracts.  Returns the reconstructor."""
        modes = _ops.asdevice(modes)
        if modes.ndim != 3 or tuple(modes.shape[1:]) != tuple(self.x.shape):
            raise ValueError(f'modes must be (K, H, W) on the pupil grid {tuple(self.x.shape)}')
        a = torch.ones_like(self.x) if amp is None else _ops.asdevice(amp, self.x.dtype)

        def measure(opd):
            wave = Wavefront.from_amp_and_phase(a, opd, self.wavelength, self.dx)
            return self.centroids(self.forward_model(wave), self.threshold, scale=1.0 / self.efl)

        s0, f0 = measure(torch.zeros_like(self.x))
        f0 = _ops.asnumpy(f0).astype(np.float64)
        valid = f0 >= valid_fraction * f0.max()
        s0 = _ops.asnumpy(s0).astype(np.float64)
        cols = []
        for k in range(modes.shape[0]):
            sp, _ = measure(modes[k] * amplitude)
            sm, _ = measure(modes[k] * -amplitude)
            d = (_ops.asnumpy(sp).astype(np.float64) - _ops.asnumpy(sm).astype(np.float64)) / (2 * amplitude)
            cols.append(np.concatenate((d[0][valid], d[1][valid])))
        D = np.stack(cols, axis=1)
        R = np.linalg.pinv(D, rcond=rcond)
        flat = np.flatnonzero(valid.ravel())
        idx = np.concatenate((flat, valid.size + flat)).astype(np.int32)
        self.valid, self.interaction, self.reconstructor, self.reference_slopes = valid, D, R, s0
        self._idx = _ops.asdevice(idx)
        self._ref = _ops.asdevice(np.concatenate((s0[0][valid], s0[1][valid])))
        self._R = _ops.asdevice(np.ascontiguousarray(R))
        return R

    def reconstruct(self, slopes):
        """Modal coefficients R (s - s_ref) over the valid subapertures, (K,) for slopes (2, n_rows, n_cols) or (F, K)
        for (F, 2, n_rows, n_cols), one launch (pb_sh_reconstruct).  The result stays on the device and nothing
        synchronises, so the call can be captured in a CUDA graph.  A NaN slope in a valid subaperture propagates to
        every coefficient.  Slopes of another shape or dtype (float32 and float64 are accepted) raise ValueError
        before anything is launched."""
        if self.reconstructor is None:
            raise RuntimeError('calibrate() the sensor before reconstructing')
        s = _ops.asdevice(slopes)
        frame = (2, *self.valid.shape)
        if s.ndim not in (3, 4) or tuple(s.shape[-3:]) != frame:
            raise ValueError(f'slopes must be {frame} or (F, {", ".join(map(str, frame))}), got {tuple(s.shape)}')
        if s.dtype not in (torch.float32, torch.float64):
            raise ValueError(f'slopes must be float32 or float64, got {s.dtype}')
        single = s.ndim == 3
        out = _ops.sh_reconstruct(s[None] if single else s, self._idx, self._ref, self._R, frame)
        return out[0] if single else out
