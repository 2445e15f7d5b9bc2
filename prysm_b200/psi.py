"""Phase-shifting interferometry on the device (reference prysm/x/psi.py).

`psi_accumulate` and `degroot_formalism_psi` are one pass over the frames (pb_psi): both weighted sums accumulate in
fp64 (in int64, exactly, for integer frames and integer weights) and the wrapped phase atan2(num, den) is written in
the same pass, so a 13-frame reconstruction reads each frame once and launches one kernel.  Frames may be a (N, ...)
array or a sequence of N arrays (read in place through a pointer list, never stacked), of float32, float64, uint16 or
int32.

Output types.  Float frames keep their type: the weights are rounded to it first, as the reference's
`sum_of_2d_modes` does.  Integer frames give int64 sums with integer weights and float64 sums otherwise, and a float64
phase.  (The reference casts the weights to the frames' type, so uint16 frames wrap the negative weights modulo 2^16;
the engine does not reproduce that.)

`unwrap_phase` is not provided: the reference wraps scikit-image's unwrapper.
"""
from collections import namedtuple

import numpy as np
import torch
from scipy import signal

from . import _ops

Scheme = namedtuple('Scheme', ['shifts', 's', 'c'])


def _fftrange(n):
    return np.arange(-(n // 2), -(n // 2) + n)


ZYGO_THIRTEEN_FRAME = Scheme(
    _fftrange(13) * np.pi / 4,
    np.asarray((-3, -4, 0, 12, 21, 16, 0, -16, -21, -12, 0, 4, 3)),
    np.asarray((0, -4, -12, -12, 0, 16, 24, 16, 0, -12, -12, -4, 0)),
)

SCHWIDER = Scheme(
    _fftrange(5) * np.pi / 2,
    np.asarray((0, 2, 0, -2, 0)),
    np.asarray((-1, 0, 2, 0, -1)),
)

_FLOAT = {torch.float32: np.float32, torch.float64: np.float64}


def _frames(gs):
    """A (N, ...) device tensor, or a list of N device tensors, of the frames gs (RichData unwrapped)."""
    if isinstance(gs, torch.Tensor):
        return _ops.asdevice(gs)
    if isinstance(gs, np.ndarray):
        return _ops.asdevice(gs)
    return [_ops.asdevice(getattr(g, 'data', g)) for g in gs]


def _run(gs, scheme, want_num, want_phase):
    frames = _frames(gs)
    dt = frames.dtype if isinstance(frames, torch.Tensor) else frames[0].dtype
    s, c = np.asarray(scheme.s), np.asarray(scheme.c)
    if dt in _FLOAT:
        # sum_of_2d_modes converts the weights to the frames' dtype (polynomials/fitting.py:32-34)
        s, c = s.astype(_FLOAT[dt]), c.astype(_FLOAT[dt])
        num_dt = phase_dt = dt
    else:
        integral = s.dtype.kind in 'iub' and c.dtype.kind in 'iub'
        num_dt, phase_dt = (torch.int64 if integral else torch.float64), torch.float64
    return _ops.psi(frames, s.astype(np.float64), c.astype(np.float64), num_dt, phase_dt, want_num=want_num,
                    want_phase=want_phase)


def psi_accumulate(gs, scheme):
    """Numerator (sine) and denominator (cosine) sums of a PSI scheme over the frames gs (psi.py:45-71), one pass."""
    num, den, _ = _run(gs, scheme, True, False)
    return num, den


def degroot_formalism_psi(gs, scheme):
    """Wrapped phase atan2(sum s g, sum c g) of the frames gs (psi.py:74-109), one kernel launch.  RichData frames give
    a RichData of the first frame's dx and wavelength."""
    first = gs[0]
    was_rd = not isinstance(gs, (torch.Tensor, np.ndarray)) and hasattr(first, 'data') and hasattr(first, 'dx')
    _, _, out = _run(gs, scheme, False, True)
    if was_rd:
        from ._richdata import RichData
        out = RichData(out, first.dx, first.wavelength)
    return out


def design_scheme(N, stepsize=None, window=None):
    """A PSI scheme of N steps, the sines and cosines of the shifts times an optional window (psi.py:112-157); host
    arrays."""
    if stepsize is None:
        stepsize = (2 * np.pi) / (N - 1)
    shifts = _fftrange(N) * stepsize
    s = np.sin(shifts)
    c = np.cos(shifts)
    if window is not None:
        if isinstance(window, str):
            window = signal.windows.get_window(window, N)
        s *= window
        c *= window
    return Scheme(shifts, s, c)
