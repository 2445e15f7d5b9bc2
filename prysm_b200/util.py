"""NaN-aware statistics of prysm/util.py:7-97 (mean, pv, rms, Sa, std) on the device.

All five come from one pair of launches (pb_nan_stats): the first pass reduces the finite count, sum, min, max and
sum of squares, the second reads the mean from device memory and reduces sum |x - mean| and sum (x - mean)^2, so
std is numpy's two-pass population std (ddof 0).  The sums are fp64 at either storage precision and the results are
Python floats.  Only finite samples count: NaN and +-inf are ignored, as `np.isfinite` ignores them in the reference.
"""
import numpy as np

from . import _ops


def _data(array):
    a = _ops.asdevice(array)
    if a.dtype not in (_ops.torch.float32, _ops.torch.float64):
        a = a.to(_ops.torch.float64)
    return a


def nan_stats(array):
    """The nine fp64 sums of pb_nan_stats as a host array: finite count, sum, min, max, sum of squares, NaN count,
    mean, sum |x - mean|, sum (x - mean)^2."""
    return _ops.nan_stats(_data(array))


def _div(a, b):
    with np.errstate(divide='ignore', invalid='ignore'):
        return float(np.float64(a) / np.float64(b))


def mean(array):
    """Mean of the finite elements of an array."""
    s = nan_stats(array)
    return _div(s[1], s[0])


def pv(array):
    """Peak-to-valley of the finite elements of an array."""
    s = nan_stats(array)
    if not s[0]:
        raise ValueError('zero-size array to reduction operation maximum which has no identity')
    return float(s[3] - s[2])


def rms(array):
    """Root mean square (about zero) of the finite elements of an array."""
    s = nan_stats(array)
    return float(np.sqrt(_div(s[4], s[0])))


def Sa(array):
    """Mean absolute deviation from the mean of the finite elements of an array (DIN/ISO Sa)."""
    s = nan_stats(array)
    return _div(s[7], s[0])


def std(array):
    """Population standard deviation (ddof 0) of the finite elements of an array."""
    s = nan_stats(array)
    return float(np.sqrt(_div(s[8], s[0])))
