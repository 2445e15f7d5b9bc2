"""GPU: the generic shared-memory axis pass (csrc/axis_pass.cu, axis_pass_kernel<R>) and Bluestein's algorithm on top of
it (csrc/fft2.cu: axis_dft, get_chirp, get_chirp_filter), held to an extended-precision reference over whole arrays.

This kernel runs every complex128 transform (focus / unfocus and their adjoints, angular_spectrum, the CZT executor,
fft2, fft1, mtf_from_psf at precision 64) and every length the register engine does not take, at both precisions.
The reference is scipy.fft on np.clongdouble (tests/generic_reference.py; eps 1.1e-19) fed the exact complex64 /
complex128 values the device got, and device-built multiplier vectors (the CZT plan, the transfer-function vectors) are
pulled to the host and upcast, so a figure is the error of the transform and not of the plan.  The plan vectors are
checked on their own against their long-double closed forms (`test_czt_plan_vectors`, `test_angular_spectrum_vectors`).
Sums of impulses have a closed form (`impulse_centred_ft2`), which the public entry points use where the padded size
passes 1024.

Every output array is compared whole by rel_linf (max|a - b| / max|b|) and the relative L2 error.  Bounds are 1.5x
the figures measured on an H100 (`MEASURED`, recorded with PB_TEST_MEASUREMENTS; the arithmetic is deterministic) and
never above the ceilings 1e-14 (complex128) and 1e-6 (complex64).  A figure above a ceiling is a finding, not a reason
to raise it: a complex128 Bluestein whose chirp angle pi j^2 / n is formed in fp64 without the exact reduction of j^2
mod 2n lands near 1e-12 (tests/test_host_generic_reference.py).  Ranges of the measured figures, H100 80GB HBM3 at a 700 W power limit:

    complex128  fft1, every length, rows / cols   linf 1.0e-16-7.6e-16, l2 7.2e-17-6.4e-16 (lengths 1 and 2: exact)
    complex128  fft2, pads, shifts, crops, kinds  linf 3.1e-16-9.3e-16, l2 2.8e-16-8.0e-16
    complex128  focus family, Q 1-3, N 64-1023    linf 2.0e-16-2.2e-15, l2 2.1e-16-1.0e-15
    complex128  axis_dft with multipliers         linf 3.0e-16-9.5e-16, l2 2.3e-16-5.8e-16
    complex128  CZT, K 16-8192                    linf 2.2e-16-1.0e-15, l2 1.9e-16-4.3e-16
    complex128  angular_spectrum                  linf 3.4e-16-1.4e-15, l2 4.1e-16-1.3e-15
    complex128  polychromatic_psf(kind='czt')     linf 1.7e-15, l2 2.7e-15
    complex64   fft1, every length, rows / cols   linf 3.1e-08-3.3e-07, l2 2.8e-08-2.2e-07 (lengths 1 and 2: exact)
    complex64   fft2, pads, shifts, crops, kinds  linf 1.7e-07-6.5e-07, l2 1.6e-07-3.2e-07
    complex64   axis_dft with multipliers         linf 1.7e-07-3.7e-07, l2 1.3e-07-2.1e-07
    complex64   CZT, K 16-512, 8192, 16384        linf 1.1e-07-4.0e-07, l2 8.9e-08-2.6e-07
    complex64   angular_spectrum                  linf 4.0e-07-5.3e-07, l2 3.7e-07-4.4e-07

Every case also pins the kernel it ran, from the per-route launch counters (pb_route_launch_count): generic launches
per (L, dtype, column pass) exactly as `axis_launches` predicts -- one per power-of-two axis pass, two per Bluestein
axis at its padded length -- and no launch of the register engine, the focus pair or any other kernel.  The last test
asserts that every (L, dtype, orientation) the Python API can reach on this kernel ran in a checked case.
"""
import math
import os

import numpy as np
import pytest
import scipy.fft as sfft
import torch

import generic_reference as G
from accuracy import Ledger
from generic_reference import PB_C64, PB_C128, DT_NAME, CEILING, LD
from gpu_fixtures import pb, dev, host  # noqa: F401
from gpu_fixtures import crand as _crand
from gpu_fixtures import routes_of

pytestmark = pytest.mark.gpu

DTYPES = (PB_C64, PB_C128)
TDT = {PB_C64: torch.complex64, PB_C128: torch.complex128}
RDT = {PB_C64: torch.float32, PB_C128: torch.float64}
NPR = {PB_C64: np.float32, PB_C128: np.float64}
WEIGHT = 0.375
KSCALE = 2 * np.pi / 0.6328 / 1e3          # OPD [nm] -> radians at HeNe
TUNED = (1024, 2048, 4096)                 # power-of-two lengths the complex64 register engine takes
BLUESTEIN = (3, 5, 7, 97, 255, 257, 1000, 1023, 1025, 2047, 4093, 4095)
ROWS_COLS = ('rows', 'cols')


def pow2_lengths(dt):
    return [1 << i for i in range(G.max_pow2_len(dt).bit_length())]


def bluestein_lengths(dt):
    return BLUESTEIN + ((8191,) if dt == PB_C64 else ())


# ---- measured figures (H100 80GB HBM3, 700 W power limit); bounds are 1.5x these, capped at the ceiling of the dtype --
MEASURED = {
    'c128/after_refusal_cols/1000': dict(linf=6.79e-16, l2=5.53e-16),
    'c128/after_refusal_rows/1000': dict(linf=5.93e-16, l2=5.69e-16),
    'c128/as_matrix/1024x1024': dict(linf=4.70e-16, l2=4.43e-16),
    'c128/as_matrix/383x300': dict(linf=1.35e-15, l2=1.31e-15),
    'c128/as_matrix/512x512': dict(linf=5.24e-16, l2=4.14e-16),
    'c128/as_screen/1024x1024': dict(linf=4.82e-16, l2=4.52e-16),
    'c128/as_screen/383x300': dict(linf=1.26e-15, l2=1.32e-15),
    'c128/as_screen/512x512': dict(linf=3.41e-16, l2=4.23e-16),
    'c128/as_vectors/1024x1024': dict(linf=5.23e-16, l2=4.47e-16),
    'c128/as_vectors/383x300': dict(linf=1.32e-15, l2=1.32e-15),
    'c128/as_vectors/512x512': dict(linf=3.59e-16, l2=4.17e-16),
    'c128/axis_dft_cols/1000': dict(linf=9.38e-16, l2=5.64e-16),
    'c128/axis_dft_cols/256': dict(linf=2.95e-16, l2=2.34e-16),
    'c128/axis_dft_cols/97': dict(linf=4.11e-16, l2=4.60e-16),
    'c128/axis_dft_rows/1000': dict(linf=9.53e-16, l2=5.77e-16),
    'c128/axis_dft_rows/256': dict(linf=4.29e-16, l2=2.29e-16),
    'c128/axis_dft_rows/97': dict(linf=6.36e-16, l2=4.51e-16),
    'c128/czt/1024': dict(linf=5.01e-16, l2=3.16e-16),
    'c128/czt/128': dict(linf=3.37e-16, l2=2.60e-16),
    'c128/czt/16': dict(linf=2.82e-16, l2=2.42e-16),
    'c128/czt/2048': dict(linf=3.63e-16, l2=3.35e-16),
    'c128/czt/256': dict(linf=3.20e-16, l2=2.85e-16),
    'c128/czt/32': dict(linf=3.03e-16, l2=2.12e-16),
    'c128/czt/4096': dict(linf=3.67e-16, l2=3.47e-16),
    'c128/czt/512': dict(linf=3.08e-16, l2=3.02e-16),
    'c128/czt/64': dict(linf=3.33e-16, l2=2.57e-16),
    'c128/czt/8192': dict(linf=4.39e-16, l2=3.62e-16),
    'c128/czt_accumulate/1024': dict(linf=1.01e-15, l2=3.80e-16),
    'c128/czt_accumulate/128': dict(linf=5.52e-16, l2=3.51e-16),
    'c128/czt_accumulate/16': dict(linf=4.68e-16, l2=2.56e-16),
    'c128/czt_accumulate/2048': dict(linf=4.58e-16, l2=3.99e-16),
    'c128/czt_accumulate/256': dict(linf=4.50e-16, l2=3.52e-16),
    'c128/czt_accumulate/32': dict(linf=4.54e-16, l2=2.73e-16),
    'c128/czt_accumulate/4096': dict(linf=7.63e-16, l2=4.19e-16),
    'c128/czt_accumulate/512': dict(linf=6.94e-16, l2=3.75e-16),
    'c128/czt_accumulate/64': dict(linf=6.08e-16, l2=3.14e-16),
    'c128/czt_accumulate/8192': dict(linf=5.85e-16, l2=4.33e-16),
    'c128/czt_adjoint/1024': dict(linf=3.38e-16, l2=3.16e-16),
    'c128/czt_adjoint/128': dict(linf=2.95e-16, l2=2.65e-16),
    'c128/czt_adjoint/16': dict(linf=2.21e-16, l2=1.88e-16),
    'c128/czt_adjoint/2048': dict(linf=4.01e-16, l2=3.35e-16),
    'c128/czt_adjoint/256': dict(linf=3.91e-16, l2=2.79e-16),
    'c128/czt_adjoint/32': dict(linf=2.43e-16, l2=2.00e-16),
    'c128/czt_adjoint/4096': dict(linf=3.60e-16, l2=3.47e-16),
    'c128/czt_adjoint/512': dict(linf=2.72e-16, l2=2.96e-16),
    'c128/czt_adjoint/64': dict(linf=3.09e-16, l2=2.53e-16),
    'c128/czt_adjoint/8192': dict(linf=3.93e-16, l2=3.64e-16),
    'c128/czt_intensity/1024': dict(linf=1.03e-15, l2=3.77e-16),
    'c128/czt_intensity/128': dict(linf=4.74e-16, l2=3.40e-16),
    'c128/czt_intensity/16': dict(linf=4.91e-16, l2=3.16e-16),
    'c128/czt_intensity/2048': dict(linf=4.74e-16, l2=3.96e-16),
    'c128/czt_intensity/256': dict(linf=4.00e-16, l2=3.53e-16),
    'c128/czt_intensity/32': dict(linf=5.55e-16, l2=2.99e-16),
    'c128/czt_intensity/4096': dict(linf=7.03e-16, l2=4.16e-16),
    'c128/czt_intensity/512': dict(linf=6.72e-16, l2=3.76e-16),
    'c128/czt_intensity/64': dict(linf=5.89e-16, l2=3.24e-16),
    'c128/czt_intensity/8192': dict(linf=5.92e-16, l2=4.31e-16),
    'c128/edge_accepted_cols/4095': dict(linf=6.28e-16, l2=6.33e-16),
    'c128/edge_accepted_cols/8192': dict(linf=2.88e-16, l2=2.44e-16),
    'c128/edge_accepted_rows/4095': dict(linf=6.67e-16, l2=6.29e-16),
    'c128/edge_accepted_rows/8192': dict(linf=2.60e-16, l2=2.44e-16),
    'c128/fft1_cols_fwd/1': dict(linf=0.0, l2=0.0),
    'c128/fft1_cols_fwd/1000': dict(linf=6.07e-16, l2=5.56e-16),
    'c128/fft1_cols_fwd/1023': dict(linf=6.09e-16, l2=5.62e-16),
    'c128/fft1_cols_fwd/1024': dict(linf=2.76e-16, l2=2.10e-16),
    'c128/fft1_cols_fwd/1025': dict(linf=5.79e-16, l2=5.04e-16),
    'c128/fft1_cols_fwd/128': dict(linf=2.06e-16, l2=1.79e-16),
    'c128/fft1_cols_fwd/16': dict(linf=1.71e-16, l2=1.27e-16),
    'c128/fft1_cols_fwd/2': dict(linf=1.07e-16, l2=9.23e-17),
    'c128/fft1_cols_fwd/2047': dict(linf=5.82e-16, l2=6.08e-16),
    'c128/fft1_cols_fwd/2048': dict(linf=3.18e-16, l2=2.26e-16),
    'c128/fft1_cols_fwd/255': dict(linf=5.97e-16, l2=4.88e-16),
    'c128/fft1_cols_fwd/256': dict(linf=2.40e-16, l2=1.84e-16),
    'c128/fft1_cols_fwd/257': dict(linf=4.96e-16, l2=4.42e-16),
    'c128/fft1_cols_fwd/3': dict(linf=2.88e-16, l2=1.63e-16),
    'c128/fft1_cols_fwd/32': dict(linf=1.88e-16, l2=1.37e-16),
    'c128/fft1_cols_fwd/4': dict(linf=1.10e-16, l2=7.96e-17),
    'c128/fft1_cols_fwd/4093': dict(linf=7.50e-16, l2=6.39e-16),
    'c128/fft1_cols_fwd/4095': dict(linf=7.60e-16, l2=6.43e-16),
    'c128/fft1_cols_fwd/4096': dict(linf=2.70e-16, l2=2.33e-16),
    'c128/fft1_cols_fwd/5': dict(linf=2.51e-16, l2=2.97e-16),
    'c128/fft1_cols_fwd/512': dict(linf=2.69e-16, l2=1.97e-16),
    'c128/fft1_cols_fwd/64': dict(linf=2.35e-16, l2=1.56e-16),
    'c128/fft1_cols_fwd/7': dict(linf=2.73e-16, l2=2.06e-16),
    'c128/fft1_cols_fwd/8': dict(linf=1.45e-16, l2=9.90e-17),
    'c128/fft1_cols_fwd/8192': dict(linf=2.67e-16, l2=2.44e-16),
    'c128/fft1_cols_fwd/97': dict(linf=4.94e-16, l2=4.24e-16),
    'c128/fft1_cols_inv/1': dict(linf=0.0, l2=0.0),
    'c128/fft1_cols_inv/1000': dict(linf=6.39e-16, l2=5.65e-16),
    'c128/fft1_cols_inv/1023': dict(linf=6.57e-16, l2=5.49e-16),
    'c128/fft1_cols_inv/1024': dict(linf=2.77e-16, l2=2.10e-16),
    'c128/fft1_cols_inv/1025': dict(linf=5.61e-16, l2=5.00e-16),
    'c128/fft1_cols_inv/128': dict(linf=2.06e-16, l2=1.79e-16),
    'c128/fft1_cols_inv/16': dict(linf=1.71e-16, l2=1.27e-16),
    'c128/fft1_cols_inv/2': dict(linf=1.07e-16, l2=9.23e-17),
    'c128/fft1_cols_inv/2047': dict(linf=5.82e-16, l2=5.77e-16),
    'c128/fft1_cols_inv/2048': dict(linf=3.18e-16, l2=2.26e-16),
    'c128/fft1_cols_inv/255': dict(linf=6.13e-16, l2=4.99e-16),
    'c128/fft1_cols_inv/256': dict(linf=2.40e-16, l2=1.84e-16),
    'c128/fft1_cols_inv/257': dict(linf=5.50e-16, l2=4.52e-16),
    'c128/fft1_cols_inv/3': dict(linf=2.70e-16, l2=1.82e-16),
    'c128/fft1_cols_inv/32': dict(linf=1.88e-16, l2=1.37e-16),
    'c128/fft1_cols_inv/4': dict(linf=1.10e-16, l2=7.96e-17),
    'c128/fft1_cols_inv/4093': dict(linf=6.20e-16, l2=6.33e-16),
    'c128/fft1_cols_inv/4095': dict(linf=6.57e-16, l2=6.28e-16),
    'c128/fft1_cols_inv/4096': dict(linf=2.70e-16, l2=2.33e-16),
    'c128/fft1_cols_inv/5': dict(linf=2.92e-16, l2=2.45e-16),
    'c128/fft1_cols_inv/512': dict(linf=2.69e-16, l2=1.97e-16),
    'c128/fft1_cols_inv/64': dict(linf=2.35e-16, l2=1.56e-16),
    'c128/fft1_cols_inv/7': dict(linf=2.33e-16, l2=2.29e-16),
    'c128/fft1_cols_inv/8': dict(linf=1.45e-16, l2=9.90e-17),
    'c128/fft1_cols_inv/8192': dict(linf=2.67e-16, l2=2.44e-16),
    'c128/fft1_cols_inv/97': dict(linf=4.64e-16, l2=4.09e-16),
    'c128/fft1_pad_truncate_cols/1000_1007': dict(linf=5.76e-16, l2=5.59e-16),
    'c128/fft1_pad_truncate_cols/1000_995': dict(linf=5.67e-16, l2=5.49e-16),
    'c128/fft1_pad_truncate_cols/2047_2100': dict(linf=5.88e-16, l2=6.06e-16),
    'c128/fft1_pad_truncate_cols/512_300': dict(linf=2.77e-16, l2=1.90e-16),
    'c128/fft1_pad_truncate_cols/512_700': dict(linf=2.27e-16, l2=1.99e-16),
    'c128/fft1_pad_truncate_cols/97_1': dict(linf=1.17e-15, l2=3.77e-16),
    'c128/fft1_pad_truncate_rows/1000_1007': dict(linf=5.87e-16, l2=5.49e-16),
    'c128/fft1_pad_truncate_rows/1000_995': dict(linf=5.02e-16, l2=5.57e-16),
    'c128/fft1_pad_truncate_rows/2047_2100': dict(linf=6.75e-16, l2=6.10e-16),
    'c128/fft1_pad_truncate_rows/512_300': dict(linf=2.39e-16, l2=1.95e-16),
    'c128/fft1_pad_truncate_rows/512_700': dict(linf=2.27e-16, l2=1.99e-16),
    'c128/fft1_pad_truncate_rows/97_1': dict(linf=1.17e-15, l2=3.77e-16),
    'c128/fft1_rows_fwd/1': dict(linf=0.0, l2=0.0),
    'c128/fft1_rows_fwd/1000': dict(linf=6.36e-16, l2=5.57e-16),
    'c128/fft1_rows_fwd/1023': dict(linf=6.85e-16, l2=5.62e-16),
    'c128/fft1_rows_fwd/1024': dict(linf=2.38e-16, l2=2.10e-16),
    'c128/fft1_rows_fwd/1025': dict(linf=6.26e-16, l2=5.04e-16),
    'c128/fft1_rows_fwd/128': dict(linf=2.38e-16, l2=1.79e-16),
    'c128/fft1_rows_fwd/16': dict(linf=1.92e-16, l2=1.27e-16),
    'c128/fft1_rows_fwd/2': dict(linf=1.07e-16, l2=9.23e-17),
    'c128/fft1_rows_fwd/2047': dict(linf=7.19e-16, l2=6.09e-16),
    'c128/fft1_rows_fwd/2048': dict(linf=3.18e-16, l2=2.26e-16),
    'c128/fft1_rows_fwd/255': dict(linf=5.97e-16, l2=4.88e-16),
    'c128/fft1_rows_fwd/256': dict(linf=2.36e-16, l2=1.84e-16),
    'c128/fft1_rows_fwd/257': dict(linf=4.85e-16, l2=4.40e-16),
    'c128/fft1_rows_fwd/3': dict(linf=2.50e-16, l2=1.66e-16),
    'c128/fft1_rows_fwd/32': dict(linf=2.03e-16, l2=1.39e-16),
    'c128/fft1_rows_fwd/4': dict(linf=1.02e-16, l2=7.21e-17),
    'c128/fft1_rows_fwd/4093': dict(linf=7.50e-16, l2=6.40e-16),
    'c128/fft1_rows_fwd/4095': dict(linf=6.59e-16, l2=6.43e-16),
    'c128/fft1_rows_fwd/4096': dict(linf=2.70e-16, l2=2.32e-16),
    'c128/fft1_rows_fwd/5': dict(linf=2.51e-16, l2=2.97e-16),
    'c128/fft1_rows_fwd/512': dict(linf=2.69e-16, l2=1.97e-16),
    'c128/fft1_rows_fwd/64': dict(linf=2.10e-16, l2=1.56e-16),
    'c128/fft1_rows_fwd/7': dict(linf=2.83e-16, l2=2.03e-16),
    'c128/fft1_rows_fwd/8': dict(linf=1.65e-16, l2=9.77e-17),
    'c128/fft1_rows_fwd/8192': dict(linf=2.71e-16, l2=2.44e-16),
    'c128/fft1_rows_fwd/97': dict(linf=4.40e-16, l2=4.28e-16),
    'c128/fft1_rows_inv/1': dict(linf=0.0, l2=0.0),
    'c128/fft1_rows_inv/1000': dict(linf=6.39e-16, l2=5.65e-16),
    'c128/fft1_rows_inv/1023': dict(linf=6.57e-16, l2=5.50e-16),
    'c128/fft1_rows_inv/1024': dict(linf=2.38e-16, l2=2.10e-16),
    'c128/fft1_rows_inv/1025': dict(linf=6.80e-16, l2=4.99e-16),
    'c128/fft1_rows_inv/128': dict(linf=2.38e-16, l2=1.79e-16),
    'c128/fft1_rows_inv/16': dict(linf=1.92e-16, l2=1.27e-16),
    'c128/fft1_rows_inv/2': dict(linf=1.07e-16, l2=9.23e-17),
    'c128/fft1_rows_inv/2047': dict(linf=5.68e-16, l2=5.77e-16),
    'c128/fft1_rows_inv/2048': dict(linf=3.18e-16, l2=2.26e-16),
    'c128/fft1_rows_inv/255': dict(linf=6.13e-16, l2=4.99e-16),
    'c128/fft1_rows_inv/256': dict(linf=2.36e-16, l2=1.84e-16),
    'c128/fft1_rows_inv/257': dict(linf=5.50e-16, l2=4.52e-16),
    'c128/fft1_rows_inv/3': dict(linf=3.36e-16, l2=1.88e-16),
    'c128/fft1_rows_inv/32': dict(linf=2.03e-16, l2=1.39e-16),
    'c128/fft1_rows_inv/4': dict(linf=1.02e-16, l2=7.21e-17),
    'c128/fft1_rows_inv/4093': dict(linf=6.20e-16, l2=6.36e-16),
    'c128/fft1_rows_inv/4095': dict(linf=7.61e-16, l2=6.28e-16),
    'c128/fft1_rows_inv/4096': dict(linf=2.70e-16, l2=2.32e-16),
    'c128/fft1_rows_inv/5': dict(linf=3.79e-16, l2=2.45e-16),
    'c128/fft1_rows_inv/512': dict(linf=2.69e-16, l2=1.97e-16),
    'c128/fft1_rows_inv/64': dict(linf=2.10e-16, l2=1.56e-16),
    'c128/fft1_rows_inv/7': dict(linf=2.82e-16, l2=2.22e-16),
    'c128/fft1_rows_inv/8': dict(linf=1.65e-16, l2=9.77e-17),
    'c128/fft1_rows_inv/8192': dict(linf=2.71e-16, l2=2.44e-16),
    'c128/fft1_rows_inv/97': dict(linf=5.07e-16, l2=4.09e-16),
    'c128/fft2_accumulate': dict(linf=7.99e-16, l2=5.87e-16),
    'c128/fft2_batch_per_field_real': dict(linf=8.15e-16, l2=7.58e-16),
    'c128/fft2_batch_shared_u8': dict(linf=8.19e-16, l2=7.55e-16),
    'c128/fft2_fwd/100x101_100x101': dict(linf=7.76e-16, l2=7.05e-16),
    'c128/fft2_fwd/1x300_5x333': dict(linf=6.08e-16, l2=4.96e-16),
    'c128/fft2_fwd/200x7_256x9': dict(linf=3.06e-16, l2=2.90e-16),
    'c128/fft2_fwd/255x200_383x400': dict(linf=8.96e-16, l2=7.81e-16),
    'c128/fft2_fwd/256x255_512x511': dict(linf=6.11e-16, l2=5.79e-16),
    'c128/fft2_fwd/64x64_97x128': dict(linf=5.84e-16, l2=4.64e-16),
    'c128/fft2_intensity': dict(linf=7.75e-16, l2=5.85e-16),
    'c128/fft2_inv/100x101_100x101': dict(linf=6.73e-16, l2=6.65e-16),
    'c128/fft2_inv/1x300_5x333': dict(linf=5.27e-16, l2=4.74e-16),
    'c128/fft2_inv/200x7_256x9': dict(linf=3.14e-16, l2=2.79e-16),
    'c128/fft2_inv/255x200_383x400': dict(linf=9.25e-16, l2=8.00e-16),
    'c128/fft2_inv/256x255_512x511': dict(linf=6.79e-16, l2=5.37e-16),
    'c128/fft2_inv/64x64_97x128': dict(linf=5.39e-16, l2=4.42e-16),
    'c128/fft2_opd_amp_none': dict(linf=7.02e-16, l2=7.35e-16),
    'c128/fft2_opd_amp_real': dict(linf=7.24e-16, l2=7.38e-16),
    'c128/fft2_opd_amp_u8': dict(linf=7.64e-16, l2=7.35e-16),
    'c128/fft2_real_input': dict(linf=8.82e-16, l2=7.31e-16),
    'c128/focus/impulses/1000_q1.5': dict(linf=1.69e-15, l2=8.65e-16),
    'c128/focus/impulses/1000_q2': dict(linf=2.13e-15, l2=9.34e-16),
    'c128/focus/impulses/1000_q3': dict(linf=2.12e-15, l2=9.43e-16),
    'c128/focus/impulses/1023_q1.5': dict(linf=1.82e-15, l2=8.60e-16),
    'c128/focus/impulses/1023_q2': dict(linf=2.20e-15, l2=9.59e-16),
    'c128/focus/impulses/1023_q3': dict(linf=2.09e-15, l2=9.50e-16),
    'c128/focus/random/1000_q1': dict(linf=8.88e-16, l2=8.97e-16),
    'c128/focus/random/1023_q1': dict(linf=1.11e-15, l2=9.09e-16),
    'c128/focus/random/255_q1': dict(linf=8.40e-16, l2=7.41e-16),
    'c128/focus/random/255_q1.5': dict(linf=8.49e-16, l2=7.54e-16),
    'c128/focus/random/255_q2': dict(linf=8.42e-16, l2=8.38e-16),
    'c128/focus/random/255_q3': dict(linf=8.80e-16, l2=8.28e-16),
    'c128/focus/random/256_q1': dict(linf=3.76e-16, l2=2.63e-16),
    'c128/focus/random/256_q1.5': dict(linf=7.50e-16, l2=7.16e-16),
    'c128/focus/random/256_q2': dict(linf=3.18e-16, l2=2.74e-16),
    'c128/focus/random/256_q3': dict(linf=7.85e-16, l2=7.73e-16),
    'c128/focus/random/64_q1': dict(linf=2.04e-16, l2=2.17e-16),
    'c128/focus/random/64_q1.5': dict(linf=7.22e-16, l2=6.15e-16),
    'c128/focus/random/64_q2': dict(linf=2.99e-16, l2=2.31e-16),
    'c128/focus/random/64_q3': dict(linf=7.18e-16, l2=6.68e-16),
    'c128/focus_adjoint/impulses/1000_q1.5': dict(linf=1.70e-15, l2=8.95e-16),
    'c128/focus_adjoint/impulses/1000_q2': dict(linf=1.83e-15, l2=9.93e-16),
    'c128/focus_adjoint/impulses/1000_q3': dict(linf=1.69e-15, l2=9.86e-16),
    'c128/focus_adjoint/impulses/1023_q1.5': dict(linf=1.54e-15, l2=9.63e-16),
    'c128/focus_adjoint/impulses/1023_q2': dict(linf=1.71e-15, l2=9.78e-16),
    'c128/focus_adjoint/impulses/1023_q3': dict(linf=1.64e-15, l2=9.76e-16),
    'c128/focus_adjoint/random/1000_q1': dict(linf=9.68e-16, l2=9.01e-16),
    'c128/focus_adjoint/random/1023_q1': dict(linf=9.15e-16, l2=8.85e-16),
    'c128/focus_adjoint/random/255_q1': dict(linf=8.17e-16, l2=7.97e-16),
    'c128/focus_adjoint/random/255_q1.5': dict(linf=7.96e-16, l2=8.02e-16),
    'c128/focus_adjoint/random/255_q2': dict(linf=9.23e-16, l2=8.03e-16),
    'c128/focus_adjoint/random/255_q3': dict(linf=8.01e-16, l2=8.32e-16),
    'c128/focus_adjoint/random/256_q1': dict(linf=3.44e-16, l2=2.63e-16),
    'c128/focus_adjoint/random/256_q1.5': dict(linf=8.33e-16, l2=7.83e-16),
    'c128/focus_adjoint/random/256_q2': dict(linf=3.11e-16, l2=2.83e-16),
    'c128/focus_adjoint/random/256_q3': dict(linf=8.89e-16, l2=8.17e-16),
    'c128/focus_adjoint/random/64_q1': dict(linf=2.02e-16, l2=2.14e-16),
    'c128/focus_adjoint/random/64_q1.5': dict(linf=7.37e-16, l2=6.20e-16),
    'c128/focus_adjoint/random/64_q2': dict(linf=2.77e-16, l2=2.38e-16),
    'c128/focus_adjoint/random/64_q3': dict(linf=6.43e-16, l2=6.74e-16),
    'c128/focus_intensity/255_q2': dict(linf=9.03e-16, l2=6.60e-16),
    'c128/focus_intensity/256_q1.5': dict(linf=6.58e-16, l2=5.71e-16),
    'c128/focus_intensity/500_q2': dict(linf=1.03e-15, l2=7.55e-16),
    'c128/focus_intensity_accumulate/255_q2': dict(linf=8.69e-16, l2=2.31e-16),
    'c128/focus_intensity_accumulate/256_q1.5': dict(linf=5.65e-16, l2=2.89e-16),
    'c128/focus_intensity_accumulate/500_q2': dict(linf=8.31e-16, l2=2.65e-16),
    'c128/polychromatic_psf_czt/128_64': dict(linf=1.66e-15, l2=2.69e-15),
    'c128/psf_from_amp_and_phase/255_q2': dict(linf=2.16e-16, l2=3.67e-16),
    'c128/psf_from_amp_and_phase/256_q1.5': dict(linf=3.40e-16, l2=3.91e-16),
    'c128/psf_from_amp_and_phase/500_q2': dict(linf=2.73e-16, l2=4.35e-16),
    'c128/unfocus/impulses/1000_q1.5': dict(linf=1.72e-15, l2=8.89e-16),
    'c128/unfocus/impulses/1000_q2': dict(linf=1.84e-15, l2=9.19e-16),
    'c128/unfocus/impulses/1000_q3': dict(linf=1.87e-15, l2=9.28e-16),
    'c128/unfocus/impulses/1023_q1.5': dict(linf=2.00e-15, l2=9.35e-16),
    'c128/unfocus/impulses/1023_q2': dict(linf=1.99e-15, l2=9.83e-16),
    'c128/unfocus/impulses/1023_q3': dict(linf=1.96e-15, l2=9.46e-16),
    'c128/unfocus/random/1000_q1': dict(linf=9.72e-16, l2=9.01e-16),
    'c128/unfocus/random/1023_q1': dict(linf=9.74e-16, l2=8.85e-16),
    'c128/unfocus/random/255_q1': dict(linf=9.15e-16, l2=7.96e-16),
    'c128/unfocus/random/255_q1.5': dict(linf=8.64e-16, l2=7.95e-16),
    'c128/unfocus/random/255_q2': dict(linf=8.62e-16, l2=8.00e-16),
    'c128/unfocus/random/255_q3': dict(linf=8.40e-16, l2=8.25e-16),
    'c128/unfocus/random/256_q1': dict(linf=3.76e-16, l2=2.63e-16),
    'c128/unfocus/random/256_q1.5': dict(linf=7.34e-16, l2=7.77e-16),
    'c128/unfocus/random/256_q2': dict(linf=3.18e-16, l2=2.74e-16),
    'c128/unfocus/random/256_q3': dict(linf=8.24e-16, l2=8.10e-16),
    'c128/unfocus/random/64_q1': dict(linf=2.04e-16, l2=2.17e-16),
    'c128/unfocus/random/64_q1.5': dict(linf=5.90e-16, l2=6.23e-16),
    'c128/unfocus/random/64_q2': dict(linf=2.99e-16, l2=2.31e-16),
    'c128/unfocus/random/64_q3': dict(linf=6.96e-16, l2=6.69e-16),
    'c128/unfocus_adjoint/impulses/1000_q1.5': dict(linf=1.62e-15, l2=8.92e-16),
    'c128/unfocus_adjoint/impulses/1000_q2': dict(linf=1.87e-15, l2=9.95e-16),
    'c128/unfocus_adjoint/impulses/1000_q3': dict(linf=1.63e-15, l2=9.66e-16),
    'c128/unfocus_adjoint/impulses/1023_q1.5': dict(linf=1.79e-15, l2=9.19e-16),
    'c128/unfocus_adjoint/impulses/1023_q2': dict(linf=2.08e-15, l2=1.05e-15),
    'c128/unfocus_adjoint/impulses/1023_q3': dict(linf=1.78e-15, l2=1.02e-15),
    'c128/unfocus_adjoint/random/1000_q1': dict(linf=9.09e-16, l2=8.96e-16),
    'c128/unfocus_adjoint/random/1023_q1': dict(linf=9.24e-16, l2=9.08e-16),
    'c128/unfocus_adjoint/random/255_q1': dict(linf=6.92e-16, l2=7.39e-16),
    'c128/unfocus_adjoint/random/255_q1.5': dict(linf=8.26e-16, l2=7.62e-16),
    'c128/unfocus_adjoint/random/255_q2': dict(linf=8.82e-16, l2=8.38e-16),
    'c128/unfocus_adjoint/random/255_q3': dict(linf=7.80e-16, l2=8.37e-16),
    'c128/unfocus_adjoint/random/256_q1': dict(linf=3.44e-16, l2=2.63e-16),
    'c128/unfocus_adjoint/random/256_q1.5': dict(linf=7.54e-16, l2=7.16e-16),
    'c128/unfocus_adjoint/random/256_q2': dict(linf=3.11e-16, l2=2.83e-16),
    'c128/unfocus_adjoint/random/256_q3': dict(linf=8.31e-16, l2=7.79e-16),
    'c128/unfocus_adjoint/random/64_q1': dict(linf=2.02e-16, l2=2.14e-16),
    'c128/unfocus_adjoint/random/64_q1.5': dict(linf=6.41e-16, l2=6.21e-16),
    'c128/unfocus_adjoint/random/64_q2': dict(linf=2.77e-16, l2=2.37e-16),
    'c128/unfocus_adjoint/random/64_q3': dict(linf=6.77e-16, l2=6.69e-16),
    'c64/after_refusal_cols/1000': dict(linf=2.02e-7, l2=1.87e-7),
    'c64/after_refusal_rows/1000': dict(linf=2.13e-7, l2=1.88e-7),
    'c64/as_matrix/1000x1000': dict(linf=5.33e-7, l2=4.40e-7),
    'c64/as_matrix/383x300': dict(linf=4.35e-7, l2=3.70e-7),
    'c64/as_screen/1000x1000': dict(linf=4.35e-7, l2=4.44e-7),
    'c64/as_screen/383x300': dict(linf=3.97e-7, l2=3.73e-7),
    'c64/as_vectors/1000x1000': dict(linf=4.09e-7, l2=4.43e-7),
    'c64/as_vectors/383x300': dict(linf=4.17e-7, l2=3.73e-7),
    'c64/axis_dft_cols/1000': dict(linf=2.90e-7, l2=2.00e-7),
    'c64/axis_dft_cols/256': dict(linf=1.85e-7, l2=1.32e-7),
    'c64/axis_dft_cols/97': dict(linf=2.77e-7, l2=1.73e-7),
    'c64/axis_dft_rows/1000': dict(linf=3.72e-7, l2=2.07e-7),
    'c64/axis_dft_rows/256': dict(linf=1.71e-7, l2=1.30e-7),
    'c64/axis_dft_rows/97': dict(linf=2.43e-7, l2=1.68e-7),
    'c64/czt/128': dict(linf=2.26e-7, l2=1.49e-7),
    'c64/czt/16': dict(linf=1.13e-7, l2=9.81e-8),
    'c64/czt/16384': dict(linf=2.62e-7, l2=2.08e-7),
    'c64/czt/256': dict(linf=2.47e-7, l2=1.59e-7),
    'c64/czt/32': dict(linf=1.82e-7, l2=1.35e-7),
    'c64/czt/512': dict(linf=2.08e-7, l2=1.66e-7),
    'c64/czt/64': dict(linf=1.72e-7, l2=1.44e-7),
    'c64/czt/8192': dict(linf=2.14e-7, l2=1.98e-7),
    'c64/czt_accumulate/128': dict(linf=3.15e-7, l2=2.09e-7),
    'c64/czt_accumulate/16': dict(linf=1.20e-7, l2=8.92e-8),
    'c64/czt_accumulate/16384': dict(linf=3.53e-7, l2=2.57e-7),
    'c64/czt_accumulate/256': dict(linf=3.96e-7, l2=2.05e-7),
    'c64/czt_accumulate/32': dict(linf=3.49e-7, l2=1.96e-7),
    'c64/czt_accumulate/512': dict(linf=3.00e-7, l2=2.13e-7),
    'c64/czt_accumulate/64': dict(linf=2.71e-7, l2=1.96e-7),
    'c64/czt_accumulate/8192': dict(linf=3.33e-7, l2=2.50e-7),
    'c64/czt_adjoint/128': dict(linf=1.89e-7, l2=1.48e-7),
    'c64/czt_adjoint/16': dict(linf=1.13e-7, l2=1.13e-7),
    'c64/czt_adjoint/16384': dict(linf=2.65e-7, l2=2.08e-7),
    'c64/czt_adjoint/256': dict(linf=2.27e-7, l2=1.60e-7),
    'c64/czt_adjoint/32': dict(linf=1.54e-7, l2=1.22e-7),
    'c64/czt_adjoint/512': dict(linf=2.13e-7, l2=1.64e-7),
    'c64/czt_adjoint/64': dict(linf=1.74e-7, l2=1.42e-7),
    'c64/czt_adjoint/8192': dict(linf=2.43e-7, l2=2.04e-7),
    'c64/czt_intensity/128': dict(linf=3.13e-7, l2=2.11e-7),
    'c64/czt_intensity/16': dict(linf=1.19e-7, l2=1.07e-7),
    'c64/czt_intensity/16384': dict(linf=3.36e-7, l2=2.56e-7),
    'c64/czt_intensity/256': dict(linf=3.95e-7, l2=2.06e-7),
    'c64/czt_intensity/32': dict(linf=3.40e-7, l2=2.15e-7),
    'c64/czt_intensity/512': dict(linf=2.97e-7, l2=2.13e-7),
    'c64/czt_intensity/64': dict(linf=2.75e-7, l2=2.02e-7),
    'c64/czt_intensity/8192': dict(linf=3.40e-7, l2=2.49e-7),
    'c64/edge_accepted_cols/16384': dict(linf=1.70e-7, l2=1.38e-7),
    'c64/edge_accepted_cols/8191': dict(linf=2.28e-7, l2=2.11e-7),
    'c64/edge_accepted_rows/16384': dict(linf=1.61e-7, l2=1.39e-7),
    'c64/edge_accepted_rows/8191': dict(linf=2.13e-7, l2=2.11e-7),
    'c64/fft1_cols_fwd/1': dict(linf=0.0, l2=0.0),
    'c64/fft1_cols_fwd/1000': dict(linf=2.20e-7, l2=1.88e-7),
    'c64/fft1_cols_fwd/1023': dict(linf=2.60e-7, l2=1.88e-7),
    'c64/fft1_cols_fwd/1025': dict(linf=1.82e-7, l2=1.54e-7),
    'c64/fft1_cols_fwd/128': dict(linf=1.28e-7, l2=9.43e-8),
    'c64/fft1_cols_fwd/16': dict(linf=9.34e-8, l2=6.34e-8),
    'c64/fft1_cols_fwd/16384': dict(linf=1.74e-7, l2=1.39e-7),
    'c64/fft1_cols_fwd/2': dict(linf=4.11e-8, l2=2.75e-8),
    'c64/fft1_cols_fwd/2047': dict(linf=2.66e-7, l2=1.97e-7),
    'c64/fft1_cols_fwd/255': dict(linf=2.18e-7, l2=1.75e-7),
    'c64/fft1_cols_fwd/256': dict(linf=1.32e-7, l2=1.01e-7),
    'c64/fft1_cols_fwd/257': dict(linf=2.00e-7, l2=1.45e-7),
    'c64/fft1_cols_fwd/3': dict(linf=1.07e-7, l2=8.56e-8),
    'c64/fft1_cols_fwd/32': dict(linf=1.25e-7, l2=7.68e-8),
    'c64/fft1_cols_fwd/4': dict(linf=5.44e-8, l2=3.90e-8),
    'c64/fft1_cols_fwd/4093': dict(linf=2.21e-7, l2=2.05e-7),
    'c64/fft1_cols_fwd/4095': dict(linf=3.27e-7, l2=2.05e-7),
    'c64/fft1_cols_fwd/5': dict(linf=1.38e-7, l2=9.49e-8),
    'c64/fft1_cols_fwd/512': dict(linf=1.67e-7, l2=1.09e-7),
    'c64/fft1_cols_fwd/64': dict(linf=1.31e-7, l2=8.59e-8),
    'c64/fft1_cols_fwd/7': dict(linf=1.74e-7, l2=1.02e-7),
    'c64/fft1_cols_fwd/8': dict(linf=1.22e-7, l2=7.11e-8),
    'c64/fft1_cols_fwd/8191': dict(linf=2.43e-7, l2=2.12e-7),
    'c64/fft1_cols_fwd/8192': dict(linf=1.54e-7, l2=1.34e-7),
    'c64/fft1_cols_fwd/97': dict(linf=2.00e-7, l2=1.48e-7),
    'c64/fft1_cols_inv/1': dict(linf=0.0, l2=0.0),
    'c64/fft1_cols_inv/1000': dict(linf=1.98e-7, l2=1.81e-7),
    'c64/fft1_cols_inv/1023': dict(linf=2.28e-7, l2=1.91e-7),
    'c64/fft1_cols_inv/1025': dict(linf=2.21e-7, l2=1.54e-7),
    'c64/fft1_cols_inv/128': dict(linf=1.28e-7, l2=9.43e-8),
    'c64/fft1_cols_inv/16': dict(linf=9.34e-8, l2=6.34e-8),
    'c64/fft1_cols_inv/16384': dict(linf=1.74e-7, l2=1.39e-7),
    'c64/fft1_cols_inv/2': dict(linf=4.11e-8, l2=2.75e-8),
    'c64/fft1_cols_inv/2047': dict(linf=2.57e-7, l2=2.01e-7),
    'c64/fft1_cols_inv/255': dict(linf=1.96e-7, l2=1.63e-7),
    'c64/fft1_cols_inv/256': dict(linf=1.32e-7, l2=1.01e-7),
    'c64/fft1_cols_inv/257': dict(linf=2.12e-7, l2=1.46e-7),
    'c64/fft1_cols_inv/3': dict(linf=1.45e-7, l2=7.56e-8),
    'c64/fft1_cols_inv/32': dict(linf=1.25e-7, l2=7.68e-8),
    'c64/fft1_cols_inv/4': dict(linf=5.44e-8, l2=3.90e-8),
    'c64/fft1_cols_inv/4093': dict(linf=2.06e-7, l2=1.95e-7),
    'c64/fft1_cols_inv/4095': dict(linf=2.15e-7, l2=1.95e-7),
    'c64/fft1_cols_inv/5': dict(linf=1.19e-7, l2=9.19e-8),
    'c64/fft1_cols_inv/512': dict(linf=1.67e-7, l2=1.09e-7),
    'c64/fft1_cols_inv/64': dict(linf=1.31e-7, l2=8.59e-8),
    'c64/fft1_cols_inv/7': dict(linf=1.96e-7, l2=1.16e-7),
    'c64/fft1_cols_inv/8': dict(linf=1.22e-7, l2=7.11e-8),
    'c64/fft1_cols_inv/8191': dict(linf=2.57e-7, l2=2.20e-7),
    'c64/fft1_cols_inv/8192': dict(linf=1.54e-7, l2=1.34e-7),
    'c64/fft1_cols_inv/97': dict(linf=2.51e-7, l2=1.76e-7),
    'c64/fft1_pad_truncate_cols/1000_1007': dict(linf=1.99e-7, l2=1.86e-7),
    'c64/fft1_pad_truncate_cols/1000_995': dict(linf=2.48e-7, l2=1.90e-7),
    'c64/fft1_pad_truncate_cols/2047_2100': dict(linf=2.12e-7, l2=1.97e-7),
    'c64/fft1_pad_truncate_cols/512_300': dict(linf=1.57e-7, l2=1.05e-7),
    'c64/fft1_pad_truncate_cols/512_700': dict(linf=9.63e-8, l2=1.07e-7),
    'c64/fft1_pad_truncate_cols/97_1': dict(linf=2.35e-7, l2=1.12e-7),
    'c64/fft1_pad_truncate_rows/1000_1007': dict(linf=2.33e-7, l2=1.87e-7),
    'c64/fft1_pad_truncate_rows/1000_995': dict(linf=1.99e-7, l2=1.88e-7),
    'c64/fft1_pad_truncate_rows/2047_2100': dict(linf=1.97e-7, l2=1.97e-7),
    'c64/fft1_pad_truncate_rows/512_300': dict(linf=1.04e-7, l2=1.05e-7),
    'c64/fft1_pad_truncate_rows/512_700': dict(linf=1.30e-7, l2=1.10e-7),
    'c64/fft1_pad_truncate_rows/97_1': dict(linf=2.35e-7, l2=1.12e-7),
    'c64/fft1_rows_fwd/1': dict(linf=0.0, l2=0.0),
    'c64/fft1_rows_fwd/1000': dict(linf=2.50e-7, l2=1.88e-7),
    'c64/fft1_rows_fwd/1023': dict(linf=2.60e-7, l2=1.88e-7),
    'c64/fft1_rows_fwd/1025': dict(linf=2.11e-7, l2=1.52e-7),
    'c64/fft1_rows_fwd/128': dict(linf=1.14e-7, l2=9.41e-8),
    'c64/fft1_rows_fwd/16': dict(linf=1.02e-7, l2=6.38e-8),
    'c64/fft1_rows_fwd/16384': dict(linf=1.94e-7, l2=1.39e-7),
    'c64/fft1_rows_fwd/2': dict(linf=3.06e-8, l2=2.78e-8),
    'c64/fft1_rows_fwd/2047': dict(linf=2.66e-7, l2=1.96e-7),
    'c64/fft1_rows_fwd/255': dict(linf=2.18e-7, l2=1.74e-7),
    'c64/fft1_rows_fwd/256': dict(linf=1.49e-7, l2=1.02e-7),
    'c64/fft1_rows_fwd/257': dict(linf=2.09e-7, l2=1.45e-7),
    'c64/fft1_rows_fwd/3': dict(linf=1.07e-7, l2=8.56e-8),
    'c64/fft1_rows_fwd/32': dict(linf=1.12e-7, l2=7.73e-8),
    'c64/fft1_rows_fwd/4': dict(linf=7.19e-8, l2=4.06e-8),
    'c64/fft1_rows_fwd/4093': dict(linf=2.23e-7, l2=2.05e-7),
    'c64/fft1_rows_fwd/4095': dict(linf=2.44e-7, l2=2.04e-7),
    'c64/fft1_rows_fwd/5': dict(linf=1.28e-7, l2=9.13e-8),
    'c64/fft1_rows_fwd/512': dict(linf=1.41e-7, l2=1.09e-7),
    'c64/fft1_rows_fwd/64': dict(linf=1.15e-7, l2=8.73e-8),
    'c64/fft1_rows_fwd/7': dict(linf=1.35e-7, l2=9.90e-8),
    'c64/fft1_rows_fwd/8': dict(linf=1.22e-7, l2=7.11e-8),
    'c64/fft1_rows_fwd/8191': dict(linf=2.49e-7, l2=2.12e-7),
    'c64/fft1_rows_fwd/8192': dict(linf=1.60e-7, l2=1.33e-7),
    'c64/fft1_rows_fwd/97': dict(linf=2.18e-7, l2=1.48e-7),
    'c64/fft1_rows_inv/1': dict(linf=0.0, l2=0.0),
    'c64/fft1_rows_inv/1000': dict(linf=2.36e-7, l2=1.81e-7),
    'c64/fft1_rows_inv/1023': dict(linf=2.48e-7, l2=1.91e-7),
    'c64/fft1_rows_inv/1025': dict(linf=2.01e-7, l2=1.55e-7),
    'c64/fft1_rows_inv/128': dict(linf=1.14e-7, l2=9.41e-8),
    'c64/fft1_rows_inv/16': dict(linf=1.02e-7, l2=6.38e-8),
    'c64/fft1_rows_inv/16384': dict(linf=1.94e-7, l2=1.39e-7),
    'c64/fft1_rows_inv/2': dict(linf=3.06e-8, l2=2.78e-8),
    'c64/fft1_rows_inv/2047': dict(linf=2.57e-7, l2=2.01e-7),
    'c64/fft1_rows_inv/255': dict(linf=2.01e-7, l2=1.64e-7),
    'c64/fft1_rows_inv/256': dict(linf=1.49e-7, l2=1.02e-7),
    'c64/fft1_rows_inv/257': dict(linf=2.22e-7, l2=1.46e-7),
    'c64/fft1_rows_inv/3': dict(linf=9.70e-8, l2=7.42e-8),
    'c64/fft1_rows_inv/32': dict(linf=1.12e-7, l2=7.73e-8),
    'c64/fft1_rows_inv/4': dict(linf=7.19e-8, l2=4.06e-8),
    'c64/fft1_rows_inv/4093': dict(linf=2.29e-7, l2=1.95e-7),
    'c64/fft1_rows_inv/4095': dict(linf=2.37e-7, l2=1.95e-7),
    'c64/fft1_rows_inv/5': dict(linf=1.41e-7, l2=9.70e-8),
    'c64/fft1_rows_inv/512': dict(linf=1.41e-7, l2=1.09e-7),
    'c64/fft1_rows_inv/64': dict(linf=1.15e-7, l2=8.73e-8),
    'c64/fft1_rows_inv/7': dict(linf=1.93e-7, l2=1.10e-7),
    'c64/fft1_rows_inv/8': dict(linf=1.22e-7, l2=7.11e-8),
    'c64/fft1_rows_inv/8191': dict(linf=2.81e-7, l2=2.18e-7),
    'c64/fft1_rows_inv/8192': dict(linf=1.60e-7, l2=1.33e-7),
    'c64/fft1_rows_inv/97': dict(linf=2.57e-7, l2=1.76e-7),
    'c64/fft2_accumulate': dict(linf=6.00e-7, l2=3.18e-7),
    'c64/fft2_batch_per_field_real': dict(linf=3.26e-7, l2=2.33e-7),
    'c64/fft2_batch_shared_u8': dict(linf=2.89e-7, l2=2.31e-7),
    'c64/fft2_fwd/100x101_100x101': dict(linf=2.54e-7, l2=2.30e-7),
    'c64/fft2_fwd/1x300_5x333': dict(linf=2.36e-7, l2=1.73e-7),
    'c64/fft2_fwd/200x7_256x9': dict(linf=1.74e-7, l2=1.59e-7),
    'c64/fft2_fwd/255x200_383x400': dict(linf=3.01e-7, l2=2.41e-7),
    'c64/fft2_fwd/256x255_512x511': dict(linf=2.40e-7, l2=2.15e-7),
    'c64/fft2_fwd/64x64_97x128': dict(linf=2.26e-7, l2=1.83e-7),
    'c64/fft2_intensity': dict(linf=6.52e-7, l2=3.17e-7),
    'c64/fft2_inv/100x101_100x101': dict(linf=2.78e-7, l2=2.29e-7),
    'c64/fft2_inv/1x300_5x333': dict(linf=2.94e-7, l2=1.78e-7),
    'c64/fft2_inv/200x7_256x9': dict(linf=1.69e-7, l2=1.57e-7),
    'c64/fft2_inv/255x200_383x400': dict(linf=3.03e-7, l2=2.41e-7),
    'c64/fft2_inv/256x255_512x511': dict(linf=2.27e-7, l2=2.15e-7),
    'c64/fft2_inv/64x64_97x128': dict(linf=2.44e-7, l2=1.83e-7),
    'c64/fft2_opd_amp_none': dict(linf=3.08e-7, l2=2.39e-7),
    'c64/fft2_opd_amp_real': dict(linf=2.94e-7, l2=2.42e-7),
    'c64/fft2_opd_amp_u8': dict(linf=2.94e-7, l2=2.39e-7),
    'c64/fft2_real_input': dict(linf=3.02e-7, l2=2.34e-7),
}


CEIL_OF = {DT_NAME[dt]: CEILING[dt] for dt in DTYPES}
# a figure's worst over its test; one test per figure name in the whole file, so that MEASURED keeps every figure (not
# the last of several)
LEDGER = Ledger(MEASURED, lambda name: CEIL_OF[name.split('/', 1)[0]], per_test=True, one_test_per_name=True)


# ---- which kernels ran ----------------------------------------------------------------------------------------------
HIT = set()          # (L, dtype, cols) of every generic launch an extended-precision-checked case made
_CODES = {}


def codes():
    """the generic pass per (L, dtype, cols) and in total, every register-engine instantiation, the focus pair"""
    if not _CODES:
        from prysm_b200 import _capi
        for dt in DTYPES:
            for L in pow2_lengths(dt) + [2 * G.max_pow2_len(dt)]:
                for cols in (0, 1):
                    _CODES[('g', L, dt, cols)] = _capi.route_code(_capi.ROUTE_AXIS_GENERIC, L, dt | cols << 1)
        _CODES['generic'] = _capi.route_code(_capi.ROUTE_AXIS_GENERIC)
        for L in TUNED:
            for flags in range(32):
                _CODES[('reg', L, flags)] = _capi.route_code(_capi.ROUTE_AXIS_REG, L, flags)
        for N in (512, 1024, 2048):
            for inv in (0, 1):
                _CODES[('focus', N, inv)] = _capi.route_code(_capi.ROUTE_FOCUS_V2, N, inv)
    return _CODES


def run(case, fn, expect, others=0):
    """fn() for its result; it must launch exactly `expect` ({(L, dtype, cols): n}) on the generic pass, nothing on
    the register engine or the focus pair, and `others` launches of other kernels"""
    res, used = routes_of(fn, codes())
    gen = {k[1:]: v for k, v in used.items() if isinstance(k, tuple) and k[0] == 'g'}
    tuned = sorted(str(k) for k in used if isinstance(k, tuple) and k[0] != 'g')
    ngen = sum(gen.values())
    LEDGER.route(gen == expect, f'{case}: generic launches {gen}, expected {expect}')
    LEDGER.route(not tuned, f'{case}: tuned kernels ran: {tuned}')
    LEDGER.route(used.get('generic', 0) == ngen, f'{case}: total generic counter {used.get("generic", 0)} != {ngen}')
    LEDGER.route(used.get('all', 0) == ngen + others, f'{case}: {used.get("all", 0)} launches, expected {ngen + others}')
    HIT.update(gen)
    return res


def add(case, dt, got, ref):
    """the whole array against its long-double reference: rel_linf and the relative L2 error"""
    got = host(got)
    assert got.shape == ref.shape, (case, got.shape, ref.shape)
    for metric, v in (('linf', G.rel_linf(got, ref)), ('l2', G.rel_l2(got, ref))):
        LEDGER.record(f'{DT_NAME[dt]}/{case}/{metric}', v)


# ---- inputs -----------------------------------------------------------------------------------------------------------
def crand(shape, seed, dt):
    return _crand(shape, seed, G.CPLX[dt])


def lines_for(n):
    """line counts: one; one that leaves a partial last CTA; one that fills several (long lines stay few)"""
    if n >= 4096:
        return (1, 3)
    if n >= 1024:
        return (1, 37)
    return (1, 37, 300)


@pytest.fixture(scope='module', autouse=True)
def precision_64(pb):
    pb.config.precision = 64
    yield


# ---- lengths, one axis ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('d', (-1, 1))
@pytest.mark.parametrize('axis', (1, 0))
@pytest.mark.parametrize('dt', DTYPES)
def test_fft1_every_length(pb, dt, axis, d):
    """fft1 at every power of two up to the shared-memory cap (complex64: those the register engine does not take)
    and at every Bluestein length, rows and columns, forward and inverse (1/n), at 1, a partial CTA and several CTAs
    of lines"""
    from prysm_b200 import _ops
    cols = int(axis == 0)
    lens = [n for n in pow2_lengths(dt) if not (dt == PB_C64 and n in TUNED)] + list(bluestein_lengths(dt))
    for n in lens:
        for nl in lines_for(n):
            shape = (nl, n) if axis == 1 else (n, nl)
            a = crand(shape, n * 7 + nl + dt, dt)
            x = dev(a)
            case = f'fft1_{ROWS_COLS[cols]}_{"inv" if d > 0 else "fwd"}/{n}'
            got = run(f'{case}x{nl}', lambda: _ops.fft1(x, axis=axis, dir=d, scale=1.0 / n if d > 0 else 1.0),
                      G.axis_launches(n, dt, cols))
            ref = G.fft_ld(a, axis=axis, inverse=d > 0) / (n if d > 0 else 1)
            add(case, dt, got, ref)
    LEDGER.done()


@pytest.mark.parametrize('axis', (1, 0))
@pytest.mark.parametrize('dt', DTYPES)
def test_fft1_pad_and_truncate(pb, dt, axis):
    """n longer than the input (zero pad) and shorter (truncation), power-of-two and Bluestein n"""
    from prysm_b200 import _ops
    cols = int(axis == 0)
    for n, m in ((1000, 995), (1000, 1007), (512, 300), (512, 700), (97, 1), (2047, 2100)):
        shape = (5, m) if axis == 1 else (m, 5)
        a = crand(shape, n + m, dt)
        x = dev(a)
        got = run(f'pad/{n}/{m}', lambda: _ops.fft1(x, n, axis=axis), G.axis_launches(n, dt, cols))
        add(f'fft1_pad_truncate_{ROWS_COLS[cols]}/{n}_{m}', dt, got, G.fft_ld(a, n, axis=axis))
    LEDGER.done()


# ---- fft2 compositions ---------------------------------------------------------------------------------------------
def fft2_launches(k, dt):
    return G.merge(G.axis_launches(k[1], dt, 0), G.axis_launches(k[0], dt, 1))


FFT2_CASES = [  # (ny, nx), (ky, kx), crop, shift
    ((255, 200), (383, 400), None, True),
    ((256, 255), (512, 511), (511, 509), True),
    ((100, 101), (100, 101), (99, 100), True),
    ((64, 64), (97, 128), (96, 127), False),
    ((1, 300), (5, 333), None, True),
    ((200, 7), (256, 9), (255, 8), True),
]


@pytest.mark.parametrize('dt', DTYPES)
def test_fft2_pad_shift_crop(pb, dt):
    """centred pad (in_off), shift_in / shift_out at odd and even k, odd and even crops, both directions"""
    from prysm_b200 import _ops
    for i, (n, k, crop, shift) in enumerate(FFT2_CASES):
        a = crand(n, 40 + i, dt)
        x = dev(a)
        for d in (-1, 1):
            case = f'fft2_{"inv" if d > 0 else "fwd"}/{n[0]}x{n[1]}_{k[0]}x{k[1]}'
            got = run(case, lambda: _ops.fft2(x, k, dir=d, shift_in=shift, shift_out=shift, crop=crop),
                      fft2_launches(k, dt))
            add(case, dt, got, G.centred_ft2_ld(a, k, inverse=d > 0, crop=crop, shift=shift))
    LEDGER.done()


@pytest.mark.parametrize('dt', DTYPES)
def test_fft2_output_and_input_kinds(pb, dt):
    """|.|^2 written and accumulated with a weight; a real input (the mtf_from_psf path); the amplitude / OPD input
    with no, a real and a u8 amplitude (phases of many turns: the exact range reduction)"""
    from prysm_b200 import _ops
    capi = _ops.capi
    n, k, crop = (255, 256), (383, 384), (381, 383)
    a = crand(n, 50, dt)
    x = dev(a)
    launches = fft2_launches(k, dt)
    ref = G.centred_ft2_ld(a, k, crop=crop)
    inten = ref.real ** 2 + ref.imag ** 2
    got = run('intensity', lambda: _ops.fft2(x, k, shift_in=True, shift_out=True, crop=crop,
                                               out_kind=capi.OUT_INTENSITY), launches)
    add('fft2_intensity', dt, got, inten)
    acc0 = torch.rand(crop, generator=torch.Generator(device='cuda').manual_seed(5), device='cuda', dtype=RDT[dt])
    got = run('accumulate', lambda: _ops.fft2(x, k, shift_in=True, shift_out=True, crop=crop, weight=WEIGHT,
                                                out_kind=capi.OUT_ACCUMULATE, out=acc0.clone()), launches)
    add('fft2_accumulate', dt, got, G.ld(acc0.cpu().numpy()) + WEIGHT * inten)

    r = np.random.default_rng(51).standard_normal(n).astype(NPR[dt])
    got = run('real', lambda: _ops.fft2(dev(r), k, shift_in=True, shift_out=True), launches)
    add('fft2_real_input', dt, got, G.centred_ft2_ld(r.astype(LD), k))

    rng = np.random.default_rng(52)
    opd = (300.0 * rng.standard_normal(n)).astype(NPR[dt])
    ampr = rng.uniform(0.2, 1.0, n).astype(NPR[dt])
    ampu = (rng.random(n) > 0.3)
    for name, amp in (('none', None), ('real', ampr), ('u8', ampu)):
        got = run(f'opd_{name}', lambda: _ops.fft2(None, k, dir=-1, shift_in=True, shift_out=True, crop=crop,
                                                   opd=dev(opd), amp=None if amp is None else dev(amp),
                                                   kscale=KSCALE), launches)
        add(f'fft2_opd_amp_{name}', dt, got, G.centred_ft2_ld(G.phase_field_ld(opd, KSCALE, amp), k, crop=crop))
    LEDGER.done()


# ---- public entry points at precision 64 ---------------------------------------------------------------------------
FOCUS_NS = (64, 255, 256, 1000, 1023)
FOCUS_QS = (1, 1.5, 2, 3)


def impulses(N):
    px = [(N // 2, N // 2), (0, 0), (0, N - 1), (N // 2 + 5, N // 2 - 3)]
    return px, [0.25 - 0.5j, -0.75 + 0.25j, 1.0 + 0.0j, -0.5 - 0.75j]


@pytest.mark.parametrize('Q', FOCUS_QS)
@pytest.mark.parametrize('N', FOCUS_NS)
def test_public_focus_family(pb, N, Q):
    """focus, unfocus, focus_adjoint and unfocus_adjoint at complex128: random fields where the padded side K is at
    most 1024, sums of impulses (closed form) past that"""
    P = pb.propagation
    K = math.ceil(N * Q)
    Nb = int(K // Q)
    dt = PB_C128
    fwd = fft2_launches((K, K), dt)
    if K <= 1024:
        a = crand((N, N), N + int(10 * Q), dt)
        g = crand((K, K), K + 1, dt)
        ref_f = lambda inv: G.centred_ft2_ld(a, (K, K), inverse=inv) / K
        ref_a = lambda inv: G.centred_ft2_ld(g, (K, K), inverse=inv, crop=(Nb, Nb)) / K
        tag = 'random'
    else:
        px, vals = impulses(N)
        pxa, valsa = impulses(K)
        a = np.zeros((N, N), dtype=np.complex128)
        g = np.zeros((K, K), dtype=np.complex128)
        for p, v in zip(px, vals):
            a[p] += v
        for p, v in zip(pxa, valsa):
            g[p] += v
        ref_f = lambda inv: G.impulse_centred_ft2((N, N), (K, K), px, vals, inverse=inv) / K
        ref_a = lambda inv: G.impulse_centred_ft2((K, K), (K, K), pxa, valsa, inverse=inv, crop=(Nb, Nb)) / K
        tag = 'impulses'
    x, y = dev(a), dev(g)
    case = f'{tag}/{N}_q{Q}'
    add(f'focus/{case}', dt, run(f'focus/{case}', lambda: P.focus(x, Q), fwd), ref_f(False))
    add(f'unfocus/{case}', dt, run(f'unfocus/{case}', lambda: P.unfocus(x, Q), fwd), ref_f(True))
    add(f'focus_adjoint/{case}', dt, run(f'focus_adjoint/{case}', lambda: P.focus_adjoint(y, Q), fwd), ref_a(True))
    add(f'unfocus_adjoint/{case}', dt, run(f'unfocus_adjoint/{case}', lambda: P.unfocus_adjoint(y, Q), fwd),
        ref_a(False))
    LEDGER.done()


@pytest.mark.parametrize('N,Q', [(255, 2), (256, 1.5), (500, 2)])
def test_public_focus_intensity_and_psf(pb, N, Q):
    """focus_intensity written and accumulated; psf_from_amp_and_phase (the OPD synthesised in the first pass)"""
    P = pb.propagation
    dt = PB_C128
    K = math.ceil(N * Q)
    fwd = fft2_launches((K, K), dt)
    a = crand((N, N), N + 3, dt)
    ref = G.centred_ft2_ld(a, (K, K)) / K
    inten = ref.real ** 2 + ref.imag ** 2
    x = dev(a)
    add(f'focus_intensity/{N}_q{Q}', dt, run('fi', lambda: P.focus_intensity(x, Q), fwd), inten)
    acc0 = torch.rand((K, K), generator=torch.Generator(device='cuda').manual_seed(N), device='cuda', dtype=torch.float64)
    got = run('fia', lambda: P.focus_intensity(x, Q, weight=WEIGHT, out=acc0.clone()), fwd)
    add(f'focus_intensity_accumulate/{N}_q{Q}', dt, got, G.ld(acc0.cpu().numpy()) + WEIGHT * inten)
    rng = np.random.default_rng(N)
    opd = 200.0 * rng.standard_normal((N, N))
    amp = rng.uniform(0.0, 1.0, (N, N))
    wvl = 0.6328
    kscale = P.phase_prefix(wvl).imag
    ref = G.centred_ft2_ld(G.phase_field_ld(opd, kscale, amp), (K, K)) / K
    got = run('psf', lambda: P.psf_from_amp_and_phase(dev(amp), dev(opd), wvl, Q), fwd)
    add(f'psf_from_amp_and_phase/{N}_q{Q}', dt, got, ref.real ** 2 + ref.imag ** 2)
    LEDGER.done()


# ---- fft2_batch, one field at a time --------------------------------------------------------------------------------
@pytest.mark.parametrize('dt', DTYPES)
def test_fft2_batch_fallback(pb, dt):
    """the per-field loop of pb_fft2_batch: OPD fields with a shared u8 amplitude and with per-field real amplitudes,
    into a padded output whose row and field pitches exceed the field (nothing written outside the windows)"""
    from prysm_b200 import _ops
    nb, n, k = 3, (200, 201), (300, 301)
    rng = np.random.default_rng(60)
    opd = (500.0 * rng.standard_normal((nb,) + n)).astype(NPR[dt])
    shared = rng.random(n) > 0.25
    per = rng.uniform(0.1, 1.0, (nb,) + n).astype(NPR[dt])
    launches = {key: nb * v for key, v in fft2_launches(k, dt).items()}
    for name, amp in (('shared_u8', shared), ('per_field_real', per)):
        big0 = torch.full((nb + 1, k[0] + 2, k[1] + 5), 7.0, dtype=TDT[dt], device='cuda')

        def fn():
            big = big0.clone()
            out = big[:nb, 1:k[0] + 1, 3:k[1] + 3]
            _ops.fft2_batch(None, k, dir=-1, scale=1.0 / 17, shift_in=True, shift_out=True, amp=dev(amp), opd=dev(opd),
                            kscale=KSCALE, out=out)
            inside = torch.zeros(big.shape, dtype=torch.bool, device='cuda')
            inside[:nb, 1:k[0] + 1, 3:k[1] + 3] = True
            LEDGER.route(torch.equal(big[~inside], big0[~inside]), f'{name}: a store outside the output windows')
            return out
        got = run(name, fn, launches)
        for b in range(nb):
            ab = amp if amp.ndim == 2 else amp[b]
            ref = G.centred_ft2_ld(G.phase_field_ld(opd[b], KSCALE, ab), k) / 17
            add(f'fft2_batch_{name}', dt, got[b], ref)
    LEDGER.done()


# ---- axis_dft: fused multipliers and output windows ---------------------------------------------------------------
@pytest.mark.parametrize('axis', (1, 0))
@pytest.mark.parametrize('dt', DTYPES)
def test_axis_dft_multipliers(pb, dt, axis):
    """pre_e / pre_b / post_e / post_b with each conj flag and a nonzero output window, power-of-two and Bluestein
    lengths (on a Bluestein axis the user's multipliers ride as pre_e2 / post_e2 next to the chirp)"""
    from prysm_b200 import _ops
    cols = int(axis == 0)
    for n in (256, 1000, 97):
        nl = 11
        m = n - 3
        a = crand((nl, m) if axis == 1 else (m, nl), n, dt)
        off, no = n // 3, n - n // 3 - 5
        pre_e, post_e = crand(n, n + 1, dt), crand(no, n + 4, dt)
        pre_b, post_b = crand(nl, n + 2, dt), crand(nl, n + 3, dt)
        f = lambda v, c: np.conj(v) if c else v   # noqa: E731
        for conj in (0, 1, 2, 4, 8, 15):          # bits: pre_e, pre_b, post_e, post_b conjugated
            pc, pbc, qc, qbc = conj & 1, (conj >> 1) & 1, (conj >> 2) & 1, (conj >> 3) & 1
            got = run(f'axis_dft/{n}/{conj}', lambda: _ops.axis_dft(
                dev(a), n, axis, dir=-1, scale=0.5, pre_e=dev(pre_e), pre_e_conj=bool(pc), pre_b=dev(pre_b),
                pre_b_conj=bool(pbc), post_e=dev(post_e), post_e_conj=bool(qc), post_b=dev(post_b),
                post_b_conj=bool(qbc), out_off=off, n_out=no), G.axis_launches(n, dt, cols))
            u = G.ld(a) if axis == 1 else G.ld(a).T
            u = u * G.ld(f(pre_e, pc))[:m] * G.ld(f(pre_b, pbc))[:, None]
            U = G.fft_ld(u, n)[:, off:off + no] * G.ld(f(post_e, qc)) * G.ld(f(post_b, qbc))[:, None] * LD(0.5)
            add(f'axis_dft_{ROWS_COLS[cols]}/{n}', dt, got, U if axis == 1 else U.T)
    LEDGER.done()


# ---- CZT, the two-pass fallback ------------------------------------------------------------------------------------
def czt_Ks(dt):
    if dt == PB_C128:
        return [1 << i for i in range(4, 14)]
    return [16, 32, 64, 128, 256, 512, 8192, 16384]


@pytest.mark.parametrize('dt', DTYPES)
def test_czt_axis(pb, dt):
    """czt_axis forward (b, H, post) and adjoint (conj post, Hadj, conj b), |.|^2 written and accumulated, rows and
    columns, against the long-double transform of the plan vectors the device built"""
    from prysm_b200 import _ops
    capi = _ops.capi
    for K in czt_Ks(dt):
        N, M = K // 2, K // 2
        plan = _ops.czt_plan(N, M, K, 0.0, 0.37 / N, -1, 0.0, -M / 2 * 0.9, 0.9, TDT[dt], 'cuda')
        bd, postd, Hd, Hadjd = plan
        b, post, H, Hadj = (G.ld(t.cpu().numpy()) for t in plan)
        nl = 3 if K >= 4096 else 9
        for axis in (1, 0):
            cols = int(axis == 0)
            two = {(K, dt, cols): 2}
            a = crand((nl, N) if axis == 1 else (N, nl), K + axis, dt)
            u = G.ld(a) if axis == 1 else G.ld(a).T
            V = G.fft_ld(G.fft_ld(u * b, K) * H, inverse=True)[:, N - 1:N - 1 + M] * post * LD(0.5) / K
            tr = (lambda z: z) if axis == 1 else (lambda z: z.T)
            got = run(f'czt/{K}', lambda: _ops.czt_axis(dev(a), K, axis, bd, Hd, postd, N - 1, M, 0.5), two)
            add(f'czt/{K}', dt, got, tr(V))
            inten = V.real ** 2 + V.imag ** 2
            got = run(f'czti/{K}', lambda: _ops.czt_axis(dev(a), K, axis, bd, Hd, postd, N - 1, M, 0.5,
                                                           out_kind=capi.OUT_INTENSITY), two)
            add(f'czt_intensity/{K}', dt, got, tr(inten))
            acc0 = torch.rand(tuple(tr(inten).shape), generator=torch.Generator(device='cuda').manual_seed(K),
                              device='cuda', dtype=RDT[dt])
            got = run(f'czta/{K}', lambda: _ops.czt_axis(dev(a), K, axis, bd, Hd, postd, N - 1, M, 0.5,
                                                           out_kind=capi.OUT_ACCUMULATE, weight=WEIGHT,
                                                           out=acc0.clone()), two)
            add(f'czt_accumulate/{K}', dt, got, G.ld(acc0.cpu().numpy()) + WEIGHT * tr(inten))
            g = crand((nl, M) if axis == 1 else (M, nl), K + 5 + axis, dt)
            w = G.ld(g) if axis == 1 else G.ld(g).T
            V = G.fft_ld(G.fft_ld(w * np.conj(post), K) * Hadj, inverse=True)[:, :N] * np.conj(b) / K
            got = run(f'czt_adj/{K}', lambda: _ops.czt_axis(dev(g), K, axis, postd, Hadjd, bd, 0, N, 1.0,
                                                              pre_conj=True, post_conj=True), two)
            add(f'czt_adjoint/{K}', dt, got, tr(V))
    LEDGER.done()


# ---- angular spectrum ------------------------------------------------------------------------------------------------
AS_CASES = {PB_C128: [((256, 256), (512, 512)), ((255, 200), (383, 300)), ((1024, 1024), (1024, 1024))],
            PB_C64: [((255, 200), (383, 300)), ((500, 500), (1000, 1000))]}


@pytest.mark.parametrize('dt', DTYPES)
def test_angular_spectrum(pb, dt):
    """the full transfer-function matrix (post_mat) and the separable vectors (post_e, post_b), plain and conjugated,
    with and without a phase screen, cropped and not"""
    from prysm_b200 import _ops
    for n, k in AS_CASES[dt]:
        ty, tx = _ops.angular_spectrum_vectors(k, 0.6328, 0.01, 25.0, TDT[dt], 'cuda')
        T = np.outer(G.ld(ty.cpu().numpy()), G.ld(tx.cpu().numpy()))
        tf = crand(k, k[0], dt)
        a = crand(n, n[0] + 1, dt)
        s = np.exp(1j * np.random.default_rng(n[1]).uniform(0, 2 * np.pi, n)).astype(G.CPLX[dt])
        x, sd = dev(a), dev(s)
        crop = (n[0] - 1, n[1] - 2)
        base = G.merge(G.axis_launches(k[1], dt, 0), G.axis_launches(k[0], dt, 1))
        launches = G.merge(base, base)

        def ref(field, TT, conj, cr):
            F = sfft.fft2(_pad(field, k))
            out = sfft.ifft2(F * (np.conj(TT) if conj else TT))
            if cr is None:
                return out
            y0, x0 = -(-(k[0] - cr[0]) // 2), -(-(k[1] - cr[1]) // 2)
            return out[y0:y0 + cr[0], x0:x0 + cr[1]]
        for conj in (False, True):
            got = run('as_vec', lambda: _ops.angular_spectrum(x, k, ty=ty, tx=tx, conj_tf=conj), launches)
            add(f'as_vectors/{k[0]}x{k[1]}', dt, got, ref(G.ld(a), T, conj, None))
            got = run('as_mat', lambda: _ops.angular_spectrum(x, k, tf=dev(tf), conj_tf=conj, crop=crop), launches)
            add(f'as_matrix/{k[0]}x{k[1]}', dt, got, ref(G.ld(a), G.ld(tf), conj, crop))
            got = run('as_screen', lambda: _ops.angular_spectrum(x, k, ty=ty, tx=tx, screen=sd, conj_screen=conj),
                      launches)
            sc = np.conj(G.ld(s)) if conj else G.ld(s)
            add(f'as_screen/{k[0]}x{k[1]}', dt, got, ref(G.ld(a) * sc, T, False, None))
    LEDGER.done()


def _pad(a, k):
    p = np.zeros(k, dtype=LD)
    oy, ox = -(-(k[0] - a.shape[0]) // 2), -(-(k[1] - a.shape[1]) // 2)
    p[oy:oy + a.shape[0], ox:ox + a.shape[1]] = a
    return p


# ---- the device-built plan vectors against their long-double closed forms ----------------------------------------------
EPS = {PB_C64: float(np.finfo(np.float32).eps), PB_C128: float(np.finfo(np.float64).eps)}
EPS64 = float(np.finfo(np.float64).eps)


def phase_err(got, turns, mag, dt, k=4):
    """|got - exp(2 pi i turns)| per element over its bound: k ulps of the result type plus k fp64 ulps of the phase
    magnitude `mag` [turns] (the phases are formed in fp64 on the device)"""
    ref = G.expi_ld(turns)
    return np.abs(G.ld(got) - ref).astype(np.float64) / (k * (EPS[dt] + 2 * np.pi * EPS64 * np.abs(mag)))


@pytest.mark.parametrize('dt', DTYPES)
def test_czt_plan_vectors(pb, dt):
    """pb_czt_plan: b, post, the kernel spectrum H = FFT_K(h) and Hadj = conj(H) exp(-2 pi i (N-1) k / K) against the
    closed forms of csrc/elementwise.cu's czt_plan_kernel, evaluated in long double from the same fp64 scalars; b and
    post within a few ulps of their phase magnitude, H and Hadj within the same per-term bound summed over the K-point
    transform"""
    from prysm_b200 import _ops
    for K, N, M, shift, alpha, sign, xc, f0, df in (
            (256, 128, 64, 0.0, 0.37 / 128, -1, 0.0, -32 * 0.9, 0.9),
            (1024, 700, 300, 0.5, 3.1e-3, 1, 0.25, -150.5 * 0.7, 0.7),
            (8192, 4096, 4096, -0.25, 1.0 / 4096, -1, -1.5, -2048.25 * 0.01, 0.01)):
        b, post, H, Hadj = (t.cpu().numpy() for t in _ops.czt_plan(N, M, K, shift, alpha, sign, xc, f0, df, TDT[dt], 'cuda'))
        half = np.longdouble(0.5) * sign * np.longdouble(alpha)
        n = np.arange(N, dtype=np.longdouble) - N // 2
        e = phase_err(b, half * n * n, half * n * n, dt)
        assert e.max() < 1, ('b', K, float(e.max()))
        m = np.arange(M)
        q = (m - M // 2).astype(np.longdouble) + np.longdouble(shift)
        fm = np.longdouble(f0) + m.astype(np.longdouble) * np.longdouble(df)
        t1, t2 = half * q * q, sign * np.longdouble(xc) * fm
        mag = np.abs(t1) + abs(xc) * (abs(f0) + m * abs(df))     # f0 + m df is rounded before the product
        e = phase_err(post, t1 + t2, mag, dt)
        assert e.max() < 1, ('post', K, float(e.max()))
        nd = N + M - 1
        d = (np.arange(nd) - (M // 2) - (-(N // 2) + N - 1)).astype(np.longdouble) + np.longdouble(shift)
        h = np.zeros(K, dtype=LD)
        h[:nd] = G.expi_ld(-half * d * d)
        Href = G.fft_ld(h)
        # one rounding per term of the sum and per radix level, plus each term's phase error
        tol = 4 * (EPS[dt] * nd * math.log2(K) + 2 * np.pi * EPS64 * float(np.sum(np.abs(half * d * d))))
        err = float(np.abs(G.ld(H) - Href).max())
        assert err < tol, ('H', K, err, tol)
        k = np.arange(K, dtype=np.int64)
        Hadj_ref = np.conj(Href) * G.ramp_ld(k, N - 1, K, -1)
        err = float(np.abs(G.ld(Hadj) - Hadj_ref).max())
        assert err < tol + 4 * EPS[dt] * float(np.abs(Href).max()), ('Hadj', K, err, tol)
        assert float(np.abs(Href).max()) > 1         # a bound far below the size of any index, sign or offset error


@pytest.mark.parametrize('dt', DTYPES)
def test_angular_spectrum_vectors(pb, dt):
    """pb_angular_spectrum_vectors: exp(-i pi wvl z k^2), k = fftfreq(n, dx), against the long-double closed form from
    the same fp64 wavelength [mm], dx and z, within a few ulps of the phase magnitude; odd and even n"""
    from prysm_b200 import _ops
    for (ky, kx), wvl, dx, z in (((512, 383), 0.6328, 0.01, 25.0), ((1024, 1000), 0.55, 0.002, 400.0)):
        ty, tx = (t.cpu().numpy() for t in _ops.angular_spectrum_vectors((ky, kx), wvl, dx, z, TDT[dt], 'cuda'))
        w = np.longdouble(wvl / 1e3)
        for n, got in ((ky, ty), (kx, tx)):
            kf = np.asarray(sfft.fftfreq(n) * n, dtype=np.longdouble) / (n * np.longdouble(dx))
            turns = -0.5 * w * np.longdouble(z) * kf * kf
            e = phase_err(got, turns, turns, dt, k=8)
            assert e.max() < 1, (n, float(e.max()))


def test_polychromatic_psf_czt(pb):
    """polychromatic_psf(kind='czt') at precision 64 (one native call over the wavelengths): the weighted sum of
    |norm Ey A Ex^T|^2 with A = amp exp(i kscale opd) and E = exp(-2 pi i f x) formed in long double from the fp64
    coordinates of each wavelength"""
    dt = PB_C128
    N, M, dx, fdx, efl = 128, 64, 10.0 / 128, 0.5, 100.0
    wvls, wts = np.array([0.5, 0.6, 0.7]), np.array([0.25, 1.0, 0.5])
    rng = np.random.default_rng(90)
    opd = 150.0 * rng.standard_normal((N, N))
    amp = rng.uniform(0.3, 1.0, (N, N))
    P = pb.propagation
    ref = np.zeros((M, M), dtype=np.longdouble)
    for w, wt in zip(wvls, wts):
        x, y, fx, fy = P.coordinates_for_focus(dx, (N, N), fdx, (M, M), w, efl, (0, 0), dtype=np.float64)
        E = lambda f, v: G.expi_ld(-np.multiply.outer(f.astype(np.longdouble), v.astype(np.longdouble)))  # noqa: E731
        A = G.phase_field_ld(opd, P.phase_prefix(w).imag, amp)
        out = np.longdouble((dx * fdx) / (w * efl)) * (E(fy, y) @ A @ E(fx, x).T)
        ref += np.longdouble(wt) * (out.real ** 2 + out.imag ** 2)
    K = 256                                       # next_fast_len(N + M - 1), one plan per wavelength for both axes
    per_wvl = {(K, dt, 0): 3, (K, dt, 1): 2}      # H = FFT_K(h), then a CZT axis of two passes each way
    got = run('polychromatic_czt', lambda: pb.polychromatic.polychromatic_psf(
        dev(amp), dev(opd), wvls, wts, dx, efl, fdx, M, kind='czt', shard=False),
        {k: v * len(wvls) for k, v in per_wvl.items()}, others=2 * len(wvls))   # the plan and phase-screen kernels
    add('polychromatic_psf_czt/128_64', dt, got, ref)
    LEDGER.done()


# ---- the shared-memory edge ----------------------------------------------------------------------------------------
@pytest.mark.parametrize('axis', (1, 0))
@pytest.mark.parametrize('dt', DTYPES)
def test_shared_memory_edge(pb, dt, axis):
    """the largest accepted power of two and Bluestein length are checked like any other; one past each raises
    B200Error naming the length, the dtype and the limits, writes nothing to a caller's `out`, and leaves the handle
    working"""
    from prysm_b200 import _ops
    cols = int(axis == 0)
    lmax = G.max_pow2_len(dt)
    for n in (lmax, lmax // 2 - 1):
        a = crand((3, n) if axis == 1 else (n, 3), n + 9, dt)
        got = run(f'edge/{n}', lambda: _ops.fft1(dev(a), axis=axis), G.axis_launches(n, dt, cols))
        add(f'edge_accepted_{ROWS_COLS[cols]}/{n}', dt, got, G.fft_ld(a, axis=axis))
    for n in (2 * lmax, lmax // 2 + 1):
        assert not G.accepts(n, dt)
        a = dev(crand((3, n) if axis == 1 else (n, 3), n, dt))
        out = torch.full(tuple(a.shape), complex(1.5, -2.5), dtype=TDT[dt], device='cuda')
        before = out.clone()
        with pytest.raises(_ops.capi.B200Error) as e:
            _ops.axis_dft(a, n, axis, out=out)
        msg = str(e.value)
        for word in (f'length {n}', 'complex64' if dt == PB_C64 else 'complex128', str(lmax), str(lmax // 2)):
            assert word in msg, (word, msg)
        torch.cuda.synchronize()
        assert torch.equal(out.view(RDT[dt]), before.view(RDT[dt])), 'a refused call wrote to `out`'
        b = crand((3, 1000) if axis == 1 else (1000, 3), 3, dt)
        got = run('after_refusal', lambda: _ops.fft1(dev(b), axis=axis), G.axis_launches(1000, dt, cols))
        add(f'after_refusal_{ROWS_COLS[cols]}/1000', dt, got, G.fft_ld(b, axis=axis))
    LEDGER.done()


def _whole_module_selected(session):
    """every test of this file (each parameter set) is in the session: not a -k, node-id or --lf selection"""
    want = 0
    for name, fn in globals().items():
        if name.startswith('test_') and callable(fn):
            n = 1
            for m in getattr(fn, 'pytestmark', []):
                if m.name == 'parametrize':
                    n *= len(m.args[1])
            want += n
    return sum(1 for it in session.items if it.module.__name__ == __name__) == want


def test_zz_every_reachable_length_was_hit(pb, request):
    """runs last: every (L, dtype, orientation) of the generic pass the Python API can reach -- every power of two up to
    the cap, both dtypes, rows and columns -- ran in a case checked above"""
    if not _whole_module_selected(request.session):
        pytest.skip('only part of this file was selected: the coverage of the whole file cannot be judged')
    want = {(L, dt, cols) for dt in DTYPES for L in pow2_lengths(dt) for cols in (0, 1)}
    assert not want - HIT, sorted(want - HIT)
    assert not HIT - want, sorted(HIT - want)


def test_zz_every_figure_has_a_measurement():
    """a figure this session reached that has no MEASURED entry is held to the bare ceiling, a bound nobody measured"""
    if os.environ.get('PB_TEST_MEASUREMENTS'):
        pytest.skip('recording figures')
    assert not LEDGER.missing(), f'no MEASURED entry (record them with PB_TEST_MEASUREMENTS): {LEDGER.missing()}'
