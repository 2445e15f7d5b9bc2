"""GPU: every route of the fused focus pair and of the register axis engine (csrc/fft_tuned.cu), held to a complex128
reference over whole output arrays.

The other focus-pipeline tests check that a field of a stack has the bits of a single call; this file checks that the
bits are right.  The reference is oracle/prysm_oracle.py in complex128 (scipy.fft, all cores) fed the exact complex64 /
float32 values the device got, computed once per (input, direction) and shared by the complex, |.|^2 and accumulated
outputs.  Sums of impulses have a closed form (`impulse_focus`: a phase ramp per impulse), so those cases use no FFT and
show an index, rotation or sign error where it is.

Every output array is compared whole, by two metrics: `rel_linf` (max|a - b| / max|b|) and the relative L2 error
||a - b|| / ||b||, which sees an error spread over the whole array that an L-inf bound of 1e-6 hides (a perturbation
smaller than the 1.5x margin, such as twiddles formed from fp32-rounded angles, still passes).  Outputs of the focus pair are also bounded per class of output row, from the layout
of DESIGN §3 / §4.1 (`row_classes`): plane 0 of the intermediate (even rows from the centre), the head of plane 1 that
stays in L2 (intermediate rows j < 4 plane1_keep<L>()) and the streamed rest of plane 1.  A stack case takes the worst
field of the stack.

Bounds are 1.5x the figures measured on an H100 (`MEASURED`, recorded with PB_TEST_MEASUREMENTS; the arithmetic is
deterministic, so the figures repeat bit for bit) and never above the north-star 1e-6.  Ranges of the measured figures,
H100 80GB HBM3 at a 400 W power limit (the staged_* cases at 700 W):

    axis angular_spectrum              linf 2.4e-07-3.3e-07, l2 2.6e-07-3.1e-07
    axis angular_spectrum_adjoint      linf 2.7e-07-3.7e-07, l2 2.7e-07-3.1e-07
    axis czt                           linf 4.0e-07-5.5e-07, l2 3.6e-07-4.0e-07
    axis czt_adjoint                   linf 4.1e-07-4.7e-07, l2 3.5e-07-4.0e-07
    axis czt_intensity                 linf 6.6e-07-6.7e-07, l2 4.9e-07-5.3e-07
    axis czt_intensity_accumulate      linf 9.6e-08-3.0e-07, l2 2.6e-08-5.9e-08
    axis fft                           linf 1.8e-07-2.4e-07, l2 1.7e-07-1.9e-07
    axis fft1_cols                     linf 1.5e-07-1.6e-07, l2 1.3e-07-1.3e-07
    axis fft2_centred_crop_odd_width   linf 2.3e-07-2.3e-07, l2 1.8e-07-1.8e-07
    axis focus                         linf 1.7e-07-1.7e-07, l2 1.7e-07-1.7e-07
    axis focus_adjoint                 linf 2.0e-07-2.4e-07, l2 1.7e-07-1.9e-07
    axis ifft                          linf 2.0e-07-2.5e-07, l2 1.7e-07-1.9e-07
    axis ifft2_rows                    linf 1.5e-07-2.3e-07, l2 1.2e-07-1.7e-07
    axis screened_free_space           linf 2.4e-07-3.5e-07, l2 2.7e-07-3.1e-07
    axis unfocus_adjoint               linf 2.0e-07-2.3e-07, l2 1.7e-07-1.9e-07
    focus pair, N = 1024               linf 1.7e-07-4.4e-07, l2 8.6e-08-2.6e-07, rows 1.7e-07-4.4e-07
    focus pair, N = 2048               linf 6.3e-08-4.9e-07, l2 9.3e-08-2.7e-07, rows 3.7e-08-4.9e-07
    focus pair, N = 512                linf 8.6e-08-4.9e-07, l2 8.8e-08-2.5e-07, rows 4.2e-08-4.9e-07
    (rows: the per-row-class figures; a centred impulse focuses exactly, figure 0)

Inputs tensor TMA cannot gather (a misaligned base, an odd row or field pitch, the fused phase-screen input) are staged
field by field into a dense aligned buffer and take the same pair; those cases are named `staged_*`.

Every case also shows that it ran the kernel it is about, from the library's per-route launch counters
(pb_route_launch_count): a focus case launches exactly the kernels of the pair of its N and direction -- two per field
-- and nothing else but one phase-screen launch per staged phase-screen field (a staging copy is not a launch); an axis
case runs the `axis_reg_kernel<L, INV, COLS, TP, RT, PM, DENSE>` instantiations it names, no other route, and nothing
outside EXPECTED.  The last test asserts that every instantiation the Python API can reach was hit by a case here.
"""
import ctypes as C
import math
import os

import numpy as np
import pytest
import scipy.fft as sfft
import torch

import prysm_oracle as O
from accuracy import Ledger, rel_l2
from conftest import rel_linf
from gpu_fixtures import pb, dev, host  # noqa: F401
from gpu_fixtures import routes_of as _routes_of

pytestmark = pytest.mark.gpu

HeNe = 0.6328
NS = (512, 1024, 2048)
NSTACK = 5                  # fields of a v2 stack: both intermediates reused, odd tail
WEIGHT = 0.375              # accumulate weight (exact in fp32)
NORTH_STAR = 1e-6

# ---- the layout of the focus intermediate (DESIGN §3, §4.1; csrc/fft_tuned.cu) ---------------------------------------
PLANE1_KEEP_BYTES = 2 << 20     # kPlane1KeepBytes
CLASSES = ('plane0', 'plane1_kept', 'plane1_streamed')


def plane1_keep(L):
    """plane1_keep<L>(): line groups (L/4 lines of 128 bytes) at the head of plane 1 kept in L2, a multiple of L/64"""
    g = PLANE1_KEEP_BYTES // (32 * L)
    return min(g, L // 4) // (L // 64) * (L // 64)


def row_classes(L):
    """Class of each output row m of a 2L x 2L focus: the row kernel writes intermediate row j of plane p to output row
    (2j + p + L) mod 2L (the fftshift along y), so p = (m - L) mod 2 and j = ((m - L) mod 2L) // 2.  0: plane 0, 1: kept
    head of plane 1 (j < 4 plane1_keep(L)), 2: the streamed rest of plane 1."""
    r = (np.arange(2 * L) - L) % (2 * L)
    p, j = r & 1, r >> 1
    return np.where(p == 0, 0, np.where(j < 4 * plane1_keep(L), 1, 2))


def impulse_focus(N, Q, pixels, values, inverse=False):
    """focus (inverse: unfocus) of an N x N array that is zero but for values[i] at pixels[i] = (row, col), in closed form.
    Padded to K = N Q at offset ceil((K - N)/2), ifftshift, ortho FFT, fftshift (_centered_ft2) make an impulse at padded
    position P the ramp exp(-+2 pi i (m - K//2)(P - K//2) / K) / K per axis; the products are reduced mod K in integers."""
    K = int(round(N * Q))
    assert K % 2 == 0
    off = math.ceil((K - N) / 2)
    s = 1.0 if inverse else -1.0
    m = np.arange(K, dtype=np.int64) - K // 2
    out = np.zeros((K, K), dtype=np.complex128)
    for (a, b), v in zip(pixels, values):
        ey = np.exp(s * 2j * np.pi * ((m * (a + off - K // 2)) % K) / K)
        ex = np.exp(s * 2j * np.pi * ((m * (b + off - K // 2)) % K) / K)
        out += v * np.outer(ey, ex)
    return out / K


def impulse_pixels(N):
    """the centre; the corner (0, 0); (0, N - 1); an off-centre pixel (N/2 + 5, N/2 - 3).  An impulse reaches every
    output sample: its position only sets the phase ramp, so a wrong rotation or sign shows as a ramp error."""
    return {'centre': (N // 2, N // 2), 'corner': (0, 0), 'edge': (0, N - 1), 'off': (N // 2 + 5, N // 2 - 3)}


IMPULSE_SUMS = {'centre': (('centre', 1.0 + 0.5j),),
                'corners': (('corner', -0.75 + 0.25j), ('edge', 0.5 - 1.0j)),
                'mix': (('centre', 0.25 - 0.5j), ('edge', 1.0 + 0.0j), ('off', -0.5 - 0.75j))}


# ---- measured figures (H100); bounds are 1.5x these, capped at 1e-6 ---------------------------------------------------
MEASURED = {
    'axis/angular_spectrum_adjoint_q1/2048': dict(linf=3.27e-7, l2=2.79e-7),
    'axis/angular_spectrum_adjoint_q2/1024': dict(linf=2.71e-7, l2=2.67e-7),
    'axis/angular_spectrum_adjoint_q2/2048': dict(linf=3.06e-7, l2=2.79e-7),
    'axis/angular_spectrum_adjoint_q2/4096': dict(linf=3.69e-7, l2=3.09e-7),
    'axis/angular_spectrum_q1/1024': dict(linf=2.86e-7, l2=2.66e-7),
    'axis/angular_spectrum_q1/2048': dict(linf=2.84e-7, l2=2.79e-7),
    'axis/angular_spectrum_q2/1024': dict(linf=2.50e-7, l2=2.77e-7),
    'axis/angular_spectrum_q2/2048': dict(linf=3.27e-7, l2=3.07e-7),
    'axis/angular_spectrum_q2/512': dict(linf=2.36e-7, l2=2.64e-7),
    'axis/czt/1024': dict(linf=3.95e-7, l2=3.56e-7),
    'axis/czt/2048': dict(linf=4.82e-7, l2=3.78e-7),
    'axis/czt/4096': dict(linf=5.45e-7, l2=3.96e-7),
    'axis/czt_adjoint/1024': dict(linf=4.71e-7, l2=3.54e-7),
    'axis/czt_adjoint/2048': dict(linf=4.11e-7, l2=3.83e-7),
    'axis/czt_adjoint/4096': dict(linf=4.70e-7, l2=3.99e-7),
    'axis/czt_intensity/1024': dict(linf=6.58e-7, l2=4.89e-7),
    'axis/czt_intensity/2048': dict(linf=6.68e-7, l2=5.30e-7),
    'axis/czt_intensity_accumulate/1024': dict(linf=9.55e-8, l2=2.61e-8),
    'axis/czt_intensity_accumulate/2048': dict(linf=2.99e-7, l2=5.90e-8),
    'axis/fft1_cols1/4096': dict(linf=1.48e-7, l2=1.26e-7),
    'axis/fft1_cols3/4096': dict(linf=1.62e-7, l2=1.27e-7),
    'axis/fft2/1024': dict(linf=1.82e-7, l2=1.67e-7),
    'axis/fft2/2048': dict(linf=2.16e-7, l2=1.75e-7),
    'axis/fft2/4096': dict(linf=2.43e-7, l2=1.91e-7),
    'axis/fft2_centred_crop_odd_width/2048': dict(linf=2.25e-7, l2=1.76e-7),
    'axis/focus_adjoint_q2/1024': dict(linf=2.03e-7, l2=1.67e-7),
    'axis/focus_adjoint_q2/2048': dict(linf=2.27e-7, l2=1.75e-7),
    'axis/focus_adjoint_q2/4096': dict(linf=2.39e-7, l2=1.91e-7),
    'axis/focus_q1/1024': dict(linf=1.74e-7, l2=1.67e-7),
    'axis/ifft2/1024': dict(linf=1.95e-7, l2=1.67e-7),
    'axis/ifft2/2048': dict(linf=2.01e-7, l2=1.75e-7),
    'axis/ifft2/4096': dict(linf=2.48e-7, l2=1.91e-7),
    'axis/ifft2_rows1/2048': dict(linf=1.45e-7, l2=1.21e-7),
    'axis/ifft2_rows1023/2048': dict(linf=2.32e-7, l2=1.73e-7),
    'axis/screened_free_space_q1/1024': dict(linf=2.97e-7, l2=2.68e-7),
    'axis/screened_free_space_q1/2048': dict(linf=2.95e-7, l2=2.81e-7),
    'axis/screened_free_space_q1/4096': dict(linf=3.36e-7, l2=3.11e-7),
    'axis/screened_free_space_q2/1024': dict(linf=2.66e-7, l2=2.78e-7),
    'axis/screened_free_space_q2/2048': dict(linf=3.53e-7, l2=3.09e-7),
    'axis/screened_free_space_q2/512': dict(linf=2.39e-7, l2=2.66e-7),
    'axis/unfocus_adjoint_q2/1024': dict(linf=2.00e-7, l2=1.67e-7),
    'axis/unfocus_adjoint_q2/2048': dict(linf=2.28e-7, l2=1.75e-7),
    'axis/unfocus_adjoint_q2/4096': dict(linf=2.33e-7, l2=1.91e-7),
    'v2/1024/+1/accumulate/stack5': dict(linf=3.67e-7, l2=9.28e-8, plane0=2.62e-7, plane1_kept=3.22e-7, plane1_streamed=3.67e-7),
    'v2/1024/+1/accumulate/staged_misaligned': dict(linf=3.86e-7, l2=9.28e-8, plane0=3.06e-7, plane1_kept=3.32e-7, plane1_streamed=3.86e-7),
    'v2/1024/+1/complex/impulse_centre': dict(linf=0.0, l2=0.0, plane0=0.0, plane1_kept=0.0, plane1_streamed=0.0),
    'v2/1024/+1/complex/impulse_corners': dict(linf=1.70e-7, l2=8.72e-8, plane0=1.70e-7, plane1_kept=1.70e-7, plane1_streamed=1.70e-7),
    'v2/1024/+1/complex/impulse_mix': dict(linf=2.74e-7, l2=1.13e-7, plane0=2.74e-7, plane1_kept=2.73e-7, plane1_streamed=2.73e-7),
    'v2/1024/+1/complex/stack5': dict(linf=2.55e-7, l2=1.84e-7, plane0=2.28e-7, plane1_kept=2.30e-7, plane1_streamed=2.55e-7),
    'v2/1024/+1/complex/staged_misaligned': dict(linf=2.53e-7, l2=1.84e-7, plane0=2.05e-7, plane1_kept=2.30e-7, plane1_streamed=2.53e-7),
    'v2/1024/+1/intensity/stack5': dict(linf=4.41e-7, l2=2.58e-7, plane0=3.53e-7, plane1_kept=4.26e-7, plane1_streamed=4.41e-7),
    'v2/1024/+1/intensity/staged_misaligned': dict(linf=4.41e-7, l2=2.58e-7, plane0=3.54e-7, plane1_kept=4.26e-7, plane1_streamed=4.41e-7),
    'v2/1024/-1/accumulate/stack5': dict(linf=3.46e-7, l2=9.27e-8, plane0=3.46e-7, plane1_kept=2.95e-7, plane1_streamed=3.26e-7),
    'v2/1024/-1/accumulate/staged_misaligned': dict(linf=3.06e-7, l2=9.26e-8, plane0=2.69e-7, plane1_kept=3.06e-7, plane1_streamed=2.98e-7),
    'v2/1024/-1/complex/impulse_centre': dict(linf=0.0, l2=0.0, plane0=0.0, plane1_kept=0.0, plane1_streamed=0.0),
    'v2/1024/-1/complex/impulse_corners': dict(linf=1.77e-7, l2=8.56e-8, plane0=1.77e-7, plane1_kept=1.77e-7, plane1_streamed=1.77e-7),
    'v2/1024/-1/complex/impulse_mix': dict(linf=2.83e-7, l2=1.14e-7, plane0=2.75e-7, plane1_kept=2.77e-7, plane1_streamed=2.83e-7),
    'v2/1024/-1/complex/stack5': dict(linf=2.51e-7, l2=1.83e-7, plane0=2.32e-7, plane1_kept=2.19e-7, plane1_streamed=2.51e-7),
    'v2/1024/-1/complex/staged_misaligned': dict(linf=2.51e-7, l2=1.84e-7, plane0=2.22e-7, plane1_kept=2.09e-7, plane1_streamed=2.51e-7),
    'v2/1024/-1/intensity/stack5': dict(linf=4.01e-7, l2=2.58e-7, plane0=3.84e-7, plane1_kept=3.93e-7, plane1_streamed=4.01e-7),
    'v2/1024/-1/intensity/staged_misaligned': dict(linf=3.93e-7, l2=2.58e-7, plane0=3.70e-7, plane1_kept=3.42e-7, plane1_streamed=3.93e-7),
    'v2/2048/+1/accumulate/padded': dict(linf=3.47e-7, l2=9.54e-8, plane0=3.47e-7, plane1_kept=2.64e-7, plane1_streamed=3.47e-7),
    'v2/2048/+1/accumulate/stack5': dict(linf=3.60e-7, l2=9.54e-8, plane0=3.60e-7, plane1_kept=2.48e-7, plane1_streamed=3.44e-7),
    'v2/2048/+1/accumulate/staged_misaligned': dict(linf=2.58e-7, l2=9.53e-8, plane0=2.55e-7, plane1_kept=1.92e-7, plane1_streamed=2.58e-7),
    'v2/2048/+1/complex/impulse_centre': dict(linf=0.0, l2=0.0, plane0=0.0, plane1_kept=0.0, plane1_streamed=0.0),
    'v2/2048/+1/complex/impulse_corners': dict(linf=2.16e-7, l2=1.01e-7, plane0=2.16e-7, plane1_kept=2.16e-7, plane1_streamed=2.16e-7),
    'v2/2048/+1/complex/impulse_mix': dict(linf=3.06e-7, l2=1.10e-7, plane0=3.06e-7, plane1_kept=2.67e-7, plane1_streamed=2.83e-7),
    'v2/2048/+1/complex/overlapping': dict(linf=2.65e-7, l2=1.91e-7, plane0=2.26e-7, plane1_kept=2.25e-7, plane1_streamed=2.65e-7),
    'v2/2048/+1/complex/single': dict(linf=2.18e-7, l2=1.91e-7, plane0=1.91e-7, plane1_kept=1.87e-7, plane1_streamed=2.18e-7),
    'v2/2048/+1/complex/stack5': dict(linf=2.65e-7, l2=1.91e-7, plane0=2.26e-7, plane1_kept=2.25e-7, plane1_streamed=2.65e-7),
    'v2/2048/+1/complex/staged_misaligned': dict(linf=2.18e-7, l2=1.92e-7, plane0=1.92e-7, plane1_kept=1.88e-7, plane1_streamed=2.18e-7),
    'v2/2048/+1/complex/staged_odd_in_bs_batch9': dict(linf=2.65e-7, l2=1.92e-7, plane0=2.26e-7, plane1_kept=2.25e-7, plane1_streamed=2.65e-7),
    'v2/2048/+1/complex/staged_odd_in_ld': dict(linf=2.18e-7, l2=1.92e-7, plane0=1.92e-7, plane1_kept=1.88e-7, plane1_streamed=2.18e-7),
    'v2/2048/+1/complex/staged_opd30_amp_none': dict(linf=6.31e-8, l2=1.63e-7, plane0=5.13e-8, plane1_kept=5.51e-8, plane1_streamed=6.31e-8),
    'v2/2048/+1/intensity/stack5': dict(linf=4.13e-7, l2=2.66e-7, plane0=4.08e-7, plane1_kept=3.25e-7, plane1_streamed=4.13e-7),
    'v2/2048/+1/intensity/staged_misaligned': dict(linf=2.86e-7, l2=2.66e-7, plane0=2.75e-7, plane1_kept=2.15e-7, plane1_streamed=2.86e-7),
    'v2/2048/-1/accumulate/padded': dict(linf=3.80e-7, l2=9.54e-8, plane0=3.11e-7, plane1_kept=3.80e-7, plane1_streamed=3.66e-7),
    'v2/2048/-1/accumulate/stack5': dict(linf=4.06e-7, l2=9.54e-8, plane0=3.03e-7, plane1_kept=3.89e-7, plane1_streamed=4.06e-7),
    'v2/2048/-1/accumulate/staged_misaligned': dict(linf=3.09e-7, l2=9.54e-8, plane0=2.42e-7, plane1_kept=2.13e-7, plane1_streamed=3.09e-7),
    'v2/2048/-1/accumulate/staged_opd30_amp_real_batch9': dict(linf=1.51e-7, l2=1.34e-7, plane0=1.51e-7, plane1_kept=3.72e-8, plane1_streamed=7.05e-8),
    'v2/2048/-1/complex/impulse_centre': dict(linf=0.0, l2=0.0, plane0=0.0, plane1_kept=0.0, plane1_streamed=0.0),
    'v2/2048/-1/complex/impulse_corners': dict(linf=1.93e-7, l2=9.26e-8, plane0=1.93e-7, plane1_kept=1.93e-7, plane1_streamed=1.93e-7),
    'v2/2048/-1/complex/impulse_mix': dict(linf=3.07e-7, l2=1.12e-7, plane0=3.07e-7, plane1_kept=2.80e-7, plane1_streamed=3.06e-7),
    'v2/2048/-1/complex/overlapping': dict(linf=2.62e-7, l2=1.91e-7, plane0=2.29e-7, plane1_kept=2.54e-7, plane1_streamed=2.62e-7),
    'v2/2048/-1/complex/single': dict(linf=2.14e-7, l2=1.91e-7, plane0=1.91e-7, plane1_kept=1.78e-7, plane1_streamed=2.14e-7),
    'v2/2048/-1/complex/stack5': dict(linf=2.62e-7, l2=1.91e-7, plane0=2.29e-7, plane1_kept=2.54e-7, plane1_streamed=2.62e-7),
    'v2/2048/-1/complex/staged_misaligned': dict(linf=2.14e-7, l2=1.92e-7, plane0=1.91e-7, plane1_kept=1.78e-7, plane1_streamed=2.14e-7),
    'v2/2048/-1/complex/staged_odd_in_bs_batch9': dict(linf=2.62e-7, l2=1.92e-7, plane0=2.29e-7, plane1_kept=2.54e-7, plane1_streamed=2.62e-7),
    'v2/2048/-1/complex/staged_odd_in_ld': dict(linf=2.14e-7, l2=1.92e-7, plane0=1.91e-7, plane1_kept=1.78e-7, plane1_streamed=2.14e-7),
    'v2/2048/-1/complex/staged_opd1e4_amp_u8_shared_batch9': dict(linf=2.42e-7, l2=1.96e-7, plane0=2.42e-7, plane1_kept=2.10e-7, plane1_streamed=2.40e-7),
    'v2/2048/-1/intensity/stack5': dict(linf=4.94e-7, l2=2.66e-7, plane0=3.66e-7, plane1_kept=4.94e-7, plane1_streamed=4.75e-7),
    'v2/2048/-1/intensity/staged_misaligned': dict(linf=3.57e-7, l2=2.66e-7, plane0=2.84e-7, plane1_kept=2.30e-7, plane1_streamed=3.57e-7),
    'v2/512/+1/accumulate/padded': dict(linf=3.30e-7, l2=9.12e-8, plane0=3.30e-7, plane1_kept=3.15e-7),
    'v2/512/+1/accumulate/stack5': dict(linf=3.38e-7, l2=9.13e-8, plane0=2.92e-7, plane1_kept=3.38e-7),
    'v2/512/+1/accumulate/staged_misaligned': dict(linf=2.68e-7, l2=9.12e-8, plane0=2.04e-7, plane1_kept=2.68e-7),
    'v2/512/+1/complex/impulse_centre': dict(linf=0.0, l2=0.0, plane0=0.0, plane1_kept=0.0),
    'v2/512/+1/complex/impulse_corners': dict(linf=1.93e-7, l2=1.04e-7, plane0=1.93e-7, plane1_kept=1.93e-7),
    'v2/512/+1/complex/impulse_mix': dict(linf=2.96e-7, l2=1.17e-7, plane0=2.96e-7, plane1_kept=2.95e-7),
    'v2/512/+1/complex/overlapping': dict(linf=2.34e-7, l2=1.77e-7, plane0=2.19e-7, plane1_kept=2.34e-7),
    'v2/512/+1/complex/single': dict(linf=2.05e-7, l2=1.77e-7, plane0=1.93e-7, plane1_kept=2.05e-7),
    'v2/512/+1/complex/stack5': dict(linf=2.34e-7, l2=1.77e-7, plane0=2.19e-7, plane1_kept=2.34e-7),
    'v2/512/+1/complex/staged_misaligned': dict(linf=2.05e-7, l2=1.78e-7, plane0=1.93e-7, plane1_kept=2.05e-7),
    'v2/512/+1/complex/staged_odd_in_bs_batch9': dict(linf=2.35e-7, l2=1.78e-7, plane0=2.19e-7, plane1_kept=2.35e-7),
    'v2/512/+1/complex/staged_odd_in_ld': dict(linf=2.05e-7, l2=1.78e-7, plane0=1.93e-7, plane1_kept=2.05e-7),
    'v2/512/+1/complex/staged_opd30_amp_none': dict(linf=8.59e-8, l2=1.50e-7, plane0=8.59e-8, plane1_kept=4.16e-8),
    'v2/512/+1/intensity/stack5': dict(linf=3.93e-7, l2=2.54e-7, plane0=3.88e-7, plane1_kept=3.93e-7),
    'v2/512/+1/intensity/staged_misaligned': dict(linf=3.56e-7, l2=2.54e-7, plane0=2.70e-7, plane1_kept=3.56e-7),
    'v2/512/-1/accumulate/padded': dict(linf=3.98e-7, l2=9.16e-8, plane0=3.26e-7, plane1_kept=3.98e-7),
    'v2/512/-1/accumulate/stack5': dict(linf=3.64e-7, l2=9.17e-8, plane0=3.11e-7, plane1_kept=3.64e-7),
    'v2/512/-1/accumulate/staged_misaligned': dict(linf=3.57e-7, l2=9.12e-8, plane0=3.45e-7, plane1_kept=3.57e-7),
    'v2/512/-1/accumulate/staged_opd30_amp_real_batch9': dict(linf=1.69e-7, l2=1.49e-7, plane0=1.69e-7, plane1_kept=9.19e-8),
    'v2/512/-1/complex/impulse_centre': dict(linf=0.0, l2=0.0, plane0=0.0, plane1_kept=0.0),
    'v2/512/-1/complex/impulse_corners': dict(linf=1.68e-7, l2=8.78e-8, plane0=1.68e-7, plane1_kept=1.68e-7),
    'v2/512/-1/complex/impulse_mix': dict(linf=3.08e-7, l2=1.16e-7, plane0=2.74e-7, plane1_kept=3.08e-7),
    'v2/512/-1/complex/overlapping': dict(linf=2.48e-7, l2=1.78e-7, plane0=2.16e-7, plane1_kept=2.48e-7),
    'v2/512/-1/complex/single': dict(linf=2.48e-7, l2=1.77e-7, plane0=2.03e-7, plane1_kept=2.48e-7),
    'v2/512/-1/complex/stack5': dict(linf=2.48e-7, l2=1.78e-7, plane0=2.16e-7, plane1_kept=2.48e-7),
    'v2/512/-1/complex/staged_misaligned': dict(linf=2.48e-7, l2=1.78e-7, plane0=2.04e-7, plane1_kept=2.48e-7),
    'v2/512/-1/complex/staged_odd_in_bs_batch9': dict(linf=2.48e-7, l2=1.78e-7, plane0=2.17e-7, plane1_kept=2.48e-7),
    'v2/512/-1/complex/staged_odd_in_ld': dict(linf=2.48e-7, l2=1.78e-7, plane0=2.04e-7, plane1_kept=2.48e-7),
    'v2/512/-1/complex/staged_opd1e4_amp_u8_shared_batch9': dict(linf=2.74e-7, l2=1.82e-7, plane0=2.46e-7, plane1_kept=2.74e-7),
    'v2/512/-1/intensity/stack5': dict(linf=4.94e-7, l2=2.54e-7, plane0=3.42e-7, plane1_kept=4.94e-7),
    'v2/512/-1/intensity/staged_misaligned': dict(linf=3.88e-7, l2=2.54e-7, plane0=3.36e-7, plane1_kept=3.88e-7),
}


# a case's figure is the worst over its fields, within its test; a result that was exact (the focus of a centred
# impulse) stays exact
LEDGER = Ledger(MEASURED, NORTH_STAR, per_test=True)


def add(case, got, ref, rows=None, field=0):
    """the whole array against its reference: rel_linf, the relative L2 error and, with `rows`, the figure of each
    row class"""
    got = host(got)
    figs = {'linf': rel_linf(got, ref), 'l2': rel_l2(got, ref)}
    if rows is not None:
        rowmax = np.abs(got - ref).max(axis=1)
        den = float(np.abs(ref).max())
        for c, cname in enumerate(CLASSES):
            sel = rowmax[rows == c]
            if sel.size:
                figs[cname] = float(sel.max()) / den
    for k, v in figs.items():
        LEDGER.record(f'{case}/{k}', v, f'worst field {field}')


# ---- which kernels ran --------------------------------------------------------------------------------------------
# Routes are pinned by the library's per-route launch counters (pb_route_launch_count): each launch of an
# axis_reg_kernel instantiation, of the generic axis pass and of either focus pair counts on its own key of the handle.
HIT = set()          # (L, INV, COLS, RT, PM, DENSE) of every axis_reg_kernel instantiation an fp64-checked case ran
AXIS_ALL = [(L, inv, cols, rt, pm, dense) for L in (1024, 2048, 4096) for inv in (False, True) for cols in (False, True)
            for rt in (False, True) for pm in (False, True) for dense in (False, True)]


def axis_code(k):
    from prysm_b200 import _capi
    L, inv, cols, rt, pm, dense = k
    return _capi.route_code(_capi.ROUTE_AXIS_REG, L, int(inv) | int(cols) << 1 | int(rt) << 2 | int(pm) << 3 | int(dense) << 4)


def route_codes():
    """every axis_reg_kernel instantiation, the generic axis pass (all lengths) and the focus pair"""
    from prysm_b200 import _capi
    codes = {k: axis_code(k) for k in AXIS_ALL}
    codes['generic'] = _capi.route_code(_capi.ROUTE_AXIS_GENERIC)
    for N in NS:
        for inv in (0, 1):
            codes[('focus', N, inv)] = _capi.route_code(_capi.ROUTE_FOCUS_V2, N, inv)
    return codes


def routes_of(fn):
    """fn()'s result and the launches it made, per route (only the routes it used)"""
    return _routes_of(fn, route_codes())


def run_axis(case, fn, expect):
    """fn() for its result: every instantiation in `expect` must have run, nothing but the register engine (no generic
    axis pass, no focus pair), and no instantiation outside EXPECTED"""
    res, used = routes_of(fn)
    hits = {k for k in used if isinstance(k, tuple) and k[0] != 'focus'}
    other = sorted(str(k) for k in used if k != 'all' and k not in hits)
    LEDGER.route(not other, f'{case}: other routes ran: {other}')
    LEDGER.route(hits <= EXPECTED, f'{case}: unexpected instantiations {sorted(hits - EXPECTED)}')
    LEDGER.route(set(expect) <= hits, f'{case}: {sorted(set(expect) - hits)} did not run; ran {sorted(hits)}')
    HIT.update(hits)
    return res


# ---- fixtures -----------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module', autouse=True)
def precision_32(pb):
    pb.config.precision = 32
    yield
    _REF.clear()
    _HOST.clear()


_HOST = {}   # host inputs by key
_REF = {}    # complex128 references by (input key, field, direction), least recently used first
REF_CACHE_BYTES = 2 << 30   # about eight 4096^2 references: a stack of 5 and a few more


def crand(shape, seed):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal(shape, dtype=np.float32) + 1j * rng.standard_normal(shape, dtype=np.float32)).astype(np.complex64)


def gauss_stack(N):
    """NSTACK seeded complex Gaussian fields, complex64 on the host"""
    key = ('gauss', N)
    if key not in _HOST:
        _HOST[key] = crand((NSTACK, N, N), N)
    return _HOST[key]


def opd_stack(N, nb, sigma):
    """nb OPD fields [nm] (float32), a shared bool amplitude and per-field real amplitudes"""
    key = ('opd', N, nb, sigma)
    if key not in _HOST:
        rng = np.random.default_rng(N + nb)
        opd = (sigma * rng.standard_normal((nb, N, N))).astype(np.float32)
        mask = rng.random((N, N)) > 0.3
        amps = rng.uniform(0.2, 1.0, (nb, N, N)).astype(np.float32)
        _HOST[key] = (opd, mask, amps)
    return _HOST[key]


KSCALE = 2 * np.pi / HeNe / 1e3     # OPD [nm] -> radians, phase_prefix(HeNe).imag


def focus_ref(key, i, d, field):
    """focus (d = -1) / unfocus (d = +1) at Q = 2 of `field` (complex128), cached under (key, i, d)"""
    k = (key, i, d)
    if k in _REF:
        _REF[k] = _REF.pop(k)
    else:
        with sfft.set_workers(-1):
            _REF[k] = (O.focus if d < 0 else O.unfocus)(field, 2)
        while sum(r.nbytes for r in _REF.values()) > REF_CACHE_BYTES:
            del _REF[next(iter(_REF))]
    return _REF[k]


def gauss_ref(N, i, d):
    return focus_ref(('gauss', N), i, d, gauss_stack(N)[i].astype(np.complex128))


def opd_ref(N, nb, sigma, amp, i, d):
    """reference of field i of an OPD stack; amp: 'none', 'mask' (shared) or 'real' (per field)"""
    opd, mask, amps = opd_stack(N, nb, sigma)
    a = 1.0 if amp == 'none' else mask.astype(np.float64) if amp == 'mask' else amps[i].astype(np.float64)
    return focus_ref(('opd', N, nb, sigma, amp), i, d, a * np.exp(1j * KSCALE * opd[i].astype(np.float64)))


def derive(ref, kind, acc0=None):
    """complex, |.|^2 or acc0 + WEIGHT |.|^2 of a complex reference, in fp64"""
    if kind == 'complex':
        return ref
    inten = ref.real * ref.real + ref.imag * ref.imag
    return inten if kind == 'intensity' else acc0.astype(np.float64) + WEIGHT * inten


def acc_start(shape, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return torch.rand(shape, generator=g, device='cuda')


KINDS = ('complex', 'intensity', 'accumulate')


def out_kind(capi, kind):
    return {'complex': capi.OUT_COMPLEX, 'intensity': capi.OUT_INTENSITY, 'accumulate': capi.OUT_ACCUMULATE}[kind]


def batch_call(ops, src, N, d, nb, in_bs, in_ld, out, kind, *, in_kind=None, amp=None, amp_kind=None, amp_bs=0,
               weight=WEIGHT):
    """one direct pb_fft2_batch call: Q = 2 focus (d = -1) / unfocus of nb fields at any pitch, into the (nb, 2N, 2N)
    view `out`"""
    capi = ops.capi
    K = 2 * N
    h, st = ops._ctx(out)
    h.check(capi.lib.pb_fft2_batch(
        h.ptr, capi.PB_C64, C.c_void_p(src.data_ptr()), capi.IN_COMPLEX if in_kind is None else in_kind,
        C.c_void_p(0 if amp is None else amp.data_ptr()), capi.AMP_NONE if amp_kind is None else amp_kind, KSCALE,
        nb, in_bs, amp_bs, N, N, in_ld, K, K, d, 1.0 / K, 1, 1, C.c_void_p(out.data_ptr()), out_kind(capi, kind),
        float(weight), K, K, out.stride(1), out.stride(0), st))
    return out


def check_focus(case, N, d, fn, refs, nlaunch, nscreen=0):
    """fn() -> (nb, 2N, 2N) output; refs: {field: reference}; nlaunch: the launches of the focus pair of <N, INV> the
    call takes, and it launches nothing else but `nscreen` phase-screen kernels.  Outputs are bounded per row class of the
    tile-major intermediate."""
    got, used = routes_of(fn)
    want = {('focus', N, int(d > 0)): nlaunch, 'all': nlaunch + nscreen}
    LEDGER.route(used == want, f'{case}: launches per route {used}, the route takes {want}')
    rows = row_classes(N)
    for b, ref in refs.items():
        add(case, got[b], ref, rows, b)


# ---- the fused focus pair (tensor-TMA input, one launch pair per field) -------------------------------------------
@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('d', (-1, 1))
@pytest.mark.parametrize('N', NS)
def test_v2_stack_every_field(pb, N, d, kind):
    """a stack of 5 (both intermediates, early input: disjoint from the output), every field against fp64"""
    from prysm_b200 import _ops
    K = 2 * N
    x = torch.from_numpy(gauss_stack(N)).cuda()
    acc0 = acc_start((NSTACK, K, K), N + 1) if kind == 'accumulate' else None
    acc0h = None if acc0 is None else acc0.cpu().numpy()

    def fn():
        out = acc0.clone() if acc0 is not None else torch.empty((NSTACK, K, K), device='cuda',
                                                                  dtype=torch.complex64 if kind == 'complex' else torch.float32)
        return batch_call(_ops, x, N, d, NSTACK, N * N, N, out, kind)

    refs = {b: derive(gauss_ref(N, b, d), kind, None if acc0h is None else acc0h[b]) for b in range(NSTACK)}
    check_focus(f'v2/{N}/{d:+d}/{kind}/stack5', N, d, fn, refs, 2 * NSTACK)
    LEDGER.done()


@pytest.mark.parametrize('d', (-1, 1))
@pytest.mark.parametrize('N', (512, 2048))
def test_v2_single_overlapping_padded(pb, N, d):
    """one field through the public call; a stack inside the output allocation (the column kernels wait before their
    gather); an output with padded field and row pitches, accumulated"""
    from prysm_b200 import _ops
    P = pb.propagation
    K = 2 * N
    host = gauss_stack(N)
    x = torch.from_numpy(host).cuda()
    one = x[0].clone()
    fn = (lambda: (P.focus if d < 0 else P.unfocus)(one, 2)[None])
    check_focus(f'v2/{N}/{d:+d}/complex/single', N, d, fn, {0: gauss_ref(N, 0, d)}, 2)

    buf = torch.zeros((NSTACK, K, K + N), dtype=torch.complex64, device='cuda')
    src = buf[:, :N, K:]
    src.copy_(x)

    def inside():
        out = buf[:, :, :K]
        batch_call(_ops, src, N, d, NSTACK, src.stride(0), src.stride(1), out, 'complex')
        return out
    check_focus(f'v2/{N}/{d:+d}/complex/overlapping', N, d, inside,
           {b: gauss_ref(N, b, d) for b in range(NSTACK)}, 2 * NSTACK)
    assert torch.equal(src, x)

    big0 = acc_start((NSTACK, K + 3, K + 6), N + 2)
    acc0h = big0[:, 1:K + 1, 2:K + 2].cpu().numpy()

    def padded():
        big = big0.clone()
        out = big[:, 1:K + 1, 2:K + 2]
        batch_call(_ops, x, N, d, NSTACK, N * N, N, out, 'accumulate')
        outside = torch.ones(big.shape, dtype=torch.bool, device='cuda')
        outside[:, 1:K + 1, 2:K + 2] = False
        assert torch.equal(big[outside], big0[outside])      # no store outside the window
        return out
    check_focus(f'v2/{N}/{d:+d}/accumulate/padded', N, d, padded,
           {b: derive(gauss_ref(N, b, d), 'accumulate', acc0h[b]) for b in range(NSTACK)}, 2 * NSTACK)
    LEDGER.done()


@pytest.mark.parametrize('d', (-1, 1))
@pytest.mark.parametrize('N', NS)
def test_v2_impulses(pb, N, d):
    """sums of impulses against their closed form (no FFT in the reference)"""
    from prysm_b200 import _ops
    px = impulse_pixels(N)
    for name, terms in IMPULSE_SUMS.items():
        a = np.zeros((N, N), dtype=np.complex64)
        for p, v in terms:
            a[px[p]] += v
        x = torch.from_numpy(a).cuda()
        ref = impulse_focus(N, 2, [px[p] for p, _ in terms], [v for _, v in terms], inverse=d > 0)
        fn = (lambda: _ops.fft2(x, (2 * N, 2 * N), dir=d, scale=0.5 / N, shift_in=True, shift_out=True)[None])
        check_focus(f'v2/{N}/{d:+d}/complex/impulse_{name}', N, d, fn, {0: ref}, 2)
    LEDGER.done()


# ---- the fused focus pair, staged inputs (tensor TMA cannot gather them: staged field by field) ------------------------
@pytest.mark.parametrize('d', (-1, 1))
@pytest.mark.parametrize('N', NS)
def test_staged_misaligned_base_every_output_kind(pb, N, d):
    """a complex input whose base is 8 bytes off 16-byte alignment, through the public call (with weight)"""
    from prysm_b200 import _ops
    K = 2 * N
    flat = torch.empty(N * N + 1, dtype=torch.complex64, device='cuda')
    src = flat[1:].view(N, N)
    src.copy_(torch.from_numpy(gauss_stack(N)[0]))
    assert src.data_ptr() % 16 == 8
    acc0 = acc_start((K, K), N + 3)
    for kind in KINDS:
        def fn():
            out = acc0.clone() if kind == 'accumulate' else None
            return _ops.fft2(src, (K, K), dir=d, scale=1.0 / K, shift_in=True, shift_out=True,
                             out_kind=out_kind(_ops.capi, kind), weight=WEIGHT, out=out)[None]
        ref = derive(gauss_ref(N, 0, d), kind, acc0.cpu().numpy())
        check_focus(f'v2/{N}/{d:+d}/{kind}/staged_misaligned', N, d, fn, {0: ref}, 2)
    LEDGER.done()


@pytest.mark.parametrize('d', (-1, 1))
@pytest.mark.parametrize('N', (512, 2048))
def test_staged_odd_pitches(pb, N, d):
    """an odd row pitch (one field), and an odd field pitch on a stack of 9 whose fields repeat the Gaussian stack in the
    order 0 1 2 3 4 4 3 2 1 (a field staged from the wrong base gets the wrong field)"""
    from prysm_b200 import _ops
    K = 2 * N
    host = gauss_stack(N)
    buf = torch.zeros((N, N + 1), dtype=torch.complex64, device='cuda')
    buf[:, :N] = torch.from_numpy(host[0])

    def odd_ld():
        out = torch.empty((1, K, K), dtype=torch.complex64, device='cuda')
        return batch_call(_ops, buf, N, d, 1, 0, N + 1, out, 'complex')
    check_focus(f'v2/{N}/{d:+d}/complex/staged_odd_in_ld', N, d, odd_ld, {0: gauss_ref(N, 0, d)}, 2)

    order = (0, 1, 2, 3, 4, 4, 3, 2, 1)
    bs = N * N + 1
    flat = torch.zeros(9 * bs, dtype=torch.complex64, device='cuda')
    src = flat.as_strided((9, N, N), (bs, N, 1))
    src.copy_(torch.from_numpy(host[list(order)]))

    def odd_bs():
        out = torch.empty((9, K, K), dtype=torch.complex64, device='cuda')
        return batch_call(_ops, src, N, d, 9, bs, N, out, 'complex')
    fields = range(9) if N < 2048 else (0, 4, 7, 8)
    check_focus(f'v2/{N}/{d:+d}/complex/staged_odd_in_bs_batch9', N, d, odd_bs,
           {b: gauss_ref(N, order[b], d) for b in fields}, 18)
    LEDGER.done()


@pytest.mark.parametrize('N', (512, 2048))
def test_staged_phase_screen_input(pb, N):
    """PB_IN_AMP_OPD: no amplitude and an OPD of tens of nm (one field); a bool amplitude shared by a stack of 9 with an
    OPD of ~1e4 nm (many waves: the fp64 phase range reduction); per-field real amplitudes, |.|^2 accumulated"""
    from prysm_b200 import _ops
    K = 2 * N
    fields = range(9) if N < 2048 else (0, 7, 8)
    opd_s, mask, _ = opd_stack(N, 9, 30.0)
    opd = torch.from_numpy(opd_s).cuda()
    fn = (lambda: _ops.fft2(None, (K, K), dir=1, scale=1.0 / K, shift_in=True, shift_out=True, opd=opd[0],
                            kscale=KSCALE)[None])
    check_focus(f'v2/{N}/+1/complex/staged_opd30_amp_none', N, 1, fn, {0: opd_ref(N, 9, 30.0, 'none', 0, 1)}, 2, 1)

    opd_l, mask_l, _ = opd_stack(N, 9, 1e4)
    opdl = torch.from_numpy(opd_l).cuda()
    m = torch.from_numpy(mask_l).cuda()
    fn = (lambda: _ops.fft2_batch(None, (K, K), dir=-1, scale=1.0 / K, shift_in=True, shift_out=True, amp=m, opd=opdl,
                                  kscale=KSCALE))
    check_focus(f'v2/{N}/-1/complex/staged_opd1e4_amp_u8_shared_batch9', N, -1, fn,
           {b: opd_ref(N, 9, 1e4, 'mask', b, -1) for b in fields}, 18, 9)

    _, _, amps_s = opd_stack(N, 9, 30.0)
    amps = torch.from_numpy(amps_s).cuda()
    acc0 = acc_start((9, K, K), N + 4)
    acc0h = acc0.cpu().numpy()

    def fn2():
        out = acc0.clone()
        return batch_call(_ops, opd, N, -1, 9, N * N, N, out, 'accumulate', in_kind=_ops.capi.IN_AMP_OPD, amp=amps,
                          amp_kind=_ops.capi.AMP_REAL, amp_bs=N * N)
    check_focus(f'v2/{N}/-1/accumulate/staged_opd30_amp_real_batch9', N, -1, fn2,
           {b: derive(opd_ref(N, 9, 30.0, 'real', b, -1), 'accumulate', acc0h[b]) for b in fields}, 18, 9)
    LEDGER.done()


# ---- the register axis engine, through the public API ---------------------------------------------------------------
def _k(L, inv, cols, rt=False, pm=False, dense=False):
    return (L, inv, cols, rt, pm, dense)


def rows_cols(L, inv, dense=False):
    return [_k(L, inv, False, dense=dense), _k(L, inv, True, dense=dense)]


# Every instantiation dispatch_axis_reg can launch from the Python API.  Not reachable, and so not listed:
#  * INV = true with RT: every round trip (a CZT axis, the column pass of a free-space step) is launched forward;
#  * PM with INV, COLS or RT: only the forward row pass of a screened free-space step carries the full-matrix multiplier;
#  * DENSE with RT on rows: a dense round trip on rows takes the general round-trip kernel (only the column form has a
#    DENSE specialisation), and no round trip on rows is dense anyway (CZT has its output multiplier);
#  * DENSE without PM at L = 1024: those passes take the general kernels (the DENSE forms are for L >= 2048).
EXPECTED = set()
for _L in (1024, 2048, 4096):
    EXPECTED |= {_k(_L, inv, cols) for inv in (False, True) for cols in (False, True)}
    EXPECTED |= {_k(_L, False, False, rt=True), _k(_L, False, True, rt=True)}
    EXPECTED |= {_k(_L, False, False, pm=True), _k(_L, False, False, pm=True, dense=True)}
    if _L >= 2048:
        EXPECTED |= {_k(_L, inv, cols, dense=True) for inv in (False, True) for cols in (False, True)}
        EXPECTED.add(_k(_L, False, True, rt=True, dense=True))


@pytest.mark.parametrize('n', (1024, 2048, 4096))
def test_axis_plain_fft2(pb, n):
    """fft2 / ifft2: the DENSE row and column kernels at 2048 and 4096, the general ones at 1024"""
    from prysm_b200 import _ops
    a = crand((n, n), 100 + n)
    d = dev(a)
    dense = n >= 2048
    with sfft.set_workers(-1):
        ref = sfft.fft2(a.astype(np.complex128))
    got = run_axis(f'axis/fft2/{n}', lambda: _ops.fft2(d, (n, n), dir=-1), rows_cols(n, False, dense))
    add(f'axis/fft2/{n}', got, ref)
    del ref
    with sfft.set_workers(-1):
        ref = sfft.ifft2(a.astype(np.complex128))
    got = run_axis(f'axis/ifft2/{n}', lambda: _ops.fft2(d, (n, n), dir=1, scale=1.0 / (n * n)), rows_cols(n, True, dense))
    add(f'axis/ifft2/{n}', got, ref)
    LEDGER.done()


@pytest.mark.parametrize('n', (1024, 2048, 4096))
def test_axis_centred_and_cropped(pb, n):
    """focus(., 1); focus_adjoint / unfocus_adjoint at Q = 2 (a centred crop): the general kernels, both directions"""
    P = pb.propagation
    a = crand((n, n), 200 + n)
    d = dev(a)
    a2 = a.astype(np.complex128)
    with sfft.set_workers(-1):
        if n == 1024:
            got = run_axis(f'axis/focus_q1/{n}', lambda: P.focus(d, 1), rows_cols(n, False))
            add(f'axis/focus_q1/{n}', got, O.focus(a2, 1))
        got = run_axis(f'axis/focus_adjoint_q2/{n}', lambda: P.focus_adjoint(d, 2), rows_cols(n, True))
        add(f'axis/focus_adjoint_q2/{n}', got, O.focus_adjoint(a2, 2))
        got = run_axis(f'axis/unfocus_adjoint_q2/{n}', lambda: P.unfocus_adjoint(d, 2), rows_cols(n, False))
        add(f'axis/unfocus_adjoint_q2/{n}', got, O.unfocus_adjoint(a2, 2))
    LEDGER.done()


def test_axis_odd_width_and_line_counts(pb):
    """an odd output width (no 128-bit column access); odd and single populated row counts; odd and single column
    counts of a one-axis transform"""
    from prysm_b200 import _ops
    n = 2048

    def centred(a, shape, crop=None):
        with sfft.set_workers(-1):
            r = sfft.fftshift(sfft.fft2(sfft.ifftshift(O.pad2d(a.astype(np.complex128), out_shape=shape))))
        return r if crop is None else O.crop_center(r, crop)

    a = crand((n, n), 301)
    got = run_axis('axis/fft2_centred_crop_odd_width/2048', lambda: _ops.fft2(dev(a), (n, n), dir=-1, shift_in=True, shift_out=True, crop=(n, n - 1)),
              rows_cols(n, False))
    add('axis/fft2_centred_crop_odd_width/2048', got, centred(a, (n, n), (n, n - 1)))
    for rows in (1023, 1):
        b = crand((rows, n), 302 + rows)
        got = run_axis(f'axis/ifft2_rows{rows}/2048', lambda: _ops.fft2(dev(b), (n, n), dir=1, shift_in=True, shift_out=True), rows_cols(n, True))
        with sfft.set_workers(-1):
            ref = sfft.fftshift(sfft.ifft2(sfft.ifftshift(O.pad2d(b.astype(np.complex128), out_shape=(n, n)))) * (n * n))
        add(f'axis/ifft2_rows{rows}/2048', got, ref)
    for cols in (3, 1):
        c = crand((4096, cols), 304 + cols)
        got = run_axis(f'axis/fft1_cols{cols}/4096', lambda: _ops.fft1(dev(c), axis=0, dir=-1), [_k(4096, False, True)])
        add(f'axis/fft1_cols{cols}/4096', got, sfft.fft(c.astype(np.complex128), axis=0))
    LEDGER.done()


WVL, DX, Z = HeNe, 0.01, 25.0


@pytest.mark.parametrize('n,Q', [(1024, 1), (2048, 1), (512, 2), (1024, 2), (2048, 2)])
def test_axis_angular_spectrum(pb, n, Q):
    """angular_spectrum: rows forward, the column round trip with the transfer function, rows inverse"""
    P = pb.propagation
    L = n * Q
    f = crand((n, n), 400 + n + Q)
    dense = Q == 1 and L >= 2048
    expect = [_k(L, False, False, dense=dense), _k(L, False, True, rt=True, dense=dense), _k(L, True, False, dense=L >= 2048)]
    got = run_axis(f'axis/angular_spectrum_q{Q}/{n}', lambda: P.angular_spectrum(dev(f), WVL, DX, Z, Q), expect)
    with sfft.set_workers(-1):
        ref = O.angular_spectrum(f.astype(np.complex128), WVL, DX, Z, Q)
    add(f'axis/angular_spectrum_q{Q}/{n}', got, ref)
    LEDGER.done()


@pytest.mark.parametrize('L,Q', [(2048, 1), (1024, 2), (2048, 2), (4096, 2)])
def test_axis_angular_spectrum_adjoint(pb, L, Q):
    """angular_spectrum_adjoint: the conjugated transfer function, and the crop to L/Q in the round trip"""
    P = pb.propagation
    g = crand((L, L), 500 + L + Q)
    expect = [_k(L, False, False, dense=L >= 2048), _k(L, False, True, rt=True, dense=Q == 1 and L >= 2048)]
    got = run_axis(f'axis/angular_spectrum_adjoint_q{Q}/{L}', lambda: P.angular_spectrum_adjoint(dev(g), WVL, DX, Z, Q), expect)
    with sfft.set_workers(-1):
        ref = O.angular_spectrum_adjoint(g.astype(np.complex128), WVL, DX, Z, Q)
    add(f'axis/angular_spectrum_adjoint_q{Q}/{L}', got, ref)
    LEDGER.done()


@pytest.mark.parametrize('n,Q', [(1024, 1), (2048, 1), (4096, 1), (512, 2), (1024, 2), (2048, 2)])
def test_axis_screened_free_space(pb, n, Q):
    """angular_spectrum(screen=): the screen multiplied in the first row pass (PM; DENSE at Q = 1)"""
    P = pb.propagation
    L = n * Q
    f = crand((n, n), 600 + n + Q)
    rng = np.random.default_rng(700 + n)
    s = np.exp(1j * rng.uniform(0, 2 * np.pi, (n, n))).astype(np.complex64)
    got = run_axis(f'axis/screened_free_space_q{Q}/{n}', lambda: P.angular_spectrum(dev(f), WVL, DX, Z, Q, screen=dev(s)), [_k(L, False, False, pm=True, dense=Q == 1)])
    with sfft.set_workers(-1):
        ref = O.angular_spectrum(f.astype(np.complex128) * s.astype(np.complex128), WVL, DX, Z, Q)
    add(f'axis/screened_free_space_q{Q}/{n}', got, ref)
    LEDGER.done()


CZT_GEOMETRY = {1024: (512, 512), 2048: (1024, 1023), 4096: (2048, 1024)}   # K: (pupil samples N, focal samples M)


def czt_pair(pb, K):
    N, M = CZT_GEOMETRY[K]
    args = (0.01, (N, N), 1.5, (M, M), HeNe, 100.0, (2.0, -1.0), 'czt')
    return pb.propagation.prepare_executor(*args), O.prepare_executor(*args), N, M


@pytest.mark.parametrize('K', (1024, 2048, 4096))
def test_axis_czt(pb, K):
    """CZT forward and adjoint: one round trip per axis, rows then columns"""
    ex, exo, N, M = czt_pair(pb, K)
    a = crand((N, N), 800 + K)
    g = crand((M, M), 900 + K)
    rt = [_k(K, False, False, rt=True), _k(K, False, True, rt=True)]
    got = run_axis(f'axis/czt/{K}', lambda: ex(dev(a)), rt)
    add(f'axis/czt/{K}', got, exo(a.astype(np.complex128)))
    got = run_axis(f'axis/czt_adjoint/{K}', lambda: ex.adjoint(dev(g)), rt)
    add(f'axis/czt_adjoint/{K}', got, exo.adjoint(g.astype(np.complex128)))
    LEDGER.done()


@pytest.mark.parametrize('K', (1024, 2048))
def test_axis_czt_intensity(pb, K):
    """CZT.intensity, written and accumulated: |.|^2 in the store of the column round trip -- as aligned pairs of
    columns (vec_int, even M = 512) and one column at a time (odd M = 1023)"""
    ex, exo, N, M = czt_pair(pb, K)
    a = crand((N, N), 1000 + K)
    ref = exo(a.astype(np.complex128))
    inten = ref.real ** 2 + ref.imag ** 2
    rt = [_k(K, False, False, rt=True), _k(K, False, True, rt=True)]
    got = run_axis(f'axis/czt_intensity/{K}', lambda: ex.intensity(dev(a)), rt)
    add(f'axis/czt_intensity/{K}', got, inten)
    acc0 = acc_start((M, M), K)
    got = run_axis(f'axis/czt_intensity_accumulate/{K}', lambda: ex.intensity(dev(a), weight=WEIGHT, out=acc0.clone()), rt)
    add(f'axis/czt_intensity_accumulate/{K}', got, acc0.cpu().numpy().astype(np.float64) + WEIGHT * inten)
    LEDGER.done()


def test_zz_every_reachable_instantiation_was_hit(pb):
    """runs last: every axis_reg_kernel instantiation the Python API can reach ran in an fp64-checked case above"""
    assert not EXPECTED - HIT, sorted(EXPECTED - HIT)
    assert not HIT - EXPECTED, sorted(HIT - EXPECTED)


def test_zz_every_figure_has_a_measurement():
    """a figure this session reached that has no MEASURED entry is held to the bare ceiling, a bound nobody measured"""
    if os.environ.get('PB_TEST_MEASUREMENTS'):
        pytest.skip('recording figures')
    assert not LEDGER.missing(), f'no MEASURED entry (record them with PB_TEST_MEASUREMENTS): {LEDGER.missing()}'
