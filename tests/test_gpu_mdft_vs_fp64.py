"""GPU: every route of the matrix DFT -- the tensor-core GEMM pair of csrc/mdft_tc.cu (plain, split-K 2 / 4 / 8 + reduce,
and stream-K in either stage) and the CUDA-core GEMM of csrc/cgemm.cu -- held to fp64 references over whole arrays.

Each array is compared whole by two metrics: rel_linf (max|a - b| / max|b|) and the relative L2 error.  Each executor
output is held to two references:
  * gemm: the complex128 product of the device's own complex64 bases and the complex64 input -- the GEMM arithmetic alone;
  * e2e:  oracle/prysm_oracle.MDFT with the exact fp64 basis, so the rounding of the basis is included.
Inputs per shape: a seeded complex Gaussian; two coherent inputs (all ones, and the BASELINE pupil field
O.from_amp_and_phase(*O.synthetic_pupil(N)[:2], HeNe) cropped to the input shape), whose sums do not cancel the
accumulation's rounding bias and land on the output peak; and impulses at the corner, the centre and the last row and
column, against the closed form norm * outer(Ey[:, a], Ex[:, b]).  A failing figure names the worst 128 x 128 output tile,
and for a stream-K launch whether the restated partition cut that tile across CTAs.

Bounds are 1.5x the figures measured on an H100 (`MEASURED`, recorded with PB_TEST_MEASUREMENTS; the arithmetic is
deterministic) and never above 1e-6 for complex64.  Ranges of the measured rel L-inf, H100 80GB HBM3 at a 400 W power
limit (132 SMs), by the form of the tensor-core second stage, over every shape, both directions and all three switch
settings:

    split-K 2 / 4 / 8     gauss 3.1e-07-4.8e-07  ones 7.8e-08-2.9e-07  pupil 3.0e-07-5.0e-07  impulses 2.7e-07-4.2e-07
    stream-K              gauss 3.8e-07-5.0e-07  ones 1.1e-07-3.0e-07  pupil 3.6e-07-5.3e-07  impulses 2.9e-07-4.2e-07
    C3 (4096^2 -> 512^2)  forward 1.2e-07 (ones) to 4.5e-07 (gauss); adjoint up to 5.3e-07 (pupil, stream-K in both stages)
    CUDA-core, complex64  cgemm 3.4e-07-4.7e-07; executor gauss 3.2e-07-4.8e-07, ones up to 9.5e-07 (4000^2 <- 500^2
                          adjoint: the 500-term fp32 sums of a coherent input, the largest figure of the file)
    CUDA-core, complex128 cgemm 3.5e-16-2.0e-15 (one case against a long-double reference: 5.0e-16, the complex128
                          reference itself 3.5e-16); pb_mdft_apply 8.0e-16-3.8e-15
    basis (absolute)      complex64 1.4e-07, complex128 1.4e-16, at phases up to 1e5 turns

Every call must launch exactly the kernels tests/test_host_mdft_routes.py predicts for the device's SM count -- the
per-route counters of pb_route_launch_count (PB_ROUTE_MDFT_TC, PB_ROUTE_MDFT_REDUCE, PB_ROUTE_CGEMM) -- and nothing else.
PB_MDFT_STREAMK is read once per process, so the executor cases run again in child processes under PB_MDFT_STREAMK=0
and =2 (only the shapes whose kernels change).  The last test asserts that every tensor-core (stage, form, pieces), the
reduce kernel, all 32 cgemm_kernel instantiations and the four pb_mdft_apply branches in both dtypes were hit by a case
checked here."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import prysm_oracle as O
import test_host_mdft_routes as R
from accuracy import Ledger, rel_l2
from conftest import ROOT, rel_linf, within
from gpu_fixtures import pb, crand, host, routes_of, sm_count  # noqa: F401

pytestmark = pytest.mark.gpu

HeNe = 0.6328
NORM = 0.37                  # not 1, not a power of two
NORTH_STAR = 1e-6
TILE = 128
CHILD = os.environ.get('PB_MDFT_TEST_CHILD')          # '0' / '2': a child run under PB_MDFT_STREAMK = CHILD
STREAMK = int(CHILD) if CHILD else 1
CHUNK = max(1, int(os.environ.get('PB_MDFT_CHUNK', '2')))
SUFFIX = f'@streamk{CHILD}' if CHILD else ''
CHILD_TIMEOUT = 1200

# ---- measured figures (H100); bounds are 1.5x these, capped at 1e-6 for complex64 -----------------------------------
MEASURED = {
    'cgemm/c128/00': dict(linf=1.25e-15, l2=1.06e-15),
    'cgemm/c128/01': dict(linf=1.03e-15, l2=9.79e-16),
    'cgemm/c128/02': dict(linf=1.05e-15, l2=9.63e-16),
    'cgemm/c128/03': dict(linf=1.67e-15, l2=1.29e-15),
    'cgemm/c128/10': dict(linf=1.63e-15, l2=1.29e-15),
    'cgemm/c128/11': dict(linf=1.58e-15, l2=1.11e-15),
    'cgemm/c128/12': dict(linf=1.69e-15, l2=1.1e-15),
    'cgemm/c128/13': dict(linf=1.95e-15, l2=1.41e-15),
    'cgemm/c128/20': dict(linf=1.95e-15, l2=1.41e-15),
    'cgemm/c128/21': dict(linf=1.69e-15, l2=1.1e-15),
    'cgemm/c128/22': dict(linf=1.58e-15, l2=1.11e-15),
    'cgemm/c128/23': dict(linf=1.63e-15, l2=1.29e-15),
    'cgemm/c128/30': dict(linf=1.67e-15, l2=1.29e-15),
    'cgemm/c128/31': dict(linf=1.05e-15, l2=9.63e-16),
    'cgemm/c128/32': dict(linf=1.03e-15, l2=9.79e-16),
    'cgemm/c128/33': dict(linf=1.25e-15, l2=1.06e-15),
    'cgemm/c128/longdouble/device': dict(linf=5.03e-16),
    'cgemm/c64/00': dict(linf=4.52e-07, l2=2.53e-07),
    'cgemm/c64/01': dict(linf=4.54e-07, l2=2.89e-07),
    'cgemm/c64/02': dict(linf=4.18e-07, l2=2.58e-07),
    'cgemm/c64/03': dict(linf=4.27e-07, l2=2.64e-07),
    'cgemm/c64/10': dict(linf=3.39e-07, l2=2.53e-07),
    'cgemm/c64/11': dict(linf=4e-07, l2=2.57e-07),
    'cgemm/c64/12': dict(linf=4.7e-07, l2=2.56e-07),
    'cgemm/c64/13': dict(linf=4.69e-07, l2=2.99e-07),
    'cgemm/c64/20': dict(linf=4.69e-07, l2=2.99e-07),
    'cgemm/c64/21': dict(linf=4.7e-07, l2=2.56e-07),
    'cgemm/c64/22': dict(linf=4e-07, l2=2.57e-07),
    'cgemm/c64/23': dict(linf=3.39e-07, l2=2.53e-07),
    'cgemm/c64/30': dict(linf=4.27e-07, l2=2.64e-07),
    'cgemm/c64/31': dict(linf=4.18e-07, l2=2.58e-07),
    'cgemm/c64/32': dict(linf=4.54e-07, l2=2.89e-07),
    'cgemm/c64/33': dict(linf=4.52e-07, l2=2.53e-07),
    'mdft/1024x1024x1024x1024/adjoint/gauss/e2e': dict(linf=3.98e-07, l2=3.65e-07),
    'mdft/1024x1024x1024x1024/adjoint/gauss/e2e@streamk2': dict(linf=4.81e-07, l2=3.65e-07),
    'mdft/1024x1024x1024x1024/adjoint/gauss/gemm': dict(linf=4.05e-07, l2=3.6e-07),
    'mdft/1024x1024x1024x1024/adjoint/gauss/gemm@streamk2': dict(linf=4.88e-07, l2=3.6e-07),
    'mdft/1024x1024x1024x1024/adjoint/impulse/e2e': dict(linf=3.49e-07, l2=9.56e-08),
    'mdft/1024x1024x1024x1024/adjoint/impulse/e2e@streamk2': dict(linf=3.49e-07, l2=9.56e-08),
    'mdft/1024x1024x1024x1024/adjoint/impulse/gemm': dict(linf=3.25e-07, l2=7.51e-08),
    'mdft/1024x1024x1024x1024/adjoint/impulse/gemm@streamk2': dict(linf=3.25e-07, l2=7.51e-08),
    'mdft/1024x1024x1024x1024/adjoint/ones/e2e': dict(linf=1.06e-07, l2=1.7e-07),
    'mdft/1024x1024x1024x1024/adjoint/ones/e2e@streamk2': dict(linf=1.62e-07, l2=1.76e-07),
    'mdft/1024x1024x1024x1024/adjoint/ones/gemm': dict(linf=1.06e-07, l2=1.63e-07),
    'mdft/1024x1024x1024x1024/adjoint/ones/gemm@streamk2': dict(linf=1.62e-07, l2=1.69e-07),
    'mdft/1024x1024x1024x1024/adjoint/pupil/e2e': dict(linf=3.69e-07, l2=4.01e-07),
    'mdft/1024x1024x1024x1024/adjoint/pupil/e2e@streamk2': dict(linf=3.64e-07, l2=3.98e-07),
    'mdft/1024x1024x1024x1024/adjoint/pupil/gemm': dict(linf=3.7e-07, l2=3.99e-07),
    'mdft/1024x1024x1024x1024/adjoint/pupil/gemm@streamk2': dict(linf=3.67e-07, l2=3.97e-07),
    'mdft/1024x1024x1024x1024/forward/gauss/e2e': dict(linf=3.98e-07, l2=3.65e-07),
    'mdft/1024x1024x1024x1024/forward/gauss/e2e@streamk2': dict(linf=4.38e-07, l2=3.65e-07),
    'mdft/1024x1024x1024x1024/forward/gauss/gemm': dict(linf=4.05e-07, l2=3.6e-07),
    'mdft/1024x1024x1024x1024/forward/gauss/gemm@streamk2': dict(linf=4.24e-07, l2=3.6e-07),
    'mdft/1024x1024x1024x1024/forward/impulse/e2e': dict(linf=3.49e-07, l2=9.56e-08),
    'mdft/1024x1024x1024x1024/forward/impulse/e2e@streamk2': dict(linf=3.49e-07, l2=9.56e-08),
    'mdft/1024x1024x1024x1024/forward/impulse/gemm': dict(linf=3.25e-07, l2=7.51e-08),
    'mdft/1024x1024x1024x1024/forward/impulse/gemm@streamk2': dict(linf=3.25e-07, l2=7.51e-08),
    'mdft/1024x1024x1024x1024/forward/ones/e2e': dict(linf=1.06e-07, l2=1.7e-07),
    'mdft/1024x1024x1024x1024/forward/ones/e2e@streamk2': dict(linf=1.62e-07, l2=1.76e-07),
    'mdft/1024x1024x1024x1024/forward/ones/gemm': dict(linf=1.06e-07, l2=1.63e-07),
    'mdft/1024x1024x1024x1024/forward/ones/gemm@streamk2': dict(linf=1.62e-07, l2=1.69e-07),
    'mdft/1024x1024x1024x1024/forward/pupil/e2e': dict(linf=3.69e-07, l2=4.01e-07),
    'mdft/1024x1024x1024x1024/forward/pupil/e2e@streamk2': dict(linf=4.06e-07, l2=4.04e-07),
    'mdft/1024x1024x1024x1024/forward/pupil/gemm': dict(linf=3.7e-07, l2=3.99e-07),
    'mdft/1024x1024x1024x1024/forward/pupil/gemm@streamk2': dict(linf=4.07e-07, l2=4.02e-07),
    'mdft/128x256x128x256/adjoint/gauss/e2e': dict(linf=3.9e-07, l2=3.48e-07),
    'mdft/128x256x128x256/adjoint/gauss/gemm': dict(linf=3.94e-07, l2=3.43e-07),
    'mdft/128x256x128x256/adjoint/impulse/e2e': dict(linf=3.62e-07, l2=9.87e-08),
    'mdft/128x256x128x256/adjoint/impulse/gemm': dict(linf=2.9e-07, l2=7.61e-08),
    'mdft/128x256x128x256/adjoint/ones/e2e': dict(linf=2.2e-07, l2=1.94e-07),
    'mdft/128x256x128x256/adjoint/ones/gemm': dict(linf=2.24e-07, l2=1.87e-07),
    'mdft/128x256x128x256/adjoint/pupil/e2e': dict(linf=4.84e-07, l2=3.54e-07),
    'mdft/128x256x128x256/adjoint/pupil/gemm': dict(linf=4.89e-07, l2=3.53e-07),
    'mdft/128x256x128x256/forward/gauss/e2e': dict(linf=3.14e-07, l2=3.49e-07),
    'mdft/128x256x128x256/forward/gauss/gemm': dict(linf=3.16e-07, l2=3.43e-07),
    'mdft/128x256x128x256/forward/impulse/e2e': dict(linf=3.14e-07, l2=9.36e-08),
    'mdft/128x256x128x256/forward/impulse/gemm': dict(linf=2.7e-07, l2=7.11e-08),
    'mdft/128x256x128x256/forward/ones/e2e': dict(linf=1.44e-07, l2=1.81e-07),
    'mdft/128x256x128x256/forward/ones/gemm': dict(linf=1.45e-07, l2=1.75e-07),
    'mdft/128x256x128x256/forward/pupil/e2e': dict(linf=3.74e-07, l2=3.67e-07),
    'mdft/128x256x128x256/forward/pupil/gemm': dict(linf=3.76e-07, l2=3.68e-07),
    'mdft/256x1024x640x1024/adjoint/gauss/e2e': dict(linf=4.09e-07, l2=3.57e-07),
    'mdft/256x1024x640x1024/adjoint/gauss/e2e@streamk0': dict(linf=4.09e-07, l2=3.57e-07),
    'mdft/256x1024x640x1024/adjoint/gauss/e2e@streamk2': dict(linf=4.51e-07, l2=3.52e-07),
    'mdft/256x1024x640x1024/adjoint/gauss/gemm': dict(linf=3.98e-07, l2=3.52e-07),
    'mdft/256x1024x640x1024/adjoint/gauss/gemm@streamk0': dict(linf=3.98e-07, l2=3.52e-07),
    'mdft/256x1024x640x1024/adjoint/gauss/gemm@streamk2': dict(linf=4.25e-07, l2=3.46e-07),
    'mdft/256x1024x640x1024/adjoint/impulse/e2e': dict(linf=3.66e-07, l2=9.44e-08),
    'mdft/256x1024x640x1024/adjoint/impulse/e2e@streamk0': dict(linf=3.66e-07, l2=9.44e-08),
    'mdft/256x1024x640x1024/adjoint/impulse/e2e@streamk2': dict(linf=3.66e-07, l2=9.44e-08),
    'mdft/256x1024x640x1024/adjoint/impulse/gemm': dict(linf=3.42e-07, l2=7.34e-08),
    'mdft/256x1024x640x1024/adjoint/impulse/gemm@streamk0': dict(linf=3.42e-07, l2=7.34e-08),
    'mdft/256x1024x640x1024/adjoint/impulse/gemm@streamk2': dict(linf=3.42e-07, l2=7.34e-08),
    'mdft/256x1024x640x1024/adjoint/ones/e2e': dict(linf=1.23e-07, l2=1.74e-07),
    'mdft/256x1024x640x1024/adjoint/ones/e2e@streamk0': dict(linf=1.23e-07, l2=1.74e-07),
    'mdft/256x1024x640x1024/adjoint/ones/e2e@streamk2': dict(linf=1.73e-07, l2=1.74e-07),
    'mdft/256x1024x640x1024/adjoint/ones/gemm': dict(linf=1.22e-07, l2=1.67e-07),
    'mdft/256x1024x640x1024/adjoint/ones/gemm@streamk0': dict(linf=1.22e-07, l2=1.67e-07),
    'mdft/256x1024x640x1024/adjoint/ones/gemm@streamk2': dict(linf=1.74e-07, l2=1.67e-07),
    'mdft/256x1024x640x1024/adjoint/out_plane2/e2e': dict(linf=4.19e-07, l2=3.56e-07),
    'mdft/256x1024x640x1024/adjoint/pupil/e2e': dict(linf=4.44e-07, l2=3.96e-07),
    'mdft/256x1024x640x1024/adjoint/pupil/e2e@streamk0': dict(linf=4.44e-07, l2=3.96e-07),
    'mdft/256x1024x640x1024/adjoint/pupil/e2e@streamk2': dict(linf=4.44e-07, l2=3.95e-07),
    'mdft/256x1024x640x1024/adjoint/pupil/gemm': dict(linf=4.44e-07, l2=3.95e-07),
    'mdft/256x1024x640x1024/adjoint/pupil/gemm@streamk0': dict(linf=4.44e-07, l2=3.95e-07),
    'mdft/256x1024x640x1024/adjoint/pupil/gemm@streamk2': dict(linf=4.45e-07, l2=3.93e-07),
    'mdft/256x1024x640x1024/forward/gauss/e2e': dict(linf=4.24e-07, l2=3.57e-07),
    'mdft/256x1024x640x1024/forward/gauss/e2e@streamk0': dict(linf=3.74e-07, l2=3.63e-07),
    'mdft/256x1024x640x1024/forward/gauss/e2e@streamk2': dict(linf=4.22e-07, l2=3.57e-07),
    'mdft/256x1024x640x1024/forward/gauss/gemm': dict(linf=4.03e-07, l2=3.52e-07),
    'mdft/256x1024x640x1024/forward/gauss/gemm@streamk0': dict(linf=3.75e-07, l2=3.58e-07),
    'mdft/256x1024x640x1024/forward/gauss/gemm@streamk2': dict(linf=4.01e-07, l2=3.52e-07),
    'mdft/256x1024x640x1024/forward/impulse/e2e': dict(linf=3.49e-07, l2=9.75e-08),
    'mdft/256x1024x640x1024/forward/impulse/e2e@streamk0': dict(linf=3.49e-07, l2=9.75e-08),
    'mdft/256x1024x640x1024/forward/impulse/e2e@streamk2': dict(linf=3.49e-07, l2=9.75e-08),
    'mdft/256x1024x640x1024/forward/impulse/gemm': dict(linf=3.25e-07, l2=7.63e-08),
    'mdft/256x1024x640x1024/forward/impulse/gemm@streamk0': dict(linf=3.25e-07, l2=7.63e-08),
    'mdft/256x1024x640x1024/forward/impulse/gemm@streamk2': dict(linf=3.25e-07, l2=7.63e-08),
    'mdft/256x1024x640x1024/forward/ones/e2e': dict(linf=1.06e-07, l2=1.6e-07),
    'mdft/256x1024x640x1024/forward/ones/e2e@streamk0': dict(linf=1.06e-07, l2=1.6e-07),
    'mdft/256x1024x640x1024/forward/ones/e2e@streamk2': dict(linf=1.09e-07, l2=1.62e-07),
    'mdft/256x1024x640x1024/forward/ones/gemm': dict(linf=1.06e-07, l2=1.58e-07),
    'mdft/256x1024x640x1024/forward/ones/gemm@streamk0': dict(linf=1.06e-07, l2=1.57e-07),
    'mdft/256x1024x640x1024/forward/ones/gemm@streamk2': dict(linf=1.09e-07, l2=1.6e-07),
    'mdft/256x1024x640x1024/forward/out_plane2/e2e': dict(linf=4.33e-07, l2=3.58e-07),
    'mdft/256x1024x640x1024/forward/pupil/e2e': dict(linf=3.69e-07, l2=3.88e-07),
    'mdft/256x1024x640x1024/forward/pupil/e2e@streamk0': dict(linf=3.69e-07, l2=3.88e-07),
    'mdft/256x1024x640x1024/forward/pupil/e2e@streamk2': dict(linf=3.58e-07, l2=3.84e-07),
    'mdft/256x1024x640x1024/forward/pupil/gemm': dict(linf=3.7e-07, l2=3.88e-07),
    'mdft/256x1024x640x1024/forward/pupil/gemm@streamk0': dict(linf=3.7e-07, l2=3.88e-07),
    'mdft/256x1024x640x1024/forward/pupil/gemm@streamk2': dict(linf=3.6e-07, l2=3.84e-07),
    'mdft/256x128x384x16/adjoint/gauss/e2e': dict(linf=3.83e-07, l2=3.03e-07),
    'mdft/256x128x384x16/adjoint/gauss/gemm': dict(linf=3.79e-07, l2=2.95e-07),
    'mdft/256x128x384x16/adjoint/impulse/e2e': dict(linf=2.28e-07, l2=7.58e-08),
    'mdft/256x128x384x16/adjoint/impulse/gemm': dict(linf=1.14e-07, l2=3.93e-08),
    'mdft/256x128x384x16/adjoint/ones/e2e': dict(linf=3.65e-08, l2=9.85e-08),
    'mdft/256x128x384x16/adjoint/ones/gemm': dict(linf=3.66e-08, l2=9.48e-08),
    'mdft/256x128x384x16/adjoint/pupil/e2e': dict(linf=8.46e-08, l2=1.87e-07),
    'mdft/256x128x384x16/adjoint/pupil/gemm': dict(linf=8.29e-08, l2=1.82e-07),
    'mdft/256x128x384x16/forward/gauss/e2e': dict(linf=3.95e-07, l2=2.83e-07),
    'mdft/256x128x384x16/forward/gauss/gemm': dict(linf=3.72e-07, l2=2.74e-07),
    'mdft/256x128x384x16/forward/impulse/e2e': dict(linf=3.39e-07, l2=9.51e-08),
    'mdft/256x128x384x16/forward/impulse/gemm': dict(linf=2.9e-07, l2=7.21e-08),
    'mdft/256x128x384x16/forward/ones/e2e': dict(linf=2.39e-07, l2=2e-07),
    'mdft/256x128x384x16/forward/ones/gemm': dict(linf=2.45e-07, l2=1.86e-07),
    'mdft/256x128x384x16/forward/pupil/e2e': dict(linf=3.59e-07, l2=2.88e-07),
    'mdft/256x128x384x16/forward/pupil/gemm': dict(linf=3.61e-07, l2=2.78e-07),
    'mdft/256x8192x128x256/adjoint/gauss/e2e': dict(linf=4.47e-07, l2=3.49e-07),
    'mdft/256x8192x128x256/adjoint/gauss/e2e@streamk2': dict(linf=4.9e-07, l2=3.49e-07),
    'mdft/256x8192x128x256/adjoint/gauss/gemm': dict(linf=4.45e-07, l2=3.43e-07),
    'mdft/256x8192x128x256/adjoint/gauss/gemm@streamk2': dict(linf=5.02e-07, l2=3.44e-07),
    'mdft/256x8192x128x256/adjoint/impulse/e2e': dict(linf=3.62e-07, l2=9.53e-08),
    'mdft/256x8192x128x256/adjoint/impulse/e2e@streamk2': dict(linf=3.62e-07, l2=9.53e-08),
    'mdft/256x8192x128x256/adjoint/impulse/gemm': dict(linf=3.25e-07, l2=7.5e-08),
    'mdft/256x8192x128x256/adjoint/impulse/gemm@streamk2': dict(linf=3.25e-07, l2=7.5e-08),
    'mdft/256x8192x128x256/adjoint/ones/e2e': dict(linf=2.27e-07, l2=2.14e-07),
    'mdft/256x8192x128x256/adjoint/ones/e2e@streamk2': dict(linf=3.02e-07, l2=2.16e-07),
    'mdft/256x8192x128x256/adjoint/ones/gemm': dict(linf=2.28e-07, l2=2.08e-07),
    'mdft/256x8192x128x256/adjoint/ones/gemm@streamk2': dict(linf=3.04e-07, l2=2.1e-07),
    'mdft/256x8192x128x256/adjoint/pupil/e2e': dict(linf=4.77e-07, l2=3.97e-07),
    'mdft/256x8192x128x256/adjoint/pupil/e2e@streamk2': dict(linf=5.18e-07, l2=4e-07),
    'mdft/256x8192x128x256/adjoint/pupil/gemm': dict(linf=4.84e-07, l2=3.95e-07),
    'mdft/256x8192x128x256/adjoint/pupil/gemm@streamk2': dict(linf=5.23e-07, l2=3.98e-07),
    'mdft/256x8192x128x256/forward/gauss/e2e': dict(linf=4.4e-07, l2=3.63e-07),
    'mdft/256x8192x128x256/forward/gauss/e2e@streamk2': dict(linf=4.54e-07, l2=3.63e-07),
    'mdft/256x8192x128x256/forward/gauss/gemm': dict(linf=4.35e-07, l2=3.57e-07),
    'mdft/256x8192x128x256/forward/gauss/gemm@streamk2': dict(linf=4.44e-07, l2=3.57e-07),
    'mdft/256x8192x128x256/forward/impulse/e2e': dict(linf=2.99e-07, l2=9.2e-08),
    'mdft/256x8192x128x256/forward/impulse/e2e@streamk2': dict(linf=2.99e-07, l2=9.2e-08),
    'mdft/256x8192x128x256/forward/impulse/gemm': dict(linf=2.9e-07, l2=7.34e-08),
    'mdft/256x8192x128x256/forward/impulse/gemm@streamk2': dict(linf=2.9e-07, l2=7.34e-08),
    'mdft/256x8192x128x256/forward/ones/e2e': dict(linf=1.3e-07, l2=1.59e-07),
    'mdft/256x8192x128x256/forward/ones/e2e@streamk2': dict(linf=1.14e-07, l2=1.7e-07),
    'mdft/256x8192x128x256/forward/ones/gemm': dict(linf=1.29e-07, l2=1.57e-07),
    'mdft/256x8192x128x256/forward/ones/gemm@streamk2': dict(linf=1.13e-07, l2=1.67e-07),
    'mdft/384x384x128x48/adjoint/gauss/e2e': dict(linf=3.19e-07, l2=3e-07),
    'mdft/384x384x128x48/adjoint/gauss/gemm': dict(linf=3.25e-07, l2=2.93e-07),
    'mdft/384x384x128x48/adjoint/impulse/e2e': dict(linf=2.43e-07, l2=7.61e-08),
    'mdft/384x384x128x48/adjoint/impulse/gemm': dict(linf=1.14e-07, l2=4.15e-08),
    'mdft/384x384x128x48/adjoint/ones/e2e': dict(linf=9.68e-08, l2=2.21e-07),
    'mdft/384x384x128x48/adjoint/ones/gemm': dict(linf=9.47e-08, l2=2.14e-07),
    'mdft/384x384x128x48/adjoint/pupil/e2e': dict(linf=1.77e-07, l2=2.55e-07),
    'mdft/384x384x128x48/adjoint/pupil/gemm': dict(linf=1.78e-07, l2=2.52e-07),
    'mdft/384x384x128x48/forward/gauss/e2e': dict(linf=3.77e-07, l2=3.28e-07),
    'mdft/384x384x128x48/forward/gauss/gemm': dict(linf=3.61e-07, l2=3.21e-07),
    'mdft/384x384x128x48/forward/impulse/e2e': dict(linf=3.43e-07, l2=9.73e-08),
    'mdft/384x384x128x48/forward/impulse/gemm': dict(linf=2.75e-07, l2=7.27e-08),
    'mdft/384x384x128x48/forward/ones/e2e': dict(linf=1.12e-07, l2=1.66e-07),
    'mdft/384x384x128x48/forward/ones/gemm': dict(linf=1.13e-07, l2=1.54e-07),
    'mdft/384x384x128x48/forward/pupil/e2e': dict(linf=2.99e-07, l2=3.24e-07),
    'mdft/384x384x128x48/forward/pupil/gemm': dict(linf=3.02e-07, l2=3.19e-07),
    'mdft/500x4000x500x4000/adjoint/gauss/e2e': dict(linf=3.97e-07, l2=3.04e-07),
    'mdft/500x4000x500x4000/adjoint/gauss/gemm': dict(linf=3.84e-07, l2=2.97e-07),
    'mdft/500x4000x500x4000/adjoint/ones/e2e': dict(linf=9.45e-07, l2=2.93e-07),
    'mdft/500x4000x500x4000/adjoint/ones/gemm': dict(linf=9.45e-07, l2=2.89e-07),
    'mdft/500x4000x500x4000/forward/gauss/e2e': dict(linf=4.57e-07, l2=3.61e-07),
    'mdft/500x4000x500x4000/forward/gauss/gemm': dict(linf=4.78e-07, l2=3.55e-07),
    'mdft/500x4000x500x4000/forward/ones/e2e': dict(linf=2.14e-07, l2=3.35e-07),
    'mdft/500x4000x500x4000/forward/ones/gemm': dict(linf=2.14e-07, l2=3.35e-07),
    'mdft/512x1024x512x1024/adjoint/gauss/e2e': dict(linf=3.82e-07, l2=3.53e-07),
    'mdft/512x1024x512x1024/adjoint/gauss/e2e@streamk0': dict(linf=4.72e-07, l2=3.57e-07),
    'mdft/512x1024x512x1024/adjoint/gauss/e2e@streamk2': dict(linf=3.91e-07, l2=3.54e-07),
    'mdft/512x1024x512x1024/adjoint/gauss/gemm': dict(linf=3.83e-07, l2=3.48e-07),
    'mdft/512x1024x512x1024/adjoint/gauss/gemm@streamk0': dict(linf=4.82e-07, l2=3.52e-07),
    'mdft/512x1024x512x1024/adjoint/gauss/gemm@streamk2': dict(linf=3.85e-07, l2=3.49e-07),
    'mdft/512x1024x512x1024/adjoint/impulse/e2e': dict(linf=4.04e-07, l2=9.84e-08),
    'mdft/512x1024x512x1024/adjoint/impulse/e2e@streamk0': dict(linf=4.04e-07, l2=9.84e-08),
    'mdft/512x1024x512x1024/adjoint/impulse/e2e@streamk2': dict(linf=4.04e-07, l2=9.84e-08),
    'mdft/512x1024x512x1024/adjoint/impulse/gemm': dict(linf=3.22e-07, l2=7.66e-08),
    'mdft/512x1024x512x1024/adjoint/impulse/gemm@streamk0': dict(linf=3.22e-07, l2=7.66e-08),
    'mdft/512x1024x512x1024/adjoint/impulse/gemm@streamk2': dict(linf=3.22e-07, l2=7.66e-08),
    'mdft/512x1024x512x1024/adjoint/ones/e2e': dict(linf=2.7e-07, l2=2.2e-07),
    'mdft/512x1024x512x1024/adjoint/ones/e2e@streamk0': dict(linf=2.7e-07, l2=2.16e-07),
    'mdft/512x1024x512x1024/adjoint/ones/e2e@streamk2': dict(linf=2.68e-07, l2=2.13e-07),
    'mdft/512x1024x512x1024/adjoint/ones/gemm': dict(linf=2.7e-07, l2=2.15e-07),
    'mdft/512x1024x512x1024/adjoint/ones/gemm@streamk0': dict(linf=2.7e-07, l2=2.11e-07),
    'mdft/512x1024x512x1024/adjoint/ones/gemm@streamk2': dict(linf=2.68e-07, l2=2.08e-07),
    'mdft/512x1024x512x1024/adjoint/pupil/e2e': dict(linf=4.36e-07, l2=3.98e-07),
    'mdft/512x1024x512x1024/adjoint/pupil/e2e@streamk0': dict(linf=4.36e-07, l2=4e-07),
    'mdft/512x1024x512x1024/adjoint/pupil/e2e@streamk2': dict(linf=4.23e-07, l2=3.97e-07),
    'mdft/512x1024x512x1024/adjoint/pupil/gemm': dict(linf=4.36e-07, l2=3.97e-07),
    'mdft/512x1024x512x1024/adjoint/pupil/gemm@streamk0': dict(linf=4.36e-07, l2=3.99e-07),
    'mdft/512x1024x512x1024/adjoint/pupil/gemm@streamk2': dict(linf=4.22e-07, l2=3.96e-07),
    'mdft/512x1024x512x1024/forward/gauss/e2e': dict(linf=3.84e-07, l2=3.57e-07),
    'mdft/512x1024x512x1024/forward/gauss/e2e@streamk0': dict(linf=3.94e-07, l2=3.65e-07),
    'mdft/512x1024x512x1024/forward/gauss/e2e@streamk2': dict(linf=4.03e-07, l2=3.57e-07),
    'mdft/512x1024x512x1024/forward/gauss/gemm': dict(linf=3.73e-07, l2=3.52e-07),
    'mdft/512x1024x512x1024/forward/gauss/gemm@streamk0': dict(linf=3.93e-07, l2=3.6e-07),
    'mdft/512x1024x512x1024/forward/gauss/gemm@streamk2': dict(linf=3.91e-07, l2=3.52e-07),
    'mdft/512x1024x512x1024/forward/impulse/e2e': dict(linf=3.49e-07, l2=9.54e-08),
    'mdft/512x1024x512x1024/forward/impulse/e2e@streamk0': dict(linf=3.49e-07, l2=9.54e-08),
    'mdft/512x1024x512x1024/forward/impulse/e2e@streamk2': dict(linf=3.49e-07, l2=9.54e-08),
    'mdft/512x1024x512x1024/forward/impulse/gemm': dict(linf=3.25e-07, l2=7.56e-08),
    'mdft/512x1024x512x1024/forward/impulse/gemm@streamk0': dict(linf=3.25e-07, l2=7.56e-08),
    'mdft/512x1024x512x1024/forward/impulse/gemm@streamk2': dict(linf=3.25e-07, l2=7.56e-08),
    'mdft/512x1024x512x1024/forward/misaligned/e2e': dict(linf=3.68e-07, l2=3.57e-07),
    'mdft/512x1024x512x1024/forward/ones/e2e': dict(linf=1.06e-07, l2=1.63e-07),
    'mdft/512x1024x512x1024/forward/ones/e2e@streamk0': dict(linf=1.06e-07, l2=1.63e-07),
    'mdft/512x1024x512x1024/forward/ones/e2e@streamk2': dict(linf=1.06e-07, l2=1.61e-07),
    'mdft/512x1024x512x1024/forward/ones/gemm': dict(linf=1.06e-07, l2=1.6e-07),
    'mdft/512x1024x512x1024/forward/ones/gemm@streamk0': dict(linf=1.06e-07, l2=1.6e-07),
    'mdft/512x1024x512x1024/forward/ones/gemm@streamk2': dict(linf=1.06e-07, l2=1.58e-07),
    'mdft/512x1024x512x1024/forward/pupil/e2e': dict(linf=3.69e-07, l2=3.91e-07),
    'mdft/512x1024x512x1024/forward/pupil/e2e@streamk0': dict(linf=3.69e-07, l2=3.92e-07),
    'mdft/512x1024x512x1024/forward/pupil/e2e@streamk2': dict(linf=4.06e-07, l2=3.88e-07),
    'mdft/512x1024x512x1024/forward/pupil/gemm': dict(linf=3.7e-07, l2=3.91e-07),
    'mdft/512x1024x512x1024/forward/pupil/gemm@streamk0': dict(linf=3.7e-07, l2=3.92e-07),
    'mdft/512x1024x512x1024/forward/pupil/gemm@streamk2': dict(linf=4.07e-07, l2=3.88e-07),
    'mdft/512x2048x768x2048/adjoint/gauss/e2e': dict(linf=4.2e-07, l2=3.6e-07),
    'mdft/512x2048x768x2048/adjoint/gauss/e2e@streamk0': dict(linf=4.2e-07, l2=3.6e-07),
    'mdft/512x2048x768x2048/adjoint/gauss/e2e@streamk2': dict(linf=4.46e-07, l2=3.59e-07),
    'mdft/512x2048x768x2048/adjoint/gauss/gemm': dict(linf=4.19e-07, l2=3.55e-07),
    'mdft/512x2048x768x2048/adjoint/gauss/gemm@streamk0': dict(linf=4.19e-07, l2=3.55e-07),
    'mdft/512x2048x768x2048/adjoint/gauss/gemm@streamk2': dict(linf=4.4e-07, l2=3.54e-07),
    'mdft/512x2048x768x2048/adjoint/impulse/e2e': dict(linf=3.79e-07, l2=9.43e-08),
    'mdft/512x2048x768x2048/adjoint/impulse/e2e@streamk0': dict(linf=3.79e-07, l2=9.43e-08),
    'mdft/512x2048x768x2048/adjoint/impulse/e2e@streamk2': dict(linf=3.79e-07, l2=9.43e-08),
    'mdft/512x2048x768x2048/adjoint/impulse/gemm': dict(linf=3.42e-07, l2=7.49e-08),
    'mdft/512x2048x768x2048/adjoint/impulse/gemm@streamk0': dict(linf=3.42e-07, l2=7.49e-08),
    'mdft/512x2048x768x2048/adjoint/impulse/gemm@streamk2': dict(linf=3.42e-07, l2=7.49e-08),
    'mdft/512x2048x768x2048/adjoint/ones/e2e': dict(linf=2.85e-07, l2=2.09e-07),
    'mdft/512x2048x768x2048/adjoint/ones/e2e@streamk0': dict(linf=2.85e-07, l2=2.09e-07),
    'mdft/512x2048x768x2048/adjoint/ones/e2e@streamk2': dict(linf=1.98e-07, l2=2.02e-07),
    'mdft/512x2048x768x2048/adjoint/ones/gemm': dict(linf=2.86e-07, l2=2.04e-07),
    'mdft/512x2048x768x2048/adjoint/ones/gemm@streamk0': dict(linf=2.86e-07, l2=2.04e-07),
    'mdft/512x2048x768x2048/adjoint/ones/gemm@streamk2': dict(linf=1.97e-07, l2=1.96e-07),
    'mdft/512x2048x768x2048/adjoint/pupil/e2e': dict(linf=4.3e-07, l2=4.07e-07),
    'mdft/512x2048x768x2048/adjoint/pupil/e2e@streamk0': dict(linf=4.3e-07, l2=4.07e-07),
    'mdft/512x2048x768x2048/adjoint/pupil/e2e@streamk2': dict(linf=4.6e-07, l2=4.1e-07),
    'mdft/512x2048x768x2048/adjoint/pupil/gemm': dict(linf=4.3e-07, l2=4.06e-07),
    'mdft/512x2048x768x2048/adjoint/pupil/gemm@streamk0': dict(linf=4.3e-07, l2=4.06e-07),
    'mdft/512x2048x768x2048/adjoint/pupil/gemm@streamk2': dict(linf=4.62e-07, l2=4.08e-07),
    'mdft/512x2048x768x2048/forward/gauss/e2e': dict(linf=4.61e-07, l2=3.84e-07),
    'mdft/512x2048x768x2048/forward/gauss/e2e@streamk0': dict(linf=4.15e-07, l2=3.8e-07),
    'mdft/512x2048x768x2048/forward/gauss/e2e@streamk2': dict(linf=4.16e-07, l2=3.77e-07),
    'mdft/512x2048x768x2048/forward/gauss/gemm': dict(linf=4.65e-07, l2=3.78e-07),
    'mdft/512x2048x768x2048/forward/gauss/gemm@streamk0': dict(linf=4.19e-07, l2=3.75e-07),
    'mdft/512x2048x768x2048/forward/gauss/gemm@streamk2': dict(linf=4.18e-07, l2=3.72e-07),
    'mdft/512x2048x768x2048/forward/impulse/e2e': dict(linf=4.05e-07, l2=9.54e-08),
    'mdft/512x2048x768x2048/forward/impulse/e2e@streamk0': dict(linf=4.05e-07, l2=9.54e-08),
    'mdft/512x2048x768x2048/forward/impulse/e2e@streamk2': dict(linf=4.05e-07, l2=9.54e-08),
    'mdft/512x2048x768x2048/forward/impulse/gemm': dict(linf=3.22e-07, l2=7.39e-08),
    'mdft/512x2048x768x2048/forward/impulse/gemm@streamk0': dict(linf=3.22e-07, l2=7.39e-08),
    'mdft/512x2048x768x2048/forward/impulse/gemm@streamk2': dict(linf=3.22e-07, l2=7.39e-08),
    'mdft/512x2048x768x2048/forward/ones/e2e': dict(linf=1.22e-07, l2=1.62e-07),
    'mdft/512x2048x768x2048/forward/ones/e2e@streamk0': dict(linf=7.82e-08, l2=1.54e-07),
    'mdft/512x2048x768x2048/forward/ones/e2e@streamk2': dict(linf=1.22e-07, l2=1.62e-07),
    'mdft/512x2048x768x2048/forward/ones/gemm': dict(linf=1.22e-07, l2=1.6e-07),
    'mdft/512x2048x768x2048/forward/ones/gemm@streamk0': dict(linf=7.83e-08, l2=1.52e-07),
    'mdft/512x2048x768x2048/forward/ones/gemm@streamk2': dict(linf=1.22e-07, l2=1.61e-07),
    'mdft/512x2048x768x2048/forward/pupil/e2e': dict(linf=3.75e-07, l2=3.92e-07),
    'mdft/512x2048x768x2048/forward/pupil/e2e@streamk0': dict(linf=4.05e-07, l2=3.9e-07),
    'mdft/512x2048x768x2048/forward/pupil/e2e@streamk2': dict(linf=3.75e-07, l2=3.92e-07),
    'mdft/512x2048x768x2048/forward/pupil/gemm': dict(linf=3.76e-07, l2=3.92e-07),
    'mdft/512x2048x768x2048/forward/pupil/gemm@streamk0': dict(linf=4.06e-07, l2=3.9e-07),
    'mdft/512x2048x768x2048/forward/pupil/gemm@streamk2': dict(linf=3.76e-07, l2=3.92e-07),
    'mdft/512x4096x512x4096/adjoint/gauss/e2e': dict(linf=3.96e-07, l2=3.57e-07),
    'mdft/512x4096x512x4096/adjoint/gauss/e2e@streamk2': dict(linf=4.31e-07, l2=3.58e-07),
    'mdft/512x4096x512x4096/adjoint/gauss/gemm': dict(linf=3.97e-07, l2=3.51e-07),
    'mdft/512x4096x512x4096/adjoint/gauss/gemm@streamk2': dict(linf=4.34e-07, l2=3.53e-07),
    'mdft/512x4096x512x4096/adjoint/impulse/e2e': dict(linf=4.17e-07, l2=9.42e-08),
    'mdft/512x4096x512x4096/adjoint/impulse/e2e@streamk2': dict(linf=4.17e-07, l2=9.42e-08),
    'mdft/512x4096x512x4096/adjoint/impulse/gemm': dict(linf=3.42e-07, l2=7.44e-08),
    'mdft/512x4096x512x4096/adjoint/impulse/gemm@streamk2': dict(linf=3.42e-07, l2=7.44e-08),
    'mdft/512x4096x512x4096/adjoint/ones/e2e': dict(linf=2.71e-07, l2=2.28e-07),
    'mdft/512x4096x512x4096/adjoint/ones/e2e@streamk2': dict(linf=2.86e-07, l2=2.32e-07),
    'mdft/512x4096x512x4096/adjoint/ones/gemm': dict(linf=2.73e-07, l2=2.23e-07),
    'mdft/512x4096x512x4096/adjoint/ones/gemm@streamk2': dict(linf=2.87e-07, l2=2.26e-07),
    'mdft/512x4096x512x4096/adjoint/pupil/e2e': dict(linf=4.96e-07, l2=4.05e-07),
    'mdft/512x4096x512x4096/adjoint/pupil/e2e@streamk2': dict(linf=5.27e-07, l2=4.08e-07),
    'mdft/512x4096x512x4096/adjoint/pupil/gemm': dict(linf=4.95e-07, l2=4.03e-07),
    'mdft/512x4096x512x4096/adjoint/pupil/gemm@streamk2': dict(linf=5.28e-07, l2=4.06e-07),
    'mdft/512x4096x512x4096/forward/gauss/e2e': dict(linf=4.51e-07, l2=4.08e-07),
    'mdft/512x4096x512x4096/forward/gauss/e2e@streamk2': dict(linf=4.25e-07, l2=4.04e-07),
    'mdft/512x4096x512x4096/forward/gauss/gemm': dict(linf=4.51e-07, l2=4.03e-07),
    'mdft/512x4096x512x4096/forward/gauss/gemm@streamk2': dict(linf=4.33e-07, l2=3.99e-07),
    'mdft/512x4096x512x4096/forward/impulse/e2e': dict(linf=3.73e-07, l2=9.36e-08),
    'mdft/512x4096x512x4096/forward/impulse/e2e@streamk2': dict(linf=3.73e-07, l2=9.36e-08),
    'mdft/512x4096x512x4096/forward/impulse/gemm': dict(linf=3.22e-07, l2=7.52e-08),
    'mdft/512x4096x512x4096/forward/impulse/gemm@streamk2': dict(linf=3.22e-07, l2=7.52e-08),
    'mdft/512x4096x512x4096/forward/ones/e2e': dict(linf=1.33e-07, l2=1.89e-07),
    'mdft/512x4096x512x4096/forward/ones/e2e@streamk2': dict(linf=1.23e-07, l2=1.87e-07),
    'mdft/512x4096x512x4096/forward/ones/gemm': dict(linf=1.34e-07, l2=1.88e-07),
    'mdft/512x4096x512x4096/forward/ones/gemm@streamk2': dict(linf=1.23e-07, l2=1.87e-07),
    'mdft/512x4096x512x4096/forward/pupil/e2e': dict(linf=4.2e-07, l2=3.84e-07),
    'mdft/512x4096x512x4096/forward/pupil/e2e@streamk2': dict(linf=3.94e-07, l2=3.84e-07),
    'mdft/512x4096x512x4096/forward/pupil/gemm': dict(linf=4.21e-07, l2=3.84e-07),
    'mdft/512x4096x512x4096/forward/pupil/gemm@streamk2': dict(linf=3.95e-07, l2=3.84e-07),
    'mdft_apply/c128/adjoint/left/e2e': dict(linf=3.72e-15, l2=2.48e-15),
    'mdft_apply/c128/adjoint/left/gemm': dict(linf=1.01e-15, l2=6.25e-16),
    'mdft_apply/c128/adjoint/right/e2e': dict(linf=3.79e-15, l2=2.49e-15),
    'mdft_apply/c128/adjoint/right/gemm': dict(linf=9.23e-16, l2=6.75e-16),
    'mdft_apply/c128/forward/left/e2e': dict(linf=3.35e-15, l2=2.51e-15),
    'mdft_apply/c128/forward/left/gemm': dict(linf=8.87e-16, l2=7.47e-16),
    'mdft_apply/c128/forward/right/e2e': dict(linf=3.2e-15, l2=2.51e-15),
    'mdft_apply/c128/forward/right/gemm': dict(linf=7.98e-16, l2=7.05e-16),
    'mdft_apply/c64/adjoint/left/e2e': dict(linf=4.19e-07, l2=2.93e-07),
    'mdft_apply/c64/adjoint/left/gemm': dict(linf=4.08e-07, l2=2.86e-07),
    'mdft_apply/c64/adjoint/right/e2e': dict(linf=3.55e-07, l2=2.92e-07),
    'mdft_apply/c64/adjoint/right/gemm': dict(linf=3.62e-07, l2=2.85e-07),
    'mdft_apply/c64/forward/left/e2e': dict(linf=3.34e-07, l2=2.94e-07),
    'mdft_apply/c64/forward/left/gemm': dict(linf=3.27e-07, l2=2.87e-07),
    'mdft_apply/c64/forward/right/e2e': dict(linf=3.34e-07, l2=2.95e-07),
    'mdft_apply/c64/forward/right/gemm': dict(linf=3.2e-07, l2=2.88e-07),
}


# a case's figure is the worst over its inputs, within its test.  The cap of 1e-6 is for complex64: every complex128
# figure is a few 1e-15, so it never binds there, and holds a complex128 figure with no entry to 1e-6 as well.
LEDGER = Ledger(MEASURED, NORTH_STAR, per_test=True)


def worst_tile(got, ref):
    """(row tile, column tile, max |error| there / max |ref|) of the 128 x 128 output tile with the largest error"""
    err = np.abs(got - ref)
    r, c = err.shape
    pad = np.zeros((-(-r // TILE) * TILE, -(-c // TILE) * TILE))
    pad[:r, :c] = err
    t = pad.reshape(pad.shape[0] // TILE, TILE, pad.shape[1] // TILE, TILE).max(axis=(1, 3))
    i, j = np.unravel_index(int(np.argmax(t)), t.shape)
    return int(i), int(j), float(t[i, j]) / max(float(np.abs(ref).max()), 1e-300)


def add(case, got, ref, note=None, what=''):
    """the whole array against its reference: rel_linf and the relative L2 error, each noted with its worst tile"""
    i, j, tv = worst_tile(got, ref)
    detail = f'{what}: worst 128 x 128 output tile ({i}, {j}) at {tv:.3e}'
    if note is not None:
        detail += '; ' + note(i, j)
    for k, v in (('linf', rel_linf(got, ref)), ('l2', rel_l2(got, ref))):
        LEDGER.record(f'{case}{SUFFIX}/{k}', v, detail)


# ---- which kernels ran --------------------------------------------------------------------------------------------
HIT = set()     # ('tc', stage, form, pieces), ('reduce', pieces), ('cgemm', dtype, opA, opB), ('branch', dtype, adj, lf)
ROUTE_KEYS = ([R.route_code(R.ROUTE_MDFT_TC, L, f) for L in (1, 2, 4, 8) for f in range(8)]
              + [R.route_code(R.ROUTE_MDFT_REDUCE, L) for L in (1, 2, 4, 8)]
              + [R.cgemm_code(d, a, b) for d in (0, 1) for a in range(4) for b in range(4)])
ROUTE_CODES = {k: k for k in ROUTE_KEYS}      # routes_of's {key: route code}: each route is its own key


def expect(launches):
    want = dict(launches)
    want['all'] = sum(launches.values())
    return want


def record_hits(pred, dtype=0, adjoint=False):
    if pred[0] == 'tc':
        for stage, ((form, s), _) in enumerate(pred[1], 1):
            HIT.add(('tc', stage, form, s))
            if form == 'splitk':
                HIT.add(('reduce', s))
    else:
        HIT.add(('branch', dtype, bool(adjoint), bool(pred[1])))
        for a, b in R.cgemm_pairs(adjoint, pred[1]):
            HIT.add(('cgemm', dtype, a, b))


# ---- fixtures and inputs ------------------------------------------------------------------------------------------
@pytest.fixture(scope='module', autouse=True)
def precision_32(pb):
    pb.config.precision = 32
    yield
    _PUPIL.clear()
    path = os.environ.get('PB_MDFT_TEST_HITS')
    if CHILD and path:
        with open(path, 'w') as fh:
            json.dump(sorted(HIT, key=str), fh)


_PUPIL = {}


def pupil(rows, cols):
    """the BASELINE field at N = max(rows, cols), cropped to the centre (rows, cols), complex64"""
    N = max(rows, cols)
    if N not in _PUPIL:
        amp, opd, _ = O.synthetic_pupil(N)
        _PUPIL[N] = O.from_amp_and_phase(amp, opd.astype(np.float64), HeNe).astype(np.complex64)
    r0, c0 = (N - rows) // 2, (N - cols) // 2
    return np.ascontiguousarray(_PUPIL[N][r0:r0 + rows, c0:c0 + cols])


def coords(n, m, q):
    """n sample positions and m frequencies; q sets the sampling (phases up to about m q / 4 turns)"""
    x = (np.arange(n) - n // 2) * 0.1
    return x, (np.arange(m) - m // 2) * (q / (n * 0.1))


def geometry(shape):
    """(x, y, fx, fy) of an MDFT of shape (my, ny, mx, nx); different samplings along x and y, so that a swap shows"""
    my, ny, mx, nx = shape
    x, fx = coords(nx, mx, 0.37)
    y, fy = coords(ny, my, 0.53)
    return x, y, fx, fy


def gemm_ref(Ey, Ex, a, adjoint):
    """norm * Ey a Ex^T (adjoint: Ey^H g conj(Ex)) in complex128 from the device's complex64 bases"""
    Ey, Ex, a = Ey.astype(np.complex128), Ex.astype(np.complex128), a.astype(np.complex128)
    if adjoint:
        Ey, Ex = Ey.conj().T, Ex.conj().T
    return NORM * ((Ey @ a) @ Ex.T if Ey.shape[0] * a.shape[1] <= a.shape[0] * Ex.shape[0] else Ey @ (a @ Ex.T))


def impulse_points(rows, cols):
    return {'corner': (0, 0), 'centre': (rows // 2, cols // 2), 'last': (rows - 1, cols - 1)}


def impulse_ref(Ey, Ex, p, adjoint):
    """norm * outer(Ey[:, a], Ex[:, b]) (adjoint: outer(conj(Ey[a, :]), conj(Ex[b, :]))) for an impulse at p = (a, b)"""
    a, b = p
    if adjoint:
        return NORM * np.outer(Ey[a, :].conj(), Ex[b, :].conj())
    return NORM * np.outer(Ey[:, a], Ex[:, b])


def shape_id(s):
    return 'x'.join(map(str, s))


# ---- the executor: fttools.MDFT, tensor cores (and the CUDA-core adjoint of the narrow shapes) ----------------------
def stage_note(pred, shape, adjoint, sms):
    """what the restated stream-K partition says about an output tile (None when no stage is stream-K)"""
    if pred[0] != 'tc':
        return None
    my = shape[1] if adjoint else shape[0]
    (s1, (t1, k1)), (s2, (t2, k2)) = pred[1]
    G = min(sms, 160)
    parts = []
    if s1[0] == 'streamk':
        n = len(R.split_tiles(t1, k1 // CHUNK, G))
        parts.append(f'stage 1 stream-K: {n} of {t1} tiles of the intermediate cut across CTAs (spread over the output)')
    cut = R.split_tiles(t2, k2 // CHUNK, G) if s2[0] == 'streamk' else None
    if not parts and cut is None:
        return None

    def note(i, j):
        out = list(parts)
        if cut is not None:
            ntn = 2 * my // TILE        # stage 2: output rows 64 tn .. 64 tn + 63, columns 128 tm .. of tile tm * ntn + tn
            tiles = [j * ntn + tn for tn in (2 * i, 2 * i + 1) if tn < ntn]
            out.append(f'stage-2 stream-K tiles {tiles} behind it, cut across CTAs: {sorted(set(tiles) & cut) or "none"}')
        return '; '.join(out)
    return note


@pytest.mark.parametrize('direction', ('forward', 'adjoint'))
@pytest.mark.parametrize('sign', (-1, 1))
@pytest.mark.parametrize('shape', R.TC_SHAPES, ids=shape_id)
def test_executor_vs_fp64(pb, shape, sign, direction):
    F = pb.fttools
    adjoint = direction == 'adjoint'
    sms = sm_count()
    if CHILD and R.summary(shape, sms, STREAMK, CHUNK) == R.summary(shape, sms, 1, CHUNK):
        pytest.skip(f'PB_MDFT_STREAMK={CHILD} launches the same kernels as the default for this shape')
    x, y, fx, fy = geometry(shape)
    ex = F.MDFT(x, y, fx, fy, sign, NORM)
    pred = R.mdft_routes(*shape, sms, adjoint, STREAMK, CHUNK)
    assert ((ex._tc_adj if adjoint else ex._tc) is not None) == (pred[0] == 'tc')
    ref_ex = O.MDFT(x, y, fx, fy, sign, NORM)
    Ey, Ex = host(ex.Ey), host(ex.Ex)
    my, ny, mx, nx = shape
    rows, cols = (my, mx) if adjoint else (ny, nx)
    streamk = pred[0] == 'tc' and any(f == 'streamk' for (f, _), _ in pred[1])
    note = stage_note(pred, shape, adjoint, sms)
    fn_of = (lambda a: (lambda: ex.adjoint(a))) if adjoint else (lambda a: (lambda: ex(a)))
    base = f'mdft/{shape_id(shape)}/{direction}'

    def run(inp, what):
        a = torch.from_numpy(inp).cuda()
        got, used = routes_of(fn_of(a), ROUTE_CODES)
        LEDGER.route(used == expect(pred[2]), f'{base}/{what}: launches per route {used}, predicted {expect(pred[2])}')
        g = host(got)
        if streamk:
            LEDGER.route(np.array_equal(host(fn_of(a)()), g), f'{base}/{what}: stream-K result differs between two applies')
        return g

    inputs = {'gauss': crand((rows, cols), sum(shape) + 17 * (sign + 1), np.complex64),
              'ones': np.ones((rows, cols), np.complex64)}
    if max(rows, cols) <= 4096:
        inputs['pupil'] = pupil(rows, cols)
    for name, inp in inputs.items():
        g = run(inp, f'{name}, sign {sign:+d}')
        a128 = inp.astype(np.complex128)
        add(f'{base}/{name}/gemm', g, gemm_ref(Ey, Ex, inp, adjoint), note, f'{name}, sign {sign:+d}')
        add(f'{base}/{name}/e2e', g, (ref_ex.adjoint if adjoint else ref_ex)(a128), note, f'{name}, sign {sign:+d}')
    for pname, p in impulse_points(rows, cols).items():
        inp = np.zeros((rows, cols), np.complex64)
        inp[p] = 1.0
        g = run(inp, f'impulse {pname}, sign {sign:+d}')
        add(f'{base}/impulse/gemm', g, impulse_ref(Ey, Ex, p, adjoint), note, f'impulse {pname}, sign {sign:+d}')
        add(f'{base}/impulse/e2e', g, impulse_ref(ref_ex.Ey, ref_ex.Ex, p, adjoint), note,
            f'impulse {pname}, sign {sign:+d}')
    LEDGER.done()
    record_hits(pred, 0, adjoint)


@pytest.mark.parametrize('streamk', ('0', '2'))
def test_switch_settings_in_child(pb, streamk, tmp_path):
    """the executor cases again in a child process under PB_MDFT_STREAMK = 0 (split-K everywhere) and = 2 (stream-K
    wherever it is legal); the child's figures are recorded here and its hits count for the coverage test"""
    if CHILD:
        pytest.skip('a child run starts no children')
    mfile, hfile = tmp_path / 'measured.json', tmp_path / 'hits.json'
    env = dict(os.environ, PB_MDFT_STREAMK=streamk, PB_MDFT_TEST_CHILD=streamk, PB_TEST_MEASUREMENTS=str(mfile),
               PB_MDFT_TEST_HITS=str(hfile))
    cmd = [sys.executable] + (['-s'] if sys.flags.no_user_site else []) + [
        '-m', 'pytest', '-q', '-x', '-p', 'no:cacheprovider', '-m', 'gpu', f'{os.path.abspath(__file__)}::test_executor_vs_fp64']
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=CHILD_TIMEOUT)
    assert r.returncode == 0, f'child run under PB_MDFT_STREAMK={streamk} failed:\n{r.stdout[-6000:]}\n{r.stderr[-3000:]}'
    figures = json.loads(mfile.read_text())
    assert figures, 'the child run recorded no figures'
    for name, d in sorted(figures.items()):
        LEDGER.record(name, d['measured'])
    LEDGER.done()
    HIT.update(tuple(h) for h in json.loads(hfile.read_text()))


# ---- edges of the executor ----------------------------------------------------------------------------------------
def test_out_into_plane_of_a_stack(pb):
    """forward and adjoint written into plane 2 of a NaN-filled (4, My, Mx) / (4, Ny, Nx) stack, as the polarization
    path does; the other planes stay untouched"""
    shape = (256, 1024, 640, 1024)
    my, ny, mx, nx = shape
    x, y, fx, fy = geometry(shape)
    ex = pb.fttools.MDFT(x, y, fx, fy, -1, NORM)
    ref = O.MDFT(x, y, fx, fy, -1, NORM)
    for adjoint, (rows, cols), (orows, ocols) in ((False, (ny, nx), (my, mx)), (True, (my, mx), (ny, nx))):
        inp = crand((rows, cols), 5 + adjoint, np.complex64)
        stack = torch.full((4, orows, ocols), float('nan'), dtype=torch.complex64, device='cuda')
        a = torch.from_numpy(inp).cuda()
        (ex._adjoint if adjoint else ex._forward)(a, out=stack[2])
        s = host(stack)
        assert np.isnan(np.delete(s, 2, axis=0)).all(), 'a plane other than the output plane was written'
        d = 'adjoint' if adjoint else 'forward'
        add(f'mdft/{shape_id(shape)}/{d}/out_plane2/e2e', s[2], (ref.adjoint if adjoint else ref)(inp.astype(np.complex128)))
    LEDGER.done()


def test_misaligned_input(pb, monkeypatch):
    """a complex64 input at an address that is 8 bytes off a 16-byte boundary (flat[1:].view(N, N)) is copied to an
    aligned buffer for the TMA loads and gives the right answer; an aligned input is not copied"""
    from prysm_b200 import _ops
    shape = (512, 1024, 512, 1024)
    my, ny, mx, nx = shape
    x, y, fx, fy = geometry(shape)
    ex = pb.fttools.MDFT(x, y, fx, fy, 1, NORM)
    ref = O.MDFT(x, y, fx, fy, 1, NORM)
    seen = []
    real = _ops._tc_aligned

    def spy(a):
        out = real(a)
        seen.append((a.data_ptr(), out.data_ptr()))
        return out
    monkeypatch.setattr(_ops, '_tc_aligned', spy)
    inp = crand((ny, nx), 3, np.complex64)
    flat = torch.empty(ny * nx + 1, dtype=torch.complex64, device='cuda')
    odd = flat[1:].view(ny, nx)
    odd.copy_(torch.from_numpy(inp))
    assert odd.data_ptr() % 16 == 8 and odd.is_contiguous()
    add(f'mdft/{shape_id(shape)}/forward/misaligned/e2e', host(ex(odd)), ref(inp.astype(np.complex128)))
    (src, used), = seen
    assert src == odd.data_ptr() and used != src and used % 16 == 0, 'the misaligned input was not copied'
    aligned = torch.from_numpy(inp).cuda()
    same = host(ex(aligned))
    assert seen[1] == (aligned.data_ptr(), aligned.data_ptr()), 'an aligned input was copied'
    assert np.array_equal(same, host(ex(odd)))
    LEDGER.done()


# ---- the CUDA-core GEMM ---------------------------------------------------------------------------------------------
DT = {0: ('c64', np.complex64, torch.complex64), 1: ('c128', np.complex128, torch.complex128)}
MN = [(1, 65), (63, 64), (64, 1), (65, 63)]       # tile edges of the 64 x 64 output tile
KS = [1, 16, 48, 64, 80, 4096 + 16]                # around the fold of 64-term partial sums and its unfolded remainder
ALPHA = 0.3


def op_host(X, op):
    """op(X) for a stored operand: 0 as is, 1 transpose, 2 conjugate transpose, 3 conjugate"""
    return {0: X, 1: X.T, 2: X.conj().T, 3: X.conj()}[op]


def stored_shape(rows, cols, op):
    """the stored shape of an operand that is (rows, cols) after op"""
    return (rows, cols) if op in (R.OP_N, R.OP_C) else (cols, rows)


def pb_cgemm(dtype, opA, opB, M, N, K, A, lda, B, ldb, Cm, ldc):
    from prysm_b200 import _capi
    h = _capi.handle_for(torch.cuda.current_device(), torch.cuda.current_stream().cuda_stream)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    h.check(_capi.lib.pb_cgemm(h.ptr, dtype, opA, opB, M, N, K, float(ALPHA), C.c_void_p(A.data_ptr()), lda,
                               C.c_void_p(B.data_ptr()), ldb, C.c_void_p(Cm.data_ptr()), ldc, st))


@pytest.mark.parametrize('opB', range(4))
@pytest.mark.parametrize('opA', range(4))
@pytest.mark.parametrize('dtype', (0, 1), ids=('c64', 'c128'))
def test_cgemm_op_pairs(pb, dtype, opA, opB):
    """pb_cgemm with padded lda / ldb / ldc (C's padding must stay untouched) at M, N across the tile edges and K across
    the fold; _ops.cgemm on contiguous operands"""
    from prysm_b200 import _ops
    name, npdt, tdt = DT[dtype]
    case = f'cgemm/{name}/{opA}{opB}'
    want = expect({R.cgemm_code(dtype, opA, opB): 1})
    for M, N in MN:
        for K in KS:
            sa, sb = stored_shape(M, K, opA), stored_shape(K, N, opB)
            lda, ldb, ldc = sa[1] + 3, sb[1] + 5, N + 2
            Ah = crand((sa[0], lda), M * 7 + K, npdt)
            Bh = crand((sb[0], ldb), N * 11 + K, npdt)
            A, B = torch.from_numpy(Ah).cuda(), torch.from_numpy(Bh).cuda()
            Cm = torch.full((M, ldc), float('nan'), dtype=tdt, device='cuda')
            _, used = routes_of(lambda: pb_cgemm(dtype, opA, opB, M, N, K, A, lda, B, ldb, Cm, ldc), ROUTE_CODES)
            LEDGER.route(used == want, f'{case} M={M} N={N} K={K}: launches {used}, want {want}')
            got = host(Cm)
            assert np.isnan(got[:, N:]).all(), f'{case} M={M} N={N} K={K}: the padding of C was written'
            a, b = op_host(Ah[:, :sa[1]].astype(np.complex128), opA), op_host(Bh[:, :sb[1]].astype(np.complex128), opB)
            alpha = float(np.float32(ALPHA)) if dtype == 0 else ALPHA
            add(case, got[:, :N], alpha * (a @ b), what=f'M={M} N={N} K={K}')
    # the tensor-level wrapper: contiguous operands, alpha = 1
    Ah = crand(stored_shape(65, 80, opA), 1, npdt)
    Bh = crand(stored_shape(80, 63, opB), 2, npdt)
    got, used = routes_of(lambda: _ops.cgemm(torch.from_numpy(Ah).cuda(), torch.from_numpy(Bh).cuda(), opA, opB),
                          ROUTE_CODES)
    LEDGER.route(used == want, f'{case} _ops.cgemm: launches {used}, want {want}')
    add(case, host(got), op_host(Ah.astype(np.complex128), opA) @ op_host(Bh.astype(np.complex128), opB),
        what='_ops.cgemm 65 x 63 x 80')
    LEDGER.done()
    HIT.add(('cgemm', dtype, opA, opB))


def test_cgemm_c128_against_longdouble(pb):
    """a complex128 figure against a complex128 reference is mostly the reference's own rounding: on one case, both
    against an extended-precision (x87 long double) reference"""
    M, N, K = 63, 65, 4096 + 16
    Ah, Bh = crand((M, K), 41, np.complex128), crand((K, N), 42, np.complex128)
    Cm = torch.empty((M, N), dtype=torch.complex128, device='cuda')
    pb_cgemm(1, 0, 0, M, N, K, torch.from_numpy(Ah).cuda(), K, torch.from_numpy(Bh).cuda(), N, Cm, N)
    got = host(Cm)
    ld = np.longdouble
    ar, ai, br, bi = (v.astype(ld) for v in (Ah.real, Ah.imag, Bh.real, Bh.imag))
    rr = (ar @ br - ai @ bi) * ld(ALPHA)
    ri = (ar @ bi + ai @ br) * ld(ALPHA)
    den = np.sqrt(rr * rr + ri * ri).max()

    def err(c):
        return float((np.sqrt((c.real.astype(ld) - rr) ** 2 + (c.imag.astype(ld) - ri) ** 2)).max() / den)
    d, r = err(got), err(ALPHA * (Ah @ Bh))
    LEDGER.check('cgemm/c128/longdouble/device/linf', d)
    within('cgemm/c128/longdouble/numpy/linf', r, 1e-15)


@pytest.mark.parametrize('left_first', (False, True))
@pytest.mark.parametrize('adjoint', (False, True))
@pytest.mark.parametrize('dtype', (0, 1), ids=('c64', 'c128'))
def test_mdft_apply_branches(pb, dtype, adjoint, left_first):
    """_ops.mdft_apply called directly on each of its four branches, on a rectangular shape"""
    from prysm_b200 import _ops
    name, npdt, tdt = DT[dtype]
    shape = (130, 300, 70, 200)
    my, ny, mx, nx = shape
    x, y, fx, fy = geometry(shape)
    Ey = _ops.mdft_basis(fy, y, -1, tdt, torch.device('cuda'))
    Ex = _ops.mdft_basis(fx, x, -1, tdt, torch.device('cuda'))
    inp = crand((my, mx) if adjoint else (ny, nx), 9 + adjoint, npdt)
    got, used = routes_of(lambda: _ops.mdft_apply(Ey, Ex, torch.from_numpy(inp).cuda(), NORM, adjoint, left_first),
                          ROUTE_CODES)
    want = {}
    for a, b in R.cgemm_pairs(adjoint, left_first):
        want[R.cgemm_code(dtype, a, b)] = want.get(R.cgemm_code(dtype, a, b), 0) + 1
    LEDGER.route(used == expect(want), f'launches {used}, want {expect(want)}')
    case = f'mdft_apply/{name}/{"adjoint" if adjoint else "forward"}/{"left" if left_first else "right"}'
    g = host(got)
    ref = O.MDFT(x, y, fx, fy, -1, NORM)
    add(f'{case}/gemm', g, gemm_ref(host(Ey), host(Ex), inp, adjoint))
    add(f'{case}/e2e', g, (ref.adjoint if adjoint else ref)(inp.astype(np.complex128)))
    LEDGER.done()
    HIT.add(('branch', dtype, adjoint, left_first))
    HIT.update(('cgemm', dtype, a, b) for a, b in R.cgemm_pairs(adjoint, left_first))


@pytest.mark.parametrize('direction', ('forward', 'adjoint'))
def test_ragged_complex64_executor(pb, direction):
    """4000^2 -> 500^2 in complex64: no multiple of 128, so the CUDA-core GEMM"""
    adjoint = direction == 'adjoint'
    shape = (500, 4000, 500, 4000)
    my, ny, mx, nx = shape
    x, y, fx, fy = geometry(shape)
    ex = pb.fttools.MDFT(x, y, fx, fy, -1, NORM)
    pred = R.mdft_routes(*shape, sm_count(), adjoint)
    assert pred[0] == 'cgemm' and ex._tc is None and ex._tc_adj is None
    ref = O.MDFT(x, y, fx, fy, -1, NORM)
    Ey, Ex = host(ex.Ey), host(ex.Ex)
    rows, cols = (my, mx) if adjoint else (ny, nx)
    for name, inp in (('gauss', crand((rows, cols), 23, np.complex64)), ('ones', np.ones((rows, cols), np.complex64))):
        a = torch.from_numpy(inp).cuda()
        got, used = routes_of(lambda: ex.adjoint(a) if adjoint else ex(a), ROUTE_CODES)
        LEDGER.route(used == expect(pred[2]), f'{name}: launches {used}, predicted {expect(pred[2])}')
        g = host(got)
        case = f'mdft/{shape_id(shape)}/{direction}/{name}'
        add(f'{case}/gemm', g, gemm_ref(Ey, Ex, inp, adjoint), what=name)
        add(f'{case}/e2e', g, (ref.adjoint if adjoint else ref)(inp.astype(np.complex128)), what=name)
    LEDGER.done()
    record_hits(pred, 0, adjoint)


# ---- the basis ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('sign', (-1, 1))
@pytest.mark.parametrize('dtype', (0, 1), ids=('c64', 'c128'))
def test_basis_at_large_phases(pb, dtype, sign):
    """pb_mdft_basis at phases up to ~1e5 turns against exp(2 pi i (t - rint(t))) of the same fp64 product t = sign f x,
    evaluated in long double; the error is absolute, at most 4 units in the last place of 1"""
    from prysm_b200 import _ops
    name, npdt, tdt = DT[dtype]
    f = np.linspace(-97.3, 101.7, 257)
    x = np.linspace(-1013.1, 987.9, 311)
    E = host(_ops.mdft_basis(f, x, sign, tdt, torch.device('cuda')))
    t = (sign * f)[:, None] * x[None, :]
    assert np.abs(t).max() > 9e4
    ld = np.longdouble
    ang = 2 * np.arccos(ld(-1)) * (t - np.rint(t)).astype(ld)
    err = float(np.sqrt((E.real.astype(ld) - np.cos(ang)) ** 2 + (E.imag.astype(ld) - np.sin(ang)) ** 2).max())
    ulp1 = float(np.finfo(np.float32 if dtype == 0 else np.float64).eps)
    within(f'basis/{name}/{sign:+d}/abs', err, 4 * ulp1)


# ---- coverage -------------------------------------------------------------------------------------------------------
def test_every_route_was_checked(pb):
    """every tensor-core (stage, form, pieces), the reduce kernel, all 32 cgemm_kernel instantiations and the four
    pb_mdft_apply branches in both dtypes were run by a case above (here or in a child run) and held to fp64"""
    if CHILD:
        pytest.skip('the coverage of a child run counts in its parent')
    need = {('tc', 1, 'plain', 1), ('tc', 1, 'streamk', 1), ('tc', 2, 'streamk', 1)}
    need |= {('tc', 2, 'splitk', s) for s in (2, 4, 8)} | {('reduce', s) for s in (2, 4, 8)}
    need |= {('cgemm', d, a, b) for d in (0, 1) for a in range(4) for b in range(4)}
    need |= {('branch', d, adj, lf) for d in (0, 1) for adj in (False, True) for lf in (False, True)}
    missing = sorted(need - HIT, key=str)
    assert not missing, f'not run by an fp64-checked case: {missing}'


def test_zz_every_figure_has_a_measurement():
    """a figure this session reached that has no MEASURED entry is held to the bare ceiling, a bound nobody measured"""
    if os.environ.get('PB_TEST_MEASUREMENTS'):
        pytest.skip('recording figures')
    assert not LEDGER.missing(), f'no MEASURED entry (record them with PB_TEST_MEASUREMENTS): {LEDGER.missing()}'
