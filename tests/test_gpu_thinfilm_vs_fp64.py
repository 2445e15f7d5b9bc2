"""GPU: the thin-film and coating-design kernels of csrc/thinfilm.cu held to the long-double references of
tests/thinfilm_reference.py, each kernel alone through the `_ops` level and end to end through `prysm_b200.coatings`.

- pb_stack_eval: r, t, the boundary fields, R, T, A, eta0 and eta_sub of every stack class (no layers, one layer, a
  quarter-wave pair, the 40-layer HL stack, an absorbing layer, silver at 50 nm and 2 um, the TIR gap, a zero-thickness
  layer, 200 high-contrast layers, a complex ambient index, a 0.2 mm layer) at 0 to 89.9 degrees, in both assembly
  modes, the angle in degrees through theta_scale, both sides of a critical angle and at an exact one.
- pb_stack_grad: thickness, index and both, under each of dR, dT, dA and dEsq alone and all four together; counts
  1, 31, 32, 33 and one grid sweep - 1, exactly, + 1 and two sweeps + 33 of this device's sm_count.
- pb_coating_merit: the six quantities under s, p and avg; value, residuals and both gradients; the peak's exact tie;
  the sweep counts of the 256- and the 128-thread instances; stride-0 and per-sample target and weight.
- pb_needle: R and T terms, a per-wavelength needle index, the sweep counts of both instances.
- pb_field_at_depth: every boundary and one ulp either side of it, depths outside the stack, nz past one sweep; from
  the device's own boundary fields and end to end.
- Layouts: a (wvl, 1) x (1, theta) grid, per-pixel index and thickness maps with a non-unit layer stride, a 4-D
  collapsed shape.

fp64 figures: per-sample relative error of r, t, R, T, eta0, eta_sub; the fields over each sample's largest boundary
magnitude; A over its flux majorant; gradients, merit values and P(z) over the sum of the absolute per-sample
contributions (their majorant).  The 0.2 mm layer's phase is known only to |beta| 2^-53 from its inputs, so its figures
are in units of sum |Re beta_k| 2^-53.  float32 figures (`*_ulps`): the error in ulps of the float32-rounded
reference, never below the fp64 majorant x 2^-52 where a sum cancels.

Bounds are 1.5x the figures measured on an H100 (`MEASURED`, recorded with PB_TEST_MEASUREMENTS) and never above the
ceilings tests/test_host_thinfilm_reference.py shows every modelled defect exceeds by 10x or more.
"""
import os

import numpy as np
import pytest
import torch

import thinfilm_reference as T
from accuracy import Ledger, sweep
from gpu_fixtures import pb, host, sm_count  # noqa: F401

pytestmark = pytest.mark.gpu

PRECS = (64, 32)
RT = {32: torch.float32, 64: torch.float64}

# ceilings, shown by the host test to sit 10x or more below every modelled defect; float32 figures are in ulps
CEIL = {'rt': 1e-12, 'field': 1e-12, 'flux': 1e-12, 'grad': 1e-12, 'merit': 1e-12, 'needle': 1e-12, 'fad': 1e-12,
        'beta_units': 64.0, 'critical': 1e-6, 'ulps': 2.0, 'ulps_acc': 3.0}

# ---- measured figures (H100 80GB HBM3, 700 W power limit, 1980 MHz SM clock); bounds are 1.5x these, capped at the
# ceiling ------------------------------------------------------------------------------------------------------------
MEASURED = {
    '32/absorb/A/merit_grad_ulps': 0.471,
    '32/absorb/A/merit_resid_ulps': 0.49,
    '32/absorb/Esq/merit_grad_ulps': 0.493,
    '32/absorb/Esq/merit_resid_ulps': 0.498,
    '32/absorb/R/merit_grad_ulps': 0.47,
    '32/absorb/R/merit_resid_ulps': 0.494,
    '32/absorb/T/merit_grad_ulps': 0.409,
    '32/absorb/T/merit_resid_ulps': 0.497,
    '32/absorb/fad_e2e_ulps': 0.706,
    '32/absorb/fad_ulps': 0.706,
    '32/absorb/field_E_ulps': 0.517,
    '32/absorb/field_Esq_ulps': 0.491,
    '32/absorb/field_H_ulps': 0.532,
    '32/absorb/flux_A_ulps': 0.762,
    '32/absorb/grad_ulps': 0.498,
    '32/absorb/layer/merit_grad_ulps': 0.498,
    '32/absorb/layer/merit_resid_ulps': 0.494,
    '32/absorb/needle_ulps': 0.499,
    '32/absorb/peak/merit_grad_ulps': 0.469,
    '32/absorb/peak/merit_resid_ulps': 0.495,
    '32/absorb/rt_R_ulps': 0.489,
    '32/absorb/rt_T_ulps': 0.497,
    '32/absorb/rt_eta0_ulps': 0.495,
    '32/absorb/rt_eta_sub_ulps': 0.454,
    '32/absorb/rt_ml_r_ulps': 0.601,
    '32/absorb/rt_ml_t_ulps': 0.529,
    '32/absorb/rt_r_ulps': 0.601,
    '32/absorb/rt_t_ulps': 0.498,
    '32/absorb/tie/merit_grad_ulps': 0.493,
    '32/absorb/tie/merit_resid_ulps': 0.498,
    '32/ag2um/field_E_ulps': 0.541,
    '32/ag2um/field_Esq_ulps': 0.494,
    '32/ag2um/field_H_ulps': 0.501,
    '32/ag2um/flux_A_ulps': 0.494,
    '32/ag2um/grad_ulps': 0.444,
    '32/ag2um/rt_R_ulps': 0.497,
    '32/ag2um/rt_T_ulps': 2.99e-12,
    '32/ag2um/rt_eta0_ulps': 0.495,
    '32/ag2um/rt_eta_sub_ulps': 0.454,
    '32/ag2um/rt_ml_r_ulps': 0.559,
    '32/ag2um/rt_ml_t_ulps': 0.621,
    '32/ag2um/rt_r_ulps': 0.559,
    '32/ag2um/rt_t_ulps': 0.621,
    '32/ag50/A/merit_grad_ulps': 0.481,
    '32/ag50/A/merit_resid_ulps': 0.489,
    '32/ag50/Esq/merit_grad_ulps': 0.482,
    '32/ag50/Esq/merit_resid_ulps': 0.451,
    '32/ag50/R/merit_grad_ulps': 0.475,
    '32/ag50/R/merit_resid_ulps': 0.479,
    '32/ag50/T/merit_grad_ulps': 0.499,
    '32/ag50/T/merit_resid_ulps': 0.495,
    '32/ag50/field_E_ulps': 0.665,
    '32/ag50/field_Esq_ulps': 0.5,
    '32/ag50/field_H_ulps': 0.534,
    '32/ag50/flux_A_ulps': 0.487,
    '32/ag50/grad_ulps': 0.489,
    '32/ag50/layer/merit_grad_ulps': 0.498,
    '32/ag50/layer/merit_resid_ulps': 0.492,
    '32/ag50/needle_ulps': 0.483,
    '32/ag50/peak/merit_grad_ulps': 0.497,
    '32/ag50/peak/merit_resid_ulps': 0.493,
    '32/ag50/rt_R_ulps': 0.491,
    '32/ag50/rt_T_ulps': 0.496,
    '32/ag50/rt_eta0_ulps': 0.495,
    '32/ag50/rt_eta_sub_ulps': 0.454,
    '32/ag50/rt_ml_r_ulps': 0.592,
    '32/ag50/rt_ml_t_ulps': 0.509,
    '32/ag50/rt_r_ulps': 0.592,
    '32/ag50/rt_t_ulps': 0.665,
    '32/ag50/tie/merit_grad_ulps': 0.482,
    '32/ag50/tie/merit_resid_ulps': 0.451,
    '32/ambc/field_E_ulps': 0.671,
    '32/ambc/field_Esq_ulps': 0.499,
    '32/ambc/field_H_ulps': 0.594,
    '32/ambc/flux_A_ulps': 0.655,
    '32/ambc/grad_ulps': 0.466,
    '32/ambc/rt_R_ulps': 0.491,
    '32/ambc/rt_T_ulps': 0.475,
    '32/ambc/rt_eta0_ulps': 0.446,
    '32/ambc/rt_eta_sub_ulps': 0.371,
    '32/ambc/rt_ml_r_ulps': 0.549,
    '32/ambc/rt_ml_t_ulps': 0.552,
    '32/ambc/rt_r_ulps': 0.549,
    '32/ambc/rt_t_ulps': 0.646,
    '32/dims4/field_H_ulps': 0.67,
    '32/dims4/grad_ulps': 0.421,
    '32/dims4/rt_r_ulps': 0.544,
    '32/dims4/rt_t_ulps': 0.67,
    '32/e2e/grad_ulps': 0.315,
    '32/e2e/merit_grad_acc_ulps': 0.825,
    '32/e2e/needle_ulps': 0.493,
    '32/gap/A/merit_grad_ulps': 0.0784,
    '32/gap/A/merit_resid_ulps': 0.477,
    '32/gap/Esq/merit_grad_ulps': 0.457,
    '32/gap/Esq/merit_resid_ulps': 0.489,
    '32/gap/R/merit_grad_ulps': 0.474,
    '32/gap/R/merit_resid_ulps': 0.498,
    '32/gap/T/merit_grad_ulps': 0.457,
    '32/gap/T/merit_resid_ulps': 0.497,
    '32/gap/fad_e2e_ulps': 0.705,
    '32/gap/fad_ulps': 0.705,
    '32/gap/field_E_ulps': 0.646,
    '32/gap/field_Esq_ulps': 0.493,
    '32/gap/field_H_ulps': 0.607,
    '32/gap/flux_A_ulps': 1.11,
    '32/gap/grad_ulps': 0.492,
    '32/gap/layer/merit_grad_ulps': 0.443,
    '32/gap/layer/merit_resid_ulps': 0.498,
    '32/gap/needle_ulps': 0.461,
    '32/gap/peak/merit_grad_ulps': 0.45,
    '32/gap/peak/merit_resid_ulps': 0.482,
    '32/gap/rt_R_ulps': 0.49,
    '32/gap/rt_T_ulps': 0.415,
    '32/gap/rt_eta0_ulps': 0.4,
    '32/gap/rt_eta_sub_ulps': 0.4,
    '32/gap/rt_ml_r_ulps': 0.451,
    '32/gap/rt_ml_t_ulps': 0.646,
    '32/gap/rt_r_ulps': 0.451,
    '32/gap/rt_t_ulps': 0.646,
    '32/gap/tie/merit_grad_ulps': 0.457,
    '32/gap/tie/merit_resid_ulps': 0.489,
    '32/hc200/field_E_ulps': 0.606,
    '32/hc200/field_Esq_ulps': 0.5,
    '32/hc200/field_H_ulps': 0.646,
    '32/hc200/flux_A_ulps': 0.983,
    '32/hc200/grad_ulps': 0.512,
    '32/hc200/rt_R_ulps': 0.412,
    '32/hc200/rt_T_ulps': 0.437,
    '32/hc200/rt_eta0_ulps': 0.495,
    '32/hc200/rt_eta_sub_ulps': 0.454,
    '32/hc200/rt_ml_r_ulps': 0.418,
    '32/hc200/rt_ml_t_ulps': 0.668,
    '32/hc200/rt_r_ulps': 0.418,
    '32/hc200/rt_t_ulps': 0.668,
    '32/hl40/field_E_ulps': 0.673,
    '32/hl40/field_Esq_ulps': 0.5,
    '32/hl40/field_H_ulps': 0.663,
    '32/hl40/flux_A_ulps': 0.987,
    '32/hl40/grad_ulps': 0.499,
    '32/hl40/rt_R_ulps': 0.467,
    '32/hl40/rt_T_ulps': 0.493,
    '32/hl40/rt_eta0_ulps': 0.495,
    '32/hl40/rt_eta_sub_ulps': 0.454,
    '32/hl40/rt_ml_r_ulps': 0.527,
    '32/hl40/rt_ml_t_ulps': 0.583,
    '32/hl40/rt_r_ulps': 0.527,
    '32/hl40/rt_t_ulps': 0.507,
    '32/layout/merit_grad_ulps': 0.49,
    '32/layout/merit_resid_ulps': 0.495,
    '32/none/field_E_ulps': 0.243,
    '32/none/field_Esq_ulps': 0.389,
    '32/none/field_H_ulps': 0.435,
    '32/none/rt_R_ulps': 0.364,
    '32/none/rt_T_ulps': 0.486,
    '32/none/rt_eta0_ulps': 0.495,
    '32/none/rt_eta_sub_ulps': 0.454,
    '32/none/rt_r_ulps': 0.457,
    '32/none/rt_t_ulps': 0.243,
    '32/one/field_E_ulps': 0.577,
    '32/one/field_Esq_ulps': 0.499,
    '32/one/field_H_ulps': 0.523,
    '32/one/flux_A_ulps': 0.621,
    '32/one/grad_ulps': 0.438,
    '32/one/rt_R_ulps': 0.461,
    '32/one/rt_T_ulps': 0.493,
    '32/one/rt_eta0_ulps': 0.495,
    '32/one/rt_eta_sub_ulps': 0.454,
    '32/one/rt_ml_r_ulps': 0.494,
    '32/one/rt_ml_t_ulps': 0.577,
    '32/one/rt_r_ulps': 0.494,
    '32/one/rt_t_ulps': 0.577,
    '32/pixel/field_E_ulps': 0.6,
    '32/pixel/flux_A_ulps': 0.958,
    '32/pixel/grad_ulps': 0.436,
    '32/pixel/rt_r_ulps': 0.646,
    '32/qw/A/merit_grad_ulps': 0.056,
    '32/qw/A/merit_resid_ulps': 0.477,
    '32/qw/Esq/merit_grad_ulps': 0.472,
    '32/qw/Esq/merit_resid_ulps': 0.485,
    '32/qw/R/merit_grad_ulps': 0.497,
    '32/qw/R/merit_resid_ulps': 0.493,
    '32/qw/T/merit_grad_ulps': 0.459,
    '32/qw/T/merit_resid_ulps': 0.497,
    '32/qw/fad_e2e_ulps': 0.706,
    '32/qw/fad_ulps': 0.706,
    '32/qw/field_E_ulps': 0.516,
    '32/qw/field_Esq_ulps': 0.486,
    '32/qw/field_H_ulps': 0.507,
    '32/qw/flux_A_ulps': 0.663,
    '32/qw/grad_ulps': 0.496,
    '32/qw/layer/merit_grad_ulps': 0.498,
    '32/qw/layer/merit_resid_ulps': 0.498,
    '32/qw/needle_ulps': 0.497,
    '32/qw/peak/merit_grad_ulps': 0.472,
    '32/qw/peak/merit_resid_ulps': 0.485,
    '32/qw/rt_R_ulps': 0.481,
    '32/qw/rt_T_ulps': 0.48,
    '32/qw/rt_eta0_ulps': 0.495,
    '32/qw/rt_eta_sub_ulps': 0.454,
    '32/qw/rt_ml_r_ulps': 0.499,
    '32/qw/rt_ml_t_ulps': 0.516,
    '32/qw/rt_r_ulps': 0.499,
    '32/qw/rt_t_ulps': 0.516,
    '32/qw/tie/merit_grad_ulps': 0.472,
    '32/qw/tie/merit_resid_ulps': 0.485,
    '32/sweep/grad_ulps': 0.462,
    '32/sweep_avg/merit_grad_ulps': 0.488,
    '32/sweep_avg/merit_resid_ulps': 0.5,
    '32/sweep_avg/needle_ulps': 0.494,
    '32/sweep_s/merit_grad_ulps': 0.499,
    '32/sweep_s/merit_resid_ulps': 0.5,
    '32/sweep_s/needle_ulps': 0.474,
    '32/thick/field_E_ulps': 0.664,
    '32/thick/field_Esq_ulps': 0.488,
    '32/thick/field_H_ulps': 0.639,
    '32/thick/flux_A_ulps': 0.437,
    '32/thick/grad_beta_ulps': 0.466,
    '32/thick/rt_R_ulps': 0.442,
    '32/thick/rt_T_ulps': 0.496,
    '32/thick/rt_eta0_ulps': 0.495,
    '32/thick/rt_eta_sub_ulps': 0.454,
    '32/thick/rt_ml_r_ulps': 0.489,
    '32/thick/rt_ml_t_ulps': 0.664,
    '32/thick/rt_r_ulps': 0.489,
    '32/thick/rt_t_ulps': 0.664,
    '32/zero/A/merit_grad_ulps': 0.0199,
    '32/zero/A/merit_resid_ulps': 0.477,
    '32/zero/Esq/merit_grad_ulps': 0.486,
    '32/zero/Esq/merit_resid_ulps': 0.491,
    '32/zero/R/merit_grad_ulps': 0.49,
    '32/zero/R/merit_resid_ulps': 0.484,
    '32/zero/T/merit_grad_ulps': 0.469,
    '32/zero/T/merit_resid_ulps': 0.494,
    '32/zero/field_E_ulps': 0.644,
    '32/zero/field_Esq_ulps': 0.497,
    '32/zero/field_H_ulps': 0.511,
    '32/zero/flux_A_ulps': 0.743,
    '32/zero/grad_ulps': 0.477,
    '32/zero/layer/merit_grad_ulps': 0.497,
    '32/zero/layer/merit_resid_ulps': 0.498,
    '32/zero/peak/merit_grad_ulps': 0.485,
    '32/zero/peak/merit_resid_ulps': 0.484,
    '32/zero/rt_R_ulps': 0.5,
    '32/zero/rt_T_ulps': 0.488,
    '32/zero/rt_eta0_ulps': 0.495,
    '32/zero/rt_eta_sub_ulps': 0.454,
    '32/zero/rt_ml_r_ulps': 0.488,
    '32/zero/rt_ml_t_ulps': 0.522,
    '32/zero/rt_r_ulps': 0.488,
    '32/zero/rt_t_ulps': 0.55,
    '32/zero/tie/merit_grad_ulps': 0.486,
    '32/zero/tie/merit_resid_ulps': 0.491,
    '64/absorb/A/merit_grad': 3.12e-17,
    '64/absorb/A/merit_resid': 9.37e-16,
    '64/absorb/A/merit_value': 1.18e-16,
    '64/absorb/Esq/merit_grad': 1.85e-16,
    '64/absorb/Esq/merit_resid': 7.01e-16,
    '64/absorb/Esq/merit_value': 4.05e-16,
    '64/absorb/R/merit_grad': 2.65e-17,
    '64/absorb/R/merit_resid': 5.64e-16,
    '64/absorb/R/merit_value': 1.29e-16,
    '64/absorb/T/merit_grad': 7.87e-17,
    '64/absorb/T/merit_resid': 6.76e-16,
    '64/absorb/T/merit_value': 4.19e-16,
    '64/absorb/fad': 7.14e-16,
    '64/absorb/fad_e2e': 1.27e-15,
    '64/absorb/field_E': 6.77e-16,
    '64/absorb/field_Esq': 6.61e-16,
    '64/absorb/field_H': 7.31e-16,
    '64/absorb/flux_A': 2.15e-16,
    '64/absorb/grad': 9.35e-17,
    '64/absorb/layer/merit_grad': 5.26e-17,
    '64/absorb/layer/merit_resid': 5.42e-16,
    '64/absorb/layer/merit_value': 2.94e-16,
    '64/absorb/needle': 4.78e-16,
    '64/absorb/peak/merit_grad': 6.12e-17,
    '64/absorb/peak/merit_resid': 3.62e-16,
    '64/absorb/peak/merit_value': 1.39e-16,
    '64/absorb/rt_R': 2.2e-15,
    '64/absorb/rt_T': 7.29e-16,
    '64/absorb/rt_eta0': 1.03e-16,
    '64/absorb/rt_eta_sub': 1.25e-16,
    '64/absorb/rt_ml_r': 1.38e-15,
    '64/absorb/rt_ml_t': 9.02e-16,
    '64/absorb/rt_r': 1.71e-15,
    '64/absorb/rt_t': 8.84e-16,
    '64/absorb/tie/merit_grad': 1.85e-16,
    '64/absorb/tie/merit_resid': 7.01e-16,
    '64/absorb/tie/merit_value': 4.05e-16,
    '64/ag2um/field_E': 2.47e-15,
    '64/ag2um/field_Esq': 4.78e-15,
    '64/ag2um/field_H': 2.6e-15,
    '64/ag2um/flux_A': 1.21e-16,
    '64/ag2um/grad': 4.72e-15,
    '64/ag2um/rt_R': 6.16e-16,
    '64/ag2um/rt_T': 4.17e-14,
    '64/ag2um/rt_eta0': 1.03e-16,
    '64/ag2um/rt_eta_sub': 1.25e-16,
    '64/ag2um/rt_ml_r': 9.95e-16,
    '64/ag2um/rt_ml_t': 2.11e-14,
    '64/ag2um/rt_r': 9.95e-16,
    '64/ag2um/rt_t': 2.1e-14,
    '64/ag50/A/merit_grad': 3.77e-17,
    '64/ag50/A/merit_resid': 2.27e-15,
    '64/ag50/A/merit_value': 3.17e-16,
    '64/ag50/Esq/merit_grad': 2.92e-16,
    '64/ag50/Esq/merit_resid': 6.27e-16,
    '64/ag50/Esq/merit_value': 6e-16,
    '64/ag50/R/merit_grad': 4.89e-17,
    '64/ag50/R/merit_resid': 4.63e-16,
    '64/ag50/R/merit_value': 2.8e-16,
    '64/ag50/T/merit_grad': 4.14e-16,
    '64/ag50/T/merit_resid': 4.01e-16,
    '64/ag50/T/merit_value': 2.12e-16,
    '64/ag50/field_E': 3.05e-15,
    '64/ag50/field_Esq': 6.17e-15,
    '64/ag50/field_H': 3.3e-15,
    '64/ag50/flux_A': 2.15e-16,
    '64/ag50/grad': 2.3e-16,
    '64/ag50/layer/merit_grad': 9.8e-17,
    '64/ag50/layer/merit_resid': 7.62e-16,
    '64/ag50/layer/merit_value': 1.69e-16,
    '64/ag50/needle': 5.23e-16,
    '64/ag50/peak/merit_grad': 6.6e-17,
    '64/ag50/peak/merit_resid': 8e-16,
    '64/ag50/peak/merit_value': 1.15e-16,
    '64/ag50/rt_R': 5.83e-16,
    '64/ag50/rt_T': 6.27e-15,
    '64/ag50/rt_eta0': 1.03e-16,
    '64/ag50/rt_eta_sub': 1.25e-16,
    '64/ag50/rt_ml_r': 1.03e-15,
    '64/ag50/rt_ml_t': 3.05e-15,
    '64/ag50/rt_r': 1.03e-15,
    '64/ag50/rt_t': 3.02e-15,
    '64/ag50/tie/merit_grad': 2.92e-16,
    '64/ag50/tie/merit_resid': 6.27e-16,
    '64/ag50/tie/merit_value': 6e-16,
    '64/ambc/field_E': 8.64e-16,
    '64/ambc/field_Esq': 9.06e-16,
    '64/ambc/field_H': 1.38e-15,
    '64/ambc/flux_A': 2.69e-16,
    '64/ambc/grad': 1.38e-16,
    '64/ambc/rt_R': 1.75e-15,
    '64/ambc/rt_T': 3.28e-15,
    '64/ambc/rt_eta0': 1.03e-16,
    '64/ambc/rt_eta_sub': 2.42e-15,
    '64/ambc/rt_ml_r': 2.01e-15,
    '64/ambc/rt_ml_t': 1.37e-15,
    '64/ambc/rt_r': 1.99e-15,
    '64/ambc/rt_t': 2.5e-15,
    '64/critical_R': 5.78e-09,
    '64/dims4/field_H': 5.77e-16,
    '64/dims4/grad': 4.13e-18,
    '64/dims4/rt_r': 2.1e-15,
    '64/dims4/rt_t': 7.27e-16,
    '64/e2e/grad': 1.78e-17,
    '64/e2e/merit_grad': 7.31e-18,
    '64/e2e/merit_value_32': 1.74e-16,
    '64/e2e/merit_value_64': 3.48e-16,
    '64/e2e/needle': 5.52e-16,
    '64/gap/A/merit_grad': 1.74e-17,
    '64/gap/A/merit_resid': 4.01e-15,
    '64/gap/A/merit_value': 4.67e-16,
    '64/gap/Esq/merit_grad': 4.12e-16,
    '64/gap/Esq/merit_resid': 4.03e-15,
    '64/gap/Esq/merit_value': 7.78e-16,
    '64/gap/R/merit_grad': 3.26e-17,
    '64/gap/R/merit_resid': 2.41e-15,
    '64/gap/R/merit_value': 1.53e-16,
    '64/gap/T/merit_grad': 6.16e-17,
    '64/gap/T/merit_resid': 5.77e-16,
    '64/gap/T/merit_value': 2.8e-16,
    '64/gap/fad': 8.77e-15,
    '64/gap/fad_e2e': 5.93e-15,
    '64/gap/field_E': 3.97e-15,
    '64/gap/field_Esq': 4.16e-15,
    '64/gap/field_H': 4.11e-15,
    '64/gap/flux_A': 2.47e-16,
    '64/gap/grad': 4.22e-16,
    '64/gap/layer/merit_grad': 1.02e-16,
    '64/gap/layer/merit_resid': 2.71e-15,
    '64/gap/layer/merit_value': 5.46e-17,
    '64/gap/needle': 1.6e-15,
    '64/gap/peak/merit_grad': 2.51e-16,
    '64/gap/peak/merit_resid': 4.03e-15,
    '64/gap/peak/merit_value': 3.41e-16,
    '64/gap/rt_R': 7.65e-15,
    '64/gap/rt_T': 9.09e-13,
    '64/gap/rt_eta0': 1.53e-16,
    '64/gap/rt_eta_sub': 9.08e-13,
    '64/gap/rt_ml_r': 1.21e-14,
    '64/gap/rt_ml_t': 9.52e-15,
    '64/gap/rt_r': 1.21e-14,
    '64/gap/rt_t': 9.08e-13,
    '64/gap/tie/merit_grad': 4.12e-16,
    '64/gap/tie/merit_resid': 4.03e-15,
    '64/gap/tie/merit_value': 7.78e-16,
    '64/hc200/field_E': 1.02e-13,
    '64/hc200/field_Esq': 1.44e-13,
    '64/hc200/field_H': 1.02e-13,
    '64/hc200/flux_A': 2.18e-16,
    '64/hc200/grad': 9.9e-14,
    '64/hc200/rt_R': 1.61e-13,
    '64/hc200/rt_T': 1.2e-13,
    '64/hc200/rt_eta0': 1.03e-16,
    '64/hc200/rt_eta_sub': 1.25e-16,
    '64/hc200/rt_ml_r': 1.12e-13,
    '64/hc200/rt_ml_t': 1.05e-13,
    '64/hc200/rt_r': 1.1e-13,
    '64/hc200/rt_t': 1.02e-13,
    '64/hl40/field_E': 7.54e-14,
    '64/hl40/field_Esq': 5.46e-14,
    '64/hl40/field_H': 7.42e-14,
    '64/hl40/flux_A': 2.19e-16,
    '64/hl40/grad': 4.23e-14,
    '64/hl40/rt_R': 7.05e-14,
    '64/hl40/rt_T': 4.84e-14,
    '64/hl40/rt_eta0': 1.03e-16,
    '64/hl40/rt_eta_sub': 1.25e-16,
    '64/hl40/rt_ml_r': 2.14e-13,
    '64/hl40/rt_ml_t': 7.38e-14,
    '64/hl40/rt_r': 2.14e-13,
    '64/hl40/rt_t': 7.38e-14,
    '64/layout/merit_grad': 1.29e-16,
    '64/layout/merit_resid': 5.62e-16,
    '64/layout/merit_value': 4.26e-16,
    '64/none/field_E': 2.04e-16,
    '64/none/field_Esq': 3.55e-16,
    '64/none/field_H': 1.98e-16,
    '64/none/rt_R': 1.8e-15,
    '64/none/rt_T': 2.81e-16,
    '64/none/rt_eta0': 1.03e-16,
    '64/none/rt_eta_sub': 1.25e-16,
    '64/none/rt_r': 9.32e-16,
    '64/none/rt_t': 2.04e-16,
    '64/one/field_E': 3.31e-16,
    '64/one/field_Esq': 5.69e-16,
    '64/one/field_H': 3.03e-16,
    '64/one/flux_A': 1.38e-16,
    '64/one/grad': 4.6e-17,
    '64/one/rt_R': 1.04e-14,
    '64/one/rt_T': 4.72e-16,
    '64/one/rt_eta0': 1.03e-16,
    '64/one/rt_eta_sub': 1.25e-16,
    '64/one/rt_ml_r': 6.04e-15,
    '64/one/rt_ml_t': 3.32e-16,
    '64/one/rt_r': 5.28e-15,
    '64/one/rt_t': 3.16e-16,
    '64/pixel/field_E': 6.23e-16,
    '64/pixel/flux_A': 2.64e-16,
    '64/pixel/grad': 1.16e-17,
    '64/pixel/rt_r': 3.06e-15,
    '64/qw/A/merit_grad': 1.24e-17,
    '64/qw/A/merit_resid': 2.34e-15,
    '64/qw/A/merit_value': 2.08e-16,
    '64/qw/Esq/merit_grad': 1.36e-16,
    '64/qw/Esq/merit_resid': 1.06e-15,
    '64/qw/Esq/merit_value': 1.12e-16,
    '64/qw/R/merit_grad': 4.44e-17,
    '64/qw/R/merit_resid': 6.66e-16,
    '64/qw/R/merit_value': 3.16e-16,
    '64/qw/T/merit_grad': 1.16e-16,
    '64/qw/T/merit_resid': 4.71e-16,
    '64/qw/T/merit_value': 1.97e-16,
    '64/qw/fad': 6.54e-16,
    '64/qw/fad_e2e': 6.76e-16,
    '64/qw/field_E': 6e-16,
    '64/qw/field_Esq': 1.09e-15,
    '64/qw/field_H': 5.06e-16,
    '64/qw/flux_A': 1.47e-16,
    '64/qw/grad': 7.13e-17,
    '64/qw/layer/merit_grad': 1.17e-16,
    '64/qw/layer/merit_resid': 6.04e-16,
    '64/qw/layer/merit_value': 2.18e-16,
    '64/qw/needle': 2.49e-16,
    '64/qw/peak/merit_grad': 1.36e-16,
    '64/qw/peak/merit_resid': 1.06e-15,
    '64/qw/peak/merit_value': 1.12e-16,
    '64/qw/rt_R': 7.81e-16,
    '64/qw/rt_T': 6.57e-16,
    '64/qw/rt_eta0': 1.03e-16,
    '64/qw/rt_eta_sub': 1.25e-16,
    '64/qw/rt_ml_r': 4.01e-16,
    '64/qw/rt_ml_t': 5.38e-16,
    '64/qw/rt_r': 5.81e-16,
    '64/qw/rt_t': 6.17e-16,
    '64/qw/tie/merit_grad': 1.36e-16,
    '64/qw/tie/merit_resid': 1.06e-15,
    '64/qw/tie/merit_value': 1.12e-16,
    '64/sweep/grad': 3.59e-17,
    '64/sweep_avg/merit_grad': 3.2e-16,
    '64/sweep_avg/merit_resid': 1.12e-15,
    '64/sweep_avg/merit_value': 7.9e-16,
    '64/sweep_avg/needle': 2.71e-16,
    '64/sweep_s/merit_grad': 2.26e-16,
    '64/sweep_s/merit_resid': 1.88e-15,
    '64/sweep_s/merit_value': 2.49e-16,
    '64/sweep_s/needle': 2.35e-16,
    '64/thick/field_E': 5.85e-13,
    '64/thick/field_Esq': 3.18e-14,
    '64/thick/field_H': 5.92e-13,
    '64/thick/flux_A': 9.7e-17,
    '64/thick/grad_beta': 0.00204,
    '64/thick/rt_R_beta': 0.163,
    '64/thick/rt_T_beta': 0.0775,
    '64/thick/rt_eta0_beta': 0.000497,
    '64/thick/rt_eta_sub_beta': 0.0006,
    '64/thick/rt_ml_r_beta': 0.128,
    '64/thick/rt_ml_t_beta': 1.68,
    '64/thick/rt_r_beta': 0.129,
    '64/thick/rt_t_beta': 1.68,
    '64/zero/A/merit_grad': 4.42e-18,
    '64/zero/A/merit_resid': 1.52e-16,
    '64/zero/A/merit_value': 6.2e-17,
    '64/zero/Esq/merit_grad': 1.77e-16,
    '64/zero/Esq/merit_resid': 6.24e-16,
    '64/zero/Esq/merit_value': 3.8e-16,
    '64/zero/R/merit_grad': 1.6e-17,
    '64/zero/R/merit_resid': 6.62e-16,
    '64/zero/R/merit_value': 4.25e-16,
    '64/zero/T/merit_grad': 6.05e-17,
    '64/zero/T/merit_resid': 5.93e-16,
    '64/zero/T/merit_value': 3.9e-16,
    '64/zero/field_E': 5.78e-16,
    '64/zero/field_Esq': 9.64e-16,
    '64/zero/field_H': 6.37e-16,
    '64/zero/flux_A': 1.65e-16,
    '64/zero/grad': 6.42e-17,
    '64/zero/layer/merit_grad': 9.55e-17,
    '64/zero/layer/merit_resid': 5.2e-16,
    '64/zero/layer/merit_value': 2.15e-16,
    '64/zero/peak/merit_grad': 8.02e-17,
    '64/zero/peak/merit_resid': 8.21e-16,
    '64/zero/peak/merit_value': 2.26e-16,
    '64/zero/rt_R': 1.85e-14,
    '64/zero/rt_T': 6.48e-16,
    '64/zero/rt_eta0': 1.03e-16,
    '64/zero/rt_eta_sub': 1.25e-16,
    '64/zero/rt_ml_r': 7.41e-15,
    '64/zero/rt_ml_t': 4.28e-16,
    '64/zero/rt_r': 9.38e-15,
    '64/zero/rt_t': 4.73e-16,
    '64/zero/tie/merit_grad': 1.77e-16,
    '64/zero/tie/merit_resid': 6.24e-16,
    '64/zero/tie/merit_value': 3.8e-16,
}


def ceiling(name):
    """the CEIL entry of a figure: by its last component, ulps for float32 outputs"""
    fig = name.split('/')[-1]
    if fig.endswith('_acc_ulps'):
        return CEIL['ulps_acc']
    if fig.endswith('_ulps'):
        return CEIL['ulps']
    if fig.endswith('_beta'):
        return CEIL['beta_units']
    key = fig.split('_')[0]
    return CEIL.get(key, CEIL['rt'])


LEDGER = Ledger(MEASURED, ceiling)
check, record = LEDGER.check, LEDGER.record

# ---- cases ----------------------------------------------------------------------------------------------------------
HL = [2.35, 1.46]
_rng = np.random.default_rng(20261019)
STACKS = {
    'none': ([], [], 1.52, 1.0),
    'one': ([1.38], [0.1], 1.52, 1.0),
    'qw': (HL, [0.55 / 4 / n for n in HL], 1.52, 1.0),
    'hl40': (HL * 20, [0.55 / 4 / n * (1 + 0.05 * e) for n, e in zip(HL * 20, _rng.uniform(-1, 1, 40))], 1.52, 1.0),
    'absorb': ([1.38, 1.5 + 0.2j, 2.05], [0.1, 0.05, 0.08], 1.52, 1.0),
    'ag50': ([1.46, 0.05 + 3.9j], [0.08, 0.05], 1.52, 1.0),
    'ag2um': ([1.46, 0.05 + 3.9j], [0.08, 2.0], 1.52, 1.0),
    'gap': ([1.38, 1.0], [0.1, 4.0], 1.7, 1.7),
    'zero': ([1.38, 2.05, 1.46], [0.1, 0.0, 0.09], 1.52, 1.0),
    'hc200': ([4.0, 1.38] * 100, [0.55 / 4 / n for n in [4.0, 1.38] * 100], 1.52, 1.0),
    'ambc': ([1.38, 2.05], [0.1, 0.08], 1.52, 1.5 + 0.01j),
    'thick': ([1.5], [200.0], 1.52, 1.0),
}
GRID_W = np.linspace(0.45, 0.75, 5)[:, None]
GRID_TH = np.radians([0.0, 30.0, 45.0, 89.9])[None, :]
POLS = {'s': T.POL_S, 'p': T.POL_P}


def ops_of(wvl, theta, n0, nsub, n, d):
    """the six device operands (fp64 / complex128), per-layer operands with their layer axis first"""
    r = lambda a: a if isinstance(a, torch.Tensor) else torch.as_tensor(np.asarray(a, np.float64)).cuda()
    c = lambda a: a if isinstance(a, torch.Tensor) else torch.as_tensor(np.asarray(a, np.complex128)).cuda()
    return [r(wvl), r(theta), c(n0), c(nsub), c(n), r(d)]


def stack_case(name, wvl=GRID_W, theta=GRID_TH):
    """(device operands, reference samples) of a stack class on a grid"""
    n, d, sub, amb = STACKS[name]
    n, d = np.asarray(n, np.complex128), np.asarray(d, np.float64)
    return ops_of(wvl, theta, amb, sub, n, d), T.Samples(wvl, theta, amb, sub, n, d)


def beta_units(S):
    """per sample: max(1, sum |Re beta_k|) 2^-53, the phase the inputs leave unknown"""
    b = sum(np.abs(T.Layer(S, k, T.POL_S).beta.real) for k in range(S.N)) if S.N else 0
    return np.maximum(1, np.asarray(b, np.float64)) * 2.0 ** -53


def fig_rel(name, prec, got, ref, units=None):
    """per-sample relative error (fp64) or ulps (float32)"""
    got = host(got).reshape(ref.shape)
    if prec == 32:
        record(f'32/{name}_ulps', T.ulps32(got, ref))
        return
    if units is None:
        record(f'64/{name}', T.rel_per_sample(got, ref))
    else:
        e = np.abs(got.astype(np.clongdouble) - ref) / np.where(np.abs(ref) > 0, np.abs(ref), 1)
        record(f'64/{name}_beta', float(np.max(e / units)))


def fig_bound(name, prec, got, ref):
    """fields (N + 1, P): over each sample's largest boundary magnitude (fp64) or in ulps with that floor (float32)"""
    got = host(got).reshape(ref.shape)
    if not ref.size:
        return
    if prec == 32:
        record(f'32/{name}_ulps', T.ulps32(got, ref, floor=np.abs(ref).max(axis=0)))
    else:
        record(f'64/{name}', T.rel_boundaries(got, ref))


def fig_maj(name, prec, got, ref, maj):
    """sums: |got - ref| over the majorant (fp64), or ulps never below the majorant x 2^-52 (float32)"""
    got = host(got).reshape(np.shape(ref))
    if prec == 32:
        record(f'32/{name}_ulps', T.ulps32(got, ref, floor=maj))
    else:
        record(f'64/{name}', T.over_majorant(got, ref, maj))


# ---- pb_stack_eval --------------------------------------------------------------------------------------------------
FWD = {'r': 0, 't': 1, 'E': 2, 'H': 3, 'R': 4, 'T': 5, 'A': 6, 'Esq': 7, 'eta0': 8, 'eta_sub': 9}


@pytest.mark.parametrize('prec', PRECS)
@pytest.mark.parametrize('pol', POLS)
@pytest.mark.parametrize('cls', STACKS)
def test_stack_eval(pb, cls, pol, prec):
    ops, S = stack_case(cls)
    f = T.forward(S, POLS[pol])
    res = pb._ops.stack_eval(T.COATINGS, POLS[pol], ops, tuple(FWD.values()), RT[prec])
    units = beta_units(S) if cls == 'thick' else None
    for k in ('r', 't', 'R', 'T', 'eta0', 'eta_sub'):
        fig_rel(f'{cls}/rt_{k}', prec, res[FWD[k]], f[k], units)
    for k in ('E', 'H', 'Esq'):
        fig_bound(f'{cls}/field_{k}', prec, res[FWD[k]], f[k])
    if S.N:
        fig_maj(f'{cls}/flux_A', prec, res[FWD['A']], f['A'], f['Amaj'])
    LEDGER.done()


@pytest.mark.parametrize('prec', PRECS)
@pytest.mark.parametrize('pol', POLS)
@pytest.mark.parametrize('cls', [c for c in STACKS if c != 'none'])
def test_multilayer_stack_rt_mode(pb, cls, pol, prec):
    """PB_TF_THINFILM assembly, the angle in degrees through theta_scale"""
    n, d, sub, amb = STACKS[cls]
    deg = np.degrees(GRID_TH)
    ops = ops_of(GRID_W, deg, amb, sub, n, d)
    S = T.Samples(GRID_W, deg, amb, sub, np.asarray(n, complex), np.asarray(d, float), theta_scale=np.pi / 180)
    f = T.forward(S, POLS[pol], T.THINFILM)
    res = pb._ops.stack_eval(T.THINFILM, POLS[pol], ops, (0, 1), RT[prec], theta_scale=np.pi / 180)
    units = beta_units(S) if cls == 'thick' else None
    fig_rel(f'{cls}/rt_ml_r', prec, res[0], f['r'], units)
    fig_rel(f'{cls}/rt_ml_t', prec, res[1], f['t'], units)
    LEDGER.done()


@pytest.mark.parametrize('pol', POLS)
def test_both_sides_of_a_critical_angle(pb, pol):
    """glass ambient (1.7) onto air: a few ulps of the angle either side of arcsin(1 / 1.7) take the two branches of
    the square root as the reference does; lossless total internal reflection gives |r| = 1"""
    tc = np.arcsin(1 / 1.7)
    k = np.array([-256, -64, -16, 16, 64, 256])
    th = tc * (1 + k * 2.0 ** -52)
    ops = ops_of(0.55, th, 1.7, 1.0, np.array([1.38, 2.05]), np.array([0.1, 0.08]))
    S = T.Samples(0.55, th, 1.7, 1.0, np.array([1.38, 2.05], complex), np.array([0.1, 0.08]))
    f = T.forward(S, POLS[pol])
    res = pb._ops.stack_eval(T.COATINGS, POLS[pol], ops, (0, 4), torch.float64)
    R = host(res[4])
    tir = 1.7 * np.sin(th.astype(np.longdouble)) > 1
    assert np.all(tir == (k > 0))
    assert np.all(np.abs(R[tir] - 1) < 1e-14) and np.all(R[~tir] < 1 - 1e-9)
    # sqrt(1 - s^2) has an unbounded slope here: the angle's last-bit sin error moves R by ~1e-8
    check('64/critical_R', float(np.max(np.abs(R - f['R'].astype(float)))))


def test_exact_critical_angle_nan_pattern(pb):
    """at grazing incidence with equal ambient and substrate indices, sin theta = 1 exactly and cos theta_sub = 0: the
    p admittance n / cos is not finite, and the outputs are finite exactly where the reference's are"""
    th = np.array([np.pi / 2, np.pi / 2 - 1e-3])
    for pol in POLS.values():
        ops = ops_of(0.55, th, 1.52, 1.52, np.array([1.38, 2.05]), np.array([0.1, 0.08]))
        S = T.Samples(0.55, th, 1.52, 1.52, np.array([1.38, 2.05], complex), np.array([0.1, 0.08]))
        with np.errstate(all='ignore'):
            f = T.forward(S, pol)
        res = pb._ops.stack_eval(T.COATINGS, pol, ops, (0, 1, 2, 9), torch.float64)
        for k in ('r', 't', 'E', 'eta_sub'):
            got = host(res[FWD[k]])
            assert np.array_equal(np.isfinite(got), np.isfinite(f[k].astype(np.complex128))), (pol, k)
        if pol == T.POL_P:
            assert not np.isfinite(host(res[9])[0])


# ---- pb_stack_grad --------------------------------------------------------------------------------------------------
SEEDS = ('dR', 'dT', 'dA', 'dEsq', 'all')


def seeds_of(S, which, seed):
    """the seeds of a case: standard normals of the full shapes, the one named (or all four), the others None"""
    rng = np.random.default_rng(seed)
    P, N = len(S), S.N
    full = {'dR': rng.standard_normal(P), 'dT': rng.standard_normal(P), 'dA': rng.standard_normal((N, P)),
            'dEsq': rng.standard_normal((N + 1, P))}
    return [full[k] if which in (k, 'all') else None for k in ('dR', 'dT', 'dA', 'dEsq')]


def dev_seeds(sd, shape):
    return [None if s is None else torch.as_tensor(s.reshape(s.shape[:-1] + tuple(shape))).cuda() for s in sd]


def grad_device(pb, ops, pol, kinds, shape, sd, prec):
    res = pb._ops.stack_eval(T.COATINGS, pol, ops, (2, 3), torch.float64)
    return pb._ops.stack_grad(pol, kinds, ops, res[2], res[3], dev_seeds(sd, shape), RT[prec])


@pytest.mark.parametrize('prec', PRECS)
@pytest.mark.parametrize('pol', POLS)
@pytest.mark.parametrize('cls', [c for c in STACKS if c != 'none'])
def test_stack_grad(pb, cls, pol, prec):
    ops, S = stack_case(cls)
    N = S.N
    for j, which in enumerate(SEEDS):
        sd = seeds_of(S, which, j)
        c, m = T.stack_grad(S, POLS[pol], 3, sd)
        ref, maj = c.sum(-1), m.sum(-1)
        if cls == 'thick' and prec == 64:
            maj = maj * beta_units(S).max()
        for kinds, rows in ((1, slice(0, N)), (2, slice(N, 2 * N)), (3, slice(0, 2 * N))):
            got = grad_device(pb, ops, POLS[pol], kinds, S.shape, sd, prec)
            fig_maj(f'{cls}/grad' + ('_beta' if cls == 'thick' else ''), prec, got.reshape(-1), ref[rows], maj[rows])
    LEDGER.done()


def sweep_samples(count, N=2, seed=0):
    """count samples of a 1-D wavelength / angle sweep over a 2-layer stack (the first `count` of any longer run)"""
    i = np.arange(count)
    w = 0.4 + 0.5 * ((i * 0.6180339887498949) % 1)
    th = 1.3 * ((i * 0.7548776662466927) % 1)
    n = np.array([2.35, 1.46 + 0.01j, 1.38, 2.05][:N])
    d = np.array([0.07, 0.11, 0.09, 0.05][:N])
    return (w, th, 1.0, 1.52, n, d), T.Samples(w, th, 1.0, 1.52, n, d)


_BIG = {}


def big(kind, threads, fn):
    """the reference of the longest sweep case of a kind, computed once per module; shorter counts are its prefixes"""
    key = (kind, threads)
    if key not in _BIG:
        _BIG[key] = fn(max(T.straddle_counts(sm_count(), threads)))
    return _BIG[key]


@pytest.mark.parametrize('prec', PRECS)
@pytest.mark.parametrize('idx', range(8))
def test_stack_grad_past_every_warp_slot_and_sweep(pb, idx, prec):
    counts = T.straddle_counts(sm_count(), T.TF_THREADS)
    count = counts[idx]

    def ref(cmax):
        args, S = sweep_samples(cmax)
        sd = seeds_of(S, 'all', 7)
        c, m = T.stack_grad(S, T.POL_S, 3, sd)
        return args, sd, c, m

    args, sd, c, m = big('grad', T.TF_THREADS, ref)
    a = [x[:count] if np.ndim(x) and k < 2 else x for k, x in enumerate(args)]
    sdc = [s[..., :count] for s in sd]
    got = grad_device(pb, ops_of(*a), T.POL_S, 3, (count,), sdc, prec)
    assert T.visits(count, sm_count(), T.TF_THREADS) == (1 if idx < 6 else 3 if idx == 7 else 2)
    check(f'{prec}/sweep/grad' + ('_ulps' if prec == 32 else ''), _fig_value(prec, host(got).reshape(-1),
                                                                              c[:, :count].sum(-1),
                                                                              m[:, :count].sum(-1)))


def _fig_value(prec, got, ref, maj):
    return T.ulps32(got, ref, floor=maj) if prec == 32 else T.over_majorant(got, ref, maj)


# ---- pb_coating_merit -----------------------------------------------------------------------------------------------
MERIT_STACKS = ('qw', 'absorb', 'ag50', 'gap', 'zero')
QUANT = {'R': (T.Q_R, {}), 'T': (T.Q_T, {}), 'A': (T.Q_ABS, dict(b0=1)), 'Esq': (T.Q_ESQ, dict(b0=1)),
         'peak': (T.Q_PEAK, dict(blist=None)), 'tie': (T.Q_PEAK, dict(blist=[1, 2])),
         'layer': (T.Q_LAYER, dict(b0=0, b1=2))}
MPOLS = {'s': T.POL_S, 'p': T.POL_P, 'avg': T.POL_AVG}


def merit_device(pb, ops, quantity, pol, flags, count, N, prec, b0=0, b1=0, blist=None):
    """(value, residuals, gradient) of one pb_coating_merit call (flags: the outputs asked for)"""
    v = torch.zeros(1, dtype=torch.float64, device='cuda')
    res = torch.empty(count, dtype=RT[prec], device='cuda')
    ng = (flags >> 2 & 1) + (flags >> 3 & 1)
    g = torch.empty(ng * N, dtype=RT[prec], device='cuda')
    bl = None
    if blist is not None:
        last = [int(all(blist[j] != blist[i] for j in range(i + 1, len(blist)))) for i in range(len(blist))]
        bl = torch.as_tensor(np.asarray(list(blist) + last, np.int32)).cuda()
    pb._ops.coating_merit(quantity, pol, flags, ops, b0, b1, bl, v, res, g, RT[prec])
    return v, res, g


def merit_figs(name, prec, m, N, got, rows=None):
    """value, residuals and gradient of one term against the reference dict m of T.merit"""
    v, res, g = got
    val = m['val'].sum()
    record(f'64/{name}/merit_value', T.over_majorant(host(v)[:1], np.array([val]), np.array([val])))
    if prec == 32:
        record(f'32/{name}/merit_resid_ulps', T.ulps32(host(res), m['resid'], floor=m['rmaj']))
    else:
        record(f'64/{name}/merit_resid', T.over_majorant(host(res), m['resid'], m['rmaj']))
    if 'der' in m:
        ref, maj = m['der'].sum(-1), m['maj'].sum(-1)
        rows = slice(None) if rows is None else rows
        fig_maj(f'{name}/merit_grad', prec, host(g), ref[rows], maj[rows])


@pytest.mark.parametrize('prec', PRECS)
@pytest.mark.parametrize('pol', MPOLS)
@pytest.mark.parametrize('cls', MERIT_STACKS)
def test_coating_merit(pb, cls, pol, prec):
    ops, S = stack_case(cls)
    N = S.N
    rng = np.random.default_rng(3)
    tg, w = rng.uniform(0, 0.5, S.shape), rng.uniform(0.5, 2.0, S.shape)
    mops = ops + [torch.as_tensor(tg).cuda(), torch.as_tensor(w).cuda()]
    for qname, (q, kw) in QUANT.items():
        kw = dict(kw)
        if q == T.Q_PEAK and kw['blist'] is None:
            kw['blist'] = list(range(N + 1))
        m = T.merit(S, q, MPOLS[pol], tg, w, kinds=3, **kw)
        got = merit_device(pb, mops, q, MPOLS[pol], 1 | 2 | 4 | 8, len(S), N, prec, **kw)
        merit_figs(f'{cls}/{qname}', prec, m, N, got)
        if qname == 'tie':
            # the tie between boundaries 1 and 2 across the zero-thickness layer is exact: the seed goes to the first
            if cls == 'zero':
                assert np.all(T.forward(S, T.POL_S)['Esq'][1] == T.forward(S, T.POL_S)['Esq'][2])
    LEDGER.done()


def merit_sweep_ref(pol, quantity, kw):
    def ref(cmax):
        args, S = sweep_samples(cmax, N=3)
        rng = np.random.default_rng(5)
        tg, w = rng.uniform(0, 0.5, cmax), rng.uniform(0.5, 2.0, cmax)
        return args, tg, w, T.merit(S, quantity, pol, tg, w, kinds=3, **kw)
    return ref


@pytest.mark.parametrize('prec', PRECS)
@pytest.mark.parametrize('idx', range(8))
@pytest.mark.parametrize('pol', ('s', 'avg'))
def test_coating_merit_past_every_warp_slot_and_sweep(pb, pol, idx, prec):
    threads = T.cm_threads(2 if pol == 'avg' else 1)
    count = T.straddle_counts(sm_count(), threads)[idx]
    q, kw = (T.Q_R, {}) if pol == 's' else (T.Q_LAYER, dict(b0=1, b1=3))
    args, tg, w, m = big(('merit', pol), threads, merit_sweep_ref(MPOLS[pol], q, kw))
    a = [x[:count] if np.ndim(x) and k < 2 else x for k, x in enumerate(args)]
    ops = ops_of(*a) + [torch.as_tensor(tg[:count]).cuda(), torch.as_tensor(w[:count]).cuda()]
    mc = {k: v[..., :count] for k, v in m.items()}
    got = merit_device(pb, ops, q, MPOLS[pol], 1 | 2 | 4 | 8, count, 3, prec, **kw)
    merit_figs(f'sweep_{pol}', prec, mc, 3, got)
    LEDGER.done()


@pytest.mark.parametrize('prec', PRECS)
def test_merit_target_and_weight_layouts(pb, prec):
    """stride-0 (scalar) and per-sample target and weight on the (wvl, 1) x (1, theta) grid, one kind at a time"""
    ops, S = stack_case('absorb')
    N = S.N
    rng = np.random.default_rng(11)
    for tg, w in ((0.2, 1.5), (rng.uniform(0, 0.5, S.shape), 0.7), (0.1, rng.uniform(0.5, 2, S.shape))):
        mops = ops + [torch.as_tensor(np.asarray(tg, np.float64)).cuda(), torch.as_tensor(np.asarray(w, np.float64)).cuda()]
        m = T.merit(S, T.Q_ESQ, T.POL_AVG, tg, w, kinds=3, b0=2)
        for kind, rows in ((4, slice(0, N)), (8, slice(N, 2 * N))):
            got = merit_device(pb, mops, T.Q_ESQ, T.POL_AVG, 1 | 2 | kind, len(S), N, prec, b0=2)
            merit_figs('layout', prec, m, N, got, rows)
    LEDGER.done()


# ---- pb_needle ------------------------------------------------------------------------------------------------------
def depth_args(d, z):
    """(zpart device, zlist device, zpart, layer of each depth) as coatings._depth_runs forms them at fp64"""
    N = len(d)
    Z = np.concatenate([[0.0], np.cumsum(np.asarray(d, np.float64))])
    zpart, zl = T.depth_runs(Z, z, N)
    order = np.argsort(zl, kind='stable')
    starts = np.searchsorted(zl[order], np.arange(N + 1))
    zlist = np.concatenate([starts, order]).astype(np.int32)
    return torch.as_tensor(zpart).cuda(), torch.as_tensor(zlist).cuda(), zpart, zl


def needle_depths(d):
    Z = np.concatenate([[0.0], np.cumsum(np.asarray(d, np.float64))])
    return np.concatenate([[-0.02], Z, 0.5 * (Z[1:] + Z[:-1]), [Z[-1] + 0.03]])


@pytest.mark.parametrize('prec', PRECS)
@pytest.mark.parametrize('pol', MPOLS)
@pytest.mark.parametrize('cls', ('qw', 'absorb', 'ag50', 'gap'))
def test_needle(pb, cls, pol, prec):
    ops, S = stack_case(cls)
    n, d, sub, amb = STACKS[cls]
    z = needle_depths(d)
    zp_d, zl_d, zpart, zl = depth_args(d, z)
    nn = 1.38 + 0.004 / GRID_W ** 2                # per wavelength
    rng = np.random.default_rng(13)
    tg, w = rng.uniform(0, 0.5, S.shape), rng.uniform(0.5, 2.0, S.shape)
    for q in (T.Q_R, T.Q_T):
        c, mj = T.needle(S, q, MPOLS[pol], tg, w, nn, zpart, zl)
        nops = ops + [torch.as_tensor(tg).cuda(), torch.as_tensor(w).cuda(),
                      torch.as_tensor(nn.astype(np.complex128)).cuda()]
        P = torch.empty(len(z), dtype=RT[prec], device='cuda')
        pb._ops.needle(q, MPOLS[pol], nops, zp_d, zl_d, P, False)
        fig_maj(f'{cls}/needle', prec, P, c.sum(-1), mj.sum(-1))
    LEDGER.done()


@pytest.mark.parametrize('prec', PRECS)
@pytest.mark.parametrize('idx', (3, 6, 7))
@pytest.mark.parametrize('pol', ('s', 'avg'))
def test_needle_past_every_warp_slot_and_sweep(pb, pol, idx, prec):
    threads = T.cm_threads(2 if pol == 'avg' else 1)
    count = T.straddle_counts(sm_count(), threads)[idx]
    d = np.array([0.07, 0.11])
    z = needle_depths(d)
    zp_d, zl_d, zpart, zl = depth_args(d, z)

    def ref(cmax):
        args, S = sweep_samples(cmax)
        rng = np.random.default_rng(17)
        tg, w = rng.uniform(0, 0.5, cmax), rng.uniform(0.5, 2.0, cmax)
        return args, tg, w, T.needle(S, T.Q_T, MPOLS[pol], tg, w, 1.38, zpart, zl)

    args, tg, w, (c, mj) = big(('needle', pol), threads, ref)
    a = [x[:count] if np.ndim(x) and k < 2 else x for k, x in enumerate(args)]
    nops = ops_of(*a) + [torch.as_tensor(tg[:count]).cuda(), torch.as_tensor(w[:count]).cuda(),
                         torch.as_tensor(np.complex128(1.38)).cuda()]
    P = torch.empty(len(z), dtype=RT[prec], device='cuda')
    pb._ops.needle(T.Q_T, MPOLS[pol], nops, zp_d, zl_d, P, False)
    check(f'{prec}/sweep_{pol}/needle' + ('_ulps' if prec == 32 else ''),
          _fig_value(prec, host(P), c[:, :count].sum(-1), mj[:, :count].sum(-1)))


# ---- pb_field_at_depth ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('prec', PRECS)
@pytest.mark.parametrize('pol', POLS)
@pytest.mark.parametrize('cls', ('absorb', 'gap', 'qw'))
def test_field_at_depth(pb, cls, pol, prec):
    n, d, sub, amb = STACKS[cls]
    wvl, th = 0.55, (1.0 if cls == 'gap' else 0.3)
    N = len(d)
    zb = np.concatenate([[0.0], np.cumsum(np.asarray(d, np.float64))])
    edges = np.concatenate([zb, np.nextafter(zb, -np.inf), np.nextafter(zb, np.inf), [-0.01, zb[-1] + 0.01]])
    dense = np.linspace(0, zb[-1], sweep(sm_count(), T.TF_THREADS) + 33)
    z = np.concatenate([edges, dense])
    ops = ops_of(wvl, th, amb, sub, np.asarray(n), np.asarray(d))
    res = pb._ops.stack_eval(T.COATINGS, POLS[pol], ops, (2, 3), torch.float64)
    Eb, Hb = host(res[2]), host(res[3])
    cd = torch.complex64 if prec == 32 else torch.complex128
    E, H = pb._ops.field_at_depth(POLS[pol], torch.as_tensor(z).cuda(), torch.as_tensor(zb).cuda(), ops[4], amb, wvl,
                                  th, res[2], res[3], cd)
    mag = max(np.abs(Eb).max(), np.abs(Hb).max())
    Er, Hr = T.field_at_depth(z, zb, n, amb, wvl, th, POLS[pol], Eb, Hb)
    S = T.Samples(wvl, th, amb, sub, np.asarray(n, complex), np.asarray(d, float))
    f = T.forward(S, POLS[pol])
    Ee, He = T.field_at_depth(z, zb, n, amb, wvl, th, POLS[pol], f['E'][:, 0], f['H'][:, 0])
    for tag, (er, hr) in (('fad', (Er, Hr)), ('fad_e2e', (Ee, He))):
        for got, ref in ((E, er), (H, hr)):
            got = host(got)
            if prec == 32:
                record(f'32/{cls}/{tag}_ulps', T.ulps32(got, ref, floor=np.full(ref.shape, mag)))
            else:
                record(f'64/{cls}/{tag}', float(np.max(np.abs(got.astype(np.clongdouble) - ref)) / mag))
    LEDGER.done()


# ---- layouts --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('prec', PRECS)
def test_per_pixel_maps_with_a_layer_stride(pb, prec):
    """per-pixel index and thickness maps: the index every other layer of a larger table (layer stride 2 x 8 x 6), the
    thickness pixel-major (layer stride 1)"""
    N, shp = 3, (8, 6)
    rng = np.random.default_rng(23)
    n = (np.array([1.38, 2.05, 1.5 + 0.05j])[:, None, None] * (1 + 0.02 * rng.standard_normal((N,) + shp)))
    d = np.array([0.1, 0.07, 0.05])[:, None, None] * (1 + 0.05 * rng.standard_normal((N,) + shp))
    big_n = torch.zeros((2 * N,) + shp, dtype=torch.complex128, device='cuda')
    big_n[::2] = torch.as_tensor(n).cuda()
    dn = torch.as_tensor(np.ascontiguousarray(np.moveaxis(d, 0, -1))).cuda().permute(2, 0, 1)
    theta = np.radians(np.linspace(0, 60, 48)).reshape(shp)
    ops = ops_of(0.55, theta, 1.0, 1.52, big_n[::2], dn)
    S = T.Samples(0.55, theta, 1.0, 1.52, n, d)
    for pol in POLS.values():
        f = T.forward(S, pol)
        res = pb._ops.stack_eval(T.COATINGS, pol, ops, (0, 1, 2, 6), RT[prec])
        fig_rel('pixel/rt_r', prec, res[0], f['r'])
        fig_bound('pixel/field_E', prec, res[2], f['E'])
        fig_maj('pixel/flux_A', prec, res[6], f['A'], f['Amaj'])
        sd = seeds_of(S, 'all', 29)
        c, m = T.stack_grad(S, pol, 3, sd)
        got = grad_device(pb, ops, pol, 3, shp, sd, prec)
        fig_maj('pixel/grad', prec, got.reshape(-1), c.sum(-1), m.sum(-1))
    LEDGER.done()


@pytest.mark.parametrize('prec', PRECS)
def test_four_dim_collapsed_shape(pb, prec):
    """wavelength, angle, substrate and layer thickness each vary along their own axis: four collapsed dims"""
    w = np.linspace(0.45, 0.7, 2).reshape(2, 1, 1, 1)
    th = np.radians([0.0, 20.0, 50.0]).reshape(1, 3, 1, 1)
    sub = np.linspace(1.45, 1.6, 4).reshape(1, 1, 4, 1)
    d = np.array([0.1, 0.07])[:, None, None, None, None] * np.linspace(0.9, 1.1, 5).reshape(1, 1, 1, 1, 5)
    n = np.array([1.38, 2.05 + 0.01j])
    ops = ops_of(w, th, 1.0, sub, n, d)
    S = T.Samples(w, th, 1.0, sub, n.astype(complex), d)
    for pol in POLS.values():
        f = T.forward(S, pol)
        res = pb._ops.stack_eval(T.COATINGS, pol, ops, (0, 1, 2, 3), RT[prec])
        fig_rel('dims4/rt_r', prec, res[0], f['r'])
        fig_rel('dims4/rt_t', prec, res[1], f['t'])
        fig_bound('dims4/field_H', prec, res[3], f['H'])
        sd = seeds_of(S, 'all', 31)
        c, m = T.stack_grad(S, pol, 3, sd)
        got = grad_device(pb, ops, pol, 3, S.shape, sd, prec)
        fig_maj('dims4/grad', prec, got.reshape(-1), c.sum(-1), m.sum(-1))
    LEDGER.done()


# ---- end to end through prysm_b200.coatings -------------------------------------------------------------------------
@pytest.mark.parametrize('prec', PRECS)
def test_coatings_end_to_end(pb, prec):
    """forward_eval + thickness_gradient, MeritFunction.value_and_grad of two terms (PB_CM_ACCUMULATE) and
    needle_function, against the reference evaluated on the values the device received (float32 thicknesses and
    sample grids at precision 32)"""
    from prysm_b200 import coatings as c
    pb.config.precision = prec
    try:
        n, d, sub, amb = STACKS['absorb']
        st = c.Stack(n, d, sub, amb)
        dd = np.asarray(st.thicknesses, np.float64)
        S = T.Samples(GRID_W, GRID_TH, amb, sub, np.asarray(n, complex), dd)
        N = S.N
        f = c.forward_eval(st, GRID_W, GRID_TH, 'p')
        sd = seeds_of(S, 'all', 37)
        cc, m = T.stack_grad(S, T.POL_P, 1, sd)
        g = c.thickness_gradient(f, **{k: s.reshape(s.shape[:-1] + S.shape) for k, s in zip(SEEDS, sd)})
        fig_maj('e2e/grad', prec, g, cc.sum(-1), m.sum(-1))

        t1 = c.Reflectance(GRID_W, theta=GRID_TH, pol='avg', target=0.05, weight=np.linspace(1, 2, 4)[None, :])
        t2 = c.FieldInLayer(1, GRID_W, theta=GRID_TH, pol='s', target=0.5, weight=1.0)
        v, g = c.MeritFunction([t1, t2]).value_and_grad(st, grad_fn=c.index_gradient)
        val, der, maj = 0, 0, 0
        for t, q, pol, kw in ((t1, T.Q_R, T.POL_AVG, {}), (t2, T.Q_LAYER, T.POL_S, dict(b0=1, b1=2))):
            St = T.Samples(t.wvl, t.theta, amb, sub, np.asarray(n, complex), dd)
            r = T.merit(St, q, pol, t.target, t.weight, kinds=2, **kw)
            val, der, maj = val + r['val'].sum(), der + r['der'].sum(-1), maj + r['maj'].sum(-1)
        record(f'64/e2e/merit_value_{prec}', abs(v - float(val)) / float(val))
        got = host(g)
        if prec == 32:
            record('32/e2e/merit_grad_acc_ulps', T.ulps32(got, der, floor=maj))
        else:
            record('64/e2e/merit_grad', T.over_majorant(got, der, maj))

        tn = c.Transmittance(GRID_W, theta=GRID_TH, pol='s', target=0.9, weight=1.0)
        z = np.concatenate([[0.0], np.cumsum(dd)])
        z = np.concatenate([z, 0.5 * (z[1:] + z[:-1])]).astype(np.float32 if prec == 32 else np.float64)
        P = c.needle_function(st, tn, 1.46, z)
        zpart, zlist = c._depth_runs(st, z)
        zl, zlh = np.empty(len(z), int), host(zlist)
        for k in range(N):
            zl[zlh[N + 1:][zlh[k]:zlh[k + 1]]] = k
        St = T.Samples(tn.wvl, tn.theta, amb, sub, np.asarray(n, complex), dd)
        cn, mn = T.needle(St, T.Q_T, T.POL_S, tn.target, tn.weight, 1.46, host(zpart), zl)
        fig_maj('e2e/needle', prec, P, cn.sum(-1), mn.sum(-1))
    finally:
        pb.config.precision = 64
    LEDGER.done()


def test_every_figure_has_a_measurement():
    """a figure this session reached that has no MEASURED entry is held to the bare ceiling, a bound nobody measured"""
    if os.environ.get('PB_TEST_MEASUREMENTS'):
        pytest.skip('recording figures')
    assert not LEDGER.missing(), f'no MEASURED entry (record them with PB_TEST_MEASUREMENTS): {LEDGER.missing()}'
