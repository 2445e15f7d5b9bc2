"""GPU: `(wf * screen).free_space(dz)` with the screen multiply fused into the first transform pass
(pb_angular_spectrum_screen) equals the two-step form and the oracle, on the register engine, the generic kernel,
padded (Q = 2) and odd shapes, complex64 and complex128; the pending product materialises on any other use."""
import numpy as np
import pytest
import torch

import prysm_oracle as O
from conftest import rel_linf
from gpu_fixtures import pb  # noqa: F401

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('shape,Q,prec', [((1024, 1024), 1, 32), ((2048, 2048), 1, 32), ((256, 256), 2, 32), ((96, 80), 1, 32),
                                          ((45, 63), 2, 64), ((128, 128), 1, 64)])
def test_fused_screen_equals_two_step_and_oracle(pb, shape, Q, prec):
    pb.config.precision = prec
    P = pb.propagation
    rng = np.random.default_rng(shape[0] + Q)
    cdt = np.complex64 if prec == 32 else np.complex128
    a = (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype(cdt)
    s = np.exp(1j * rng.normal(0, 0.3, shape)).astype(cdt)
    dx = 10.0 / shape[1]
    wf, scr = P.Wavefront(a, 0.6328, dx), P.Wavefront(s, 0.6328, dx)
    prod = wf * scr
    assert prod._data is None and prod._lazy_mul is not None            # pending
    fused = prod.free_space(dz=5.0, Q=Q).data
    two_step = P.Wavefront(pb._ops.binary('mul', wf.data, scr.data), 0.6328, dx).free_space(dz=5.0, Q=Q).data
    tol = 1e-6 if prec == 32 else 1e-12
    assert rel_linf(fused.cpu().numpy(), two_step.cpu().numpy()) < tol
    ref = O.angular_spectrum(a.astype(np.complex128) * s.astype(np.complex128), 0.6328, dx, 5.0, Q)
    assert rel_linf(fused.cpu().numpy(), ref) < (1.5e-6 if prec == 32 else 1e-12)
    # array API form and a raw tensor operand
    arr = P.angular_spectrum(a, 0.6328, dx, 5.0, Q=Q, screen=s)
    assert torch.equal(arr, fused)
    assert torch.equal((wf * torch.from_numpy(s).cuda()).free_space(dz=5.0, Q=Q).data, fused)


def test_pending_product_materialises(pb):
    pb.config.precision = 32
    P = pb.propagation
    rng = np.random.default_rng(0)
    a = (rng.standard_normal((64, 64)) + 1j * rng.standard_normal((64, 64))).astype(np.complex64)
    s = np.exp(1j * rng.normal(0, 0.3, (64, 64))).astype(np.complex64)
    prod = P.Wavefront(a, 0.5, 0.1) * P.Wavefront(s, 0.5, 0.1)
    assert rel_linf(prod.data.cpu().numpy(), a * s) < 1e-6              # .data materialises
    assert prod._lazy_mul is None
    again = P.Wavefront(a, 0.5, 0.1) * P.Wavefront(s, 0.5, 0.1)
    assert rel_linf(again.focus(10.0, Q=2).data.cpu().numpy(), O.focus((a * s).astype(np.complex128), 2)) < 1e-6
    assert rel_linf(again.intensity.data.cpu().numpy(), np.abs(a * s) ** 2) < 1e-6
    assert (again * 2.0).data.shape == (64, 64)
