"""GPU: CZT.intensity -- |focus_dft|^2 formed in the store of the last Bluestein pass (pb_czt_axis_intensity) -- equals the
modulus of the complex result, as a fresh array and as a weighted accumulation, on the register engine (K = 2048, 4096),
on the generic kernel (small / complex128) and for a split axis (falls back to the unfused form)."""
import numpy as np
import pytest
import torch

import prysm_oracle as O
from conftest import rel_linf
from gpu_fixtures import pb  # noqa: F401

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('N,M,prec', [(1024, 1024, 32), (2048, 2048, 32), (96, 40, 32), (64, 64, 64), (4096, 512, 32)])
def test_czt_intensity_fused(pb, N, M, prec):
    pb.config.precision = prec
    P = pb.propagation
    rng = np.random.default_rng(N + M)
    cdt = np.complex64 if prec == 32 else np.complex128
    a = (rng.standard_normal((N, N)) + 1j * rng.standard_normal((N, N))).astype(cdt)
    dx = 10.0 / N
    ex = P.prepare_executor(dx, (N, N), 2.5, (M, M), 0.55, 100.0, kind='czt')
    field = ex(pb.asdevice(a))
    want = (field.real.double() ** 2 + field.imag.double() ** 2).cpu().numpy()
    got = ex.intensity(pb.asdevice(a))
    tol = 1e-6 if prec == 32 else 1e-12
    assert got.dtype == (torch.float32 if prec == 32 else torch.float64) and tuple(got.shape) == (M, M)
    assert rel_linf(got.double().cpu().numpy(), want) < tol
    acc = torch.full((M, M), 2.0, dtype=got.dtype, device='cuda')
    r = ex.intensity(pb.asdevice(a), weight=0.25, out=acc)
    assert r is acc
    assert rel_linf(acc.double().cpu().numpy(), 2.0 + 0.25 * want) < tol
    if N <= 2048:
        ref = O.prepare_executor(dx, (N, N), 2.5, (M, M), 0.55, 100.0, kind='czt')(a.astype(np.complex128))
        assert rel_linf(got.double().cpu().numpy(), np.abs(ref) ** 2) < (1.5e-6 if prec == 32 else 1e-12)
    with pytest.raises(ValueError):
        ex.intensity(pb.asdevice(a), out=torch.zeros((M, M), dtype=torch.complex64, device='cuda'))
