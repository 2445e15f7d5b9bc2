"""GPU: BASELINE configs C4 and C5 at their FULL sizes, checked through size-independent properties
(the oracle would need minutes per case at these sizes):

  C5  4096^2 free-space chain: propagating by +z then -z is the identity (|TF| = 1), energy is conserved per
      plane, and two steps of z equal one step of 2z (the transfer functions multiply).
  C4  2048^2 -> 2048^2 fixed-sampling focus: CZT == MDFT (the reference's own identity,
      tests/test_fttools.py:140-155) with the MDFT on the tensor cores, per wavelength; the incoherent sum is
      linear in the weights.
"""
import numpy as np
import pytest
import torch

from gpu_fixtures import pb  # noqa: F401

pytestmark = pytest.mark.gpu
HeNe = 0.6328


@pytest.fixture(scope='module', autouse=True)
def precision_32(pb):
    pb.config.precision = 32


def crand(n, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return torch.complex(torch.randn((n, n), generator=g, device='cuda'), torch.randn((n, n), generator=g, device='cuda'))


def rel(a, b):
    return float((a - b).abs().max() / b.abs().max())


def test_c5_free_space_4096_properties(pb):
    P = pb.propagation
    n = 4096
    dx = 10.0 / n
    f = crand(n, 1)
    wf = P.Wavefront(f, HeNe, dx)
    fwd = wf.free_space(dz=5.0, Q=1)
    e_in = float((f.real ** 2 + f.imag ** 2).sum())
    e_out = float(fwd.intensity.data.double().sum())
    assert abs(e_out / e_in - 1) < 1e-5                                  # unitary step
    back = fwd.free_space(dz=-5.0, Q=1)
    assert rel(back.data, f) < 3e-6                                      # +z then -z
    two = fwd.free_space(dz=5.0, Q=1)
    one = wf.free_space(dz=10.0, Q=1)
    assert rel(two.data, one.data) < 3e-6                                # TF(z) * TF(z) = TF(2z)
    # a phase screen between planes (the C5 chain step) keeps the energy too
    scr = P.Wavefront.phase_screen(torch.randn((n, n), device='cuda') * 30.0, HeNe, dx)
    step = (fwd * scr).free_space(dz=5.0, Q=1)
    assert abs(float(step.intensity.data.double().sum()) / e_in - 1) < 1e-5
    assert step.dx == dx and step.space == 'pupil'


def test_c4_czt_equals_mdft_2048(pb):
    P = pb.propagation
    n = m = 2048
    dx = 10.0 / n
    g = torch.Generator(device='cuda').manual_seed(4)
    yy, xx = torch.meshgrid(torch.arange(n, device='cuda') - n // 2, torch.arange(n, device='cuda') - n // 2, indexing='ij')
    amp = (xx * xx + yy * yy) <= (n // 2) ** 2
    opd = torch.randn((n, n), generator=g, device='cuda') * 40.0
    planes = {}
    for w in (0.5, 0.7):
        wf = P.Wavefront.from_amp_and_phase(amp, opd, w, dx)
        c = wf.focus_dft(wf.prepare_executor(100.0, 2.5, m, kind='czt')).data
        ex = wf.prepare_executor(100.0, 2.5, m, kind='mdft')
        assert ex._tc is not None                                        # 2048^2 -> 2048^2 runs on the wgmma tensor cores
        d = wf.focus_dft(ex).data
        assert rel(c, d) < 5e-6
        planes[w] = (c.real ** 2 + c.imag ** 2)
    from prysm_b200.polychromatic import polychromatic_psf
    tot = polychromatic_psf(amp, opd, [0.5, 0.7], [0.25, 0.75], dx, 100.0, 2.5, m, kind='czt')
    want = 0.25 * planes[0.5] + 0.75 * planes[0.7]
    assert rel(tot, want) < 2e-6
