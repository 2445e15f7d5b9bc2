"""GPU (>= 2 devices): one process driving two GPUs.  Every kernel with opt-in shared memory (> 48 KB) must launch on
the second device too (the attributes are recorded per handle / device, not in process-wide statics), the C ABI must
leave the caller's current device alone, and the two devices must give bit-identical results."""
import numpy as np
import pytest
import torch

from gpu_fixtures import pb  # noqa: F401

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def two_devices_at_precision_32(pb):
    if torch.cuda.device_count() < 2:
        pytest.skip('needs two CUDA devices in one process')
    pb.config.precision = 32


def test_two_devices_one_process(pb):
    P = pb.propagation
    rng = np.random.default_rng(0)
    a = (rng.standard_normal((1024, 1024)) + 1j * rng.standard_normal((1024, 1024))).astype(np.complex64)
    results = []
    torch.cuda.set_device(0)
    for dev in (0, 1, 0):
        d = torch.from_numpy(a).to(f'cuda:{dev}')
        before = torch.cuda.current_device()
        with torch.cuda.device(dev):
            f = P.focus(d, 2)                                                  # fused focus pipeline (>100 KB smem)
            fs = P.angular_spectrum(d, 0.6328, 0.01, 5.0, Q=1)                # register engine round trip
            ex = P.prepare_executor(0.01, (1024, 1024), 1.5, (128, 128), 0.6328, 100.0, kind='mdft')
            m = ex(d)                                                          # wgmma GEMM (193 KB smem)
            g = pb.otf.mtf_from_psf(f.real ** 2 + f.imag ** 2, 1.0).data      # generic passes
        assert torch.cuda.current_device() == before
        assert f.device.index == dev and fs.device.index == dev and m.device.index == dev
        results.append([t.cpu() for t in (f, fs, m, g)])
    for other in results[1:]:
        for x, y in zip(results[0], other):
            assert torch.equal(x, y)


def test_call_from_a_different_current_device(pb):
    """Tensors on cuda:1 while cuda:0 is current: the library switches to the handle's device and back."""
    P = pb.propagation
    torch.cuda.set_device(0)
    a = torch.randn((512, 512), dtype=torch.complex64, device='cuda:1')
    ref = None
    with torch.cuda.device(1):
        ref = P.focus(a, 2)
    torch.cuda.set_device(0)
    got = P.focus(a, 2)
    assert torch.cuda.current_device() == 0 and got.device.index == 1
    torch.cuda.synchronize(1)
    assert torch.equal(got.cpu(), ref.cpu())
