"""GPU: the polychromatic driver against the reference recipe restated by the oracle
(docs/source/how-tos/Polychromatic Propagation.ipynb:86-98), single rank and -- when the box has two
GPUs -- two NCCL ranks."""
import os
import socket

import numpy as np
import pytest
import torch

import prysm_oracle as O
from conftest import rel_linf
from gpu_fixtures import pb  # noqa: F401

pytestmark = pytest.mark.gpu


def reference_sum(amp, opd, wvls, wts, dx, efl, fdx, M, kind):
    ref = np.zeros((M, M))
    N = amp.shape[0]
    for w, wt in zip(wvls, wts):
        ex = O.prepare_executor(dx, (N, N), fdx, (M, M), w, efl, kind=kind)
        ref += wt * O.intensity(ex(O.from_amp_and_phase(amp, opd.astype(np.float64), w)))
    return ref


@pytest.mark.parametrize('kind', ['czt', 'mdft'])
def test_polychromatic_psf_single_rank(pb, kind):
    from prysm_b200.polychromatic import polychromatic_psf
    pb.config.precision = 32
    N, M = 256, 128
    amp, opd, dx = O.synthetic_pupil(N, np.float32)
    wvls = np.linspace(0.5, 0.7, 6)
    wts = np.full(6, 1 / 6)
    out = polychromatic_psf(amp, opd, wvls, wts, dx, 100.0, 2.5, M, kind=kind)
    ref = reference_sum(amp, opd, wvls, wts, dx, 100.0, 2.5, M, kind)
    assert out.dtype == torch.float32 and tuple(out.shape) == (M, M)
    assert rel_linf(out.cpu().numpy(), ref) < 2e-6      # PSF relative L-inf vs the fp64 recipe
    pb.config.precision = 64


def test_polychromatic_fft_grid(pb):
    from prysm_b200.polychromatic import polychromatic_psf_fft
    pb.config.precision = 32
    amp, opd, dx = O.synthetic_pupil(512, np.float32)      # 512 -> tuned packed kernels, fused accumulate
    wvls = np.linspace(0.5, 0.7, 4)
    wts = np.array([0.1, 0.2, 0.3, 0.4])
    out = polychromatic_psf_fft(amp, opd, wvls, wts, Q=2)
    ref = sum(wt * O.intensity(O.focus(O.from_amp_and_phase(amp, opd.astype(np.float64), w), 2)) for w, wt in zip(wvls, wts))
    assert rel_linf(out.cpu().numpy(), ref) < 1e-6
    pb.config.precision = 64


def _nccl_worker(rank, world, port, q):
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=torch.device('cuda', rank))
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'oracle'))
    import prysm_oracle as OO
    import prysm_b200 as pbb
    from prysm_b200.polychromatic import polychromatic_psf
    pbb.config.precision = 32
    amp, opd, dx = OO.synthetic_pupil(256, np.float32)
    wvls = np.linspace(0.5, 0.7, 5)
    wts = np.full(5, 0.2)
    out = polychromatic_psf(amp, opd, wvls, wts, dx, 100.0, 2.5, 128, kind='czt', dst=0)
    torch.cuda.synchronize()
    if rank == 0:
        q.put(out.cpu().numpy())
    dist.barrier()
    dist.destroy_process_group()


def test_polychromatic_two_nccl_ranks(pb):
    if torch.cuda.device_count() < 2:
        pytest.skip('needs two GPUs')
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    procs = [ctx.Process(target=_nccl_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    out = q.get(timeout=300)
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    amp, opd, dx = O.synthetic_pupil(256, np.float32)
    wvls = np.linspace(0.5, 0.7, 5)
    ref = reference_sum(amp, opd, wvls, np.full(5, 0.2), dx, 100.0, 2.5, 128, 'czt')
    assert rel_linf(out, ref) < 2e-6


@pytest.mark.parametrize('precision,N,M', [(32, 512, 256), (32, 1024, 1024), (64, 256, 128)])
def test_native_wavelength_loop_matches_the_python_loop(pb, precision, N, M):
    """pb_polychromatic_czt (the whole loop in one library call, plans one unit ahead on the handle's helper stream) runs
    the same kernels with the same scalars as the per-wavelength Python loop: identical planes.  Called twice to cover the
    reuse of the plan buffers and events across calls."""
    from prysm_b200.polychromatic import polychromatic_psf
    pb.config.precision = precision
    rdt = np.float32 if precision == 32 else np.float64
    amp, opd, dx = O.synthetic_pupil(N, rdt)
    wvls = np.linspace(0.5, 0.7, 5)
    wts = np.array([0.1, 0.3, 0.2, 0.25, 0.15])
    try:
        os.environ['PB_POLY_NATIVE'] = '0'
        loop = polychromatic_psf(amp, opd, wvls, wts, dx, 100.0, 2.5, M, kind='czt')
        os.environ['PB_POLY_NATIVE'] = '1'
        native = polychromatic_psf(amp, opd, wvls, wts, dx, 100.0, 2.5, M, kind='czt')
        again = polychromatic_psf(amp, opd, wvls, wts, dx, 100.0, 2.5, M, kind='czt')
    finally:
        os.environ.pop('PB_POLY_NATIVE', None)
        pb.config.precision = 64
    assert native.dtype == loop.dtype and tuple(native.shape) == (M, M)
    assert torch.equal(native, again)
    assert torch.equal(native, loop)


def test_native_loop_argument_checks(pb):
    from prysm_b200 import _ops
    pb.config.precision = 32
    opd = torch.zeros((64, 64), dtype=torch.float32, device='cuda')
    units = np.zeros((1, 8))
    with pytest.raises(ValueError):
        _ops.polychromatic_czt(None, opd, 32, 128, units, torch.zeros((32, 32), dtype=torch.float64, device='cuda'))   # plane dtype
    with pytest.raises(ValueError):
        _ops.polychromatic_czt(None, opd, 32, 128, np.zeros((1, 7)), torch.zeros((32, 32), dtype=torch.float32, device='cuda'))
    with pytest.raises(ValueError):   # K < n + m - 1: rejected by the library (PB_ERR_INVALID)
        _ops.polychromatic_czt(None, opd, 32, 64, units, torch.zeros((32, 32), dtype=torch.float32, device='cuda'))
    pb.config.precision = 64
