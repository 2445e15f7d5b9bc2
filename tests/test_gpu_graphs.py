"""GPU: a CUDA-graph capture of a launch-bound composition replays to the same result as the eager calls, follows
new input data, and refuses calls that would synchronise inside the capture."""
import numpy as np
import pytest
import torch

from gpu_fixtures import pb  # noqa: F401

pytestmark = pytest.mark.gpu
HeNe = 0.6328


@pytest.fixture(scope='module', autouse=True)
def precision_32(pb):
    pb.config.precision = 32


def crand(shape, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return torch.complex(torch.randn(shape, generator=g, device='cuda'), torch.randn(shape, generator=g, device='cuda'))


@pytest.mark.parametrize('kind', ['mdft', 'czt'])
def test_captured_multiresolution_matches_eager(pb, kind):
    P = pb.propagation
    mex = P.prepare_multiresolution(0.05, 128, 4.0, 256, HeNe, 100.0, num_levels=3, fine_samples=128, kind=kind)
    fpm = P.vortex_phase_mask(2)
    a, b = crand((128, 128), 1), crand((128, 128), 2)
    step = pb.graphs.capture(lambda w: P.to_fpm_and_back_multiresolution(w, fpm, mex), a)
    n0 = pb._ops.launch_count()
    for x in (a, b, a):
        got = step(x).clone()
        assert pb._ops.launch_count() == n0                  # replay: no library calls from the host
        want = P.to_fpm_and_back_multiresolution(x, fpm, mex)
        n0 = pb._ops.launch_count()
        assert torch.equal(got, want)                        # same kernels, same order, same bits
    with pytest.raises(TypeError):
        step(a, b)


def test_captured_focus_chain_and_static_inputs(pb):
    P = pb.propagation
    a = crand((256, 256), 3)

    def chain(w):
        psf = P.focus(w, 2)
        return P.unfocus(psf, 1)

    step = pb.graphs.capture(chain, a)
    out = step(a)
    assert float((out - chain(a)).abs().max()) == 0.0
    step.inputs[0].mul_(2.0)                                 # write into the static buffer, replay without a copy
    out2 = step(step.inputs[0])
    assert float((out2 - chain(a * 2.0)).abs().max() / out2.abs().max()) < 1e-6
    with pytest.raises(ValueError):
        pb.graphs.capture(chain, np.zeros((4, 4)))
