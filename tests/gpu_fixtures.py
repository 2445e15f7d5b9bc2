"""The fixture and helper the GPU tests share: `from gpu_fixtures import pb, host`."""
import numpy as np
import pytest
import torch


@pytest.fixture(scope='module')
def pb():
    """prysm_b200, skipped without a CUDA device; on teardown precision 64 and the default backend are back, whatever
    the module's tests left behind."""
    if not torch.cuda.is_available():
        pytest.skip('needs a CUDA device')
    import prysm_b200
    yield prysm_b200
    prysm_b200.config.precision = 64
    prysm_b200.mathops.set_backend_to_defaults()


def host(t):
    return t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)
