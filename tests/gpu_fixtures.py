"""The fixture and helpers the GPU tests share: `from gpu_fixtures import pb, dev, host`, seeded inputs (`crand`), the
launch counters: all kernels (`launches(pb, fn)`) and per route (pb_route_launch_count), which pin which transform
kernels a call ran (`routes_of(fn, codes)`)."""
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


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    return t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)


def crand(shape, seed, dtype=np.complex128, scale=1.0):
    """a seeded complex Gaussian, drawn in fp64 and rounded to `dtype`"""
    rng = np.random.default_rng(seed)
    return ((rng.standard_normal(shape) + 1j * rng.standard_normal(shape)) * scale).astype(dtype)


def sm_count():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def launches(pb, fn):
    """fn()'s result and the kernels it launched"""
    torch.cuda.synchronize()
    c0 = pb._ops.launch_count()
    res = fn()
    torch.cuda.synchronize()
    return res, pb._ops.launch_count() - c0


def _handle():
    from prysm_b200 import _capi
    return _capi.handle_for(torch.cuda.current_device(), torch.cuda.current_stream().cuda_stream)


def route_counts(codes):
    """launches so far on each route of `codes` ({key: route code}), and of every kernel of the handle under 'all'"""
    h = _handle()
    out = {k: h.route_launch_count(c) for k, c in codes.items()}
    out['all'] = h.launch_count()
    return out


def routes_of(fn, codes):
    """fn()'s result and the launches it made, per key of `codes` and 'all' (only the keys it used)"""
    torch.cuda.synchronize()
    c0 = route_counts(codes)
    res = fn()
    c1 = route_counts(codes)
    return res, {k: c1[k] - c0[k] for k in c0 if c1[k] != c0[k]}
