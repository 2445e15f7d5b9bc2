"""GPU: the focus pipeline's two intermediate buffers (csrc/fft_tuned.cu).

Field f of a stack uses intermediate buffer f mod 2, and the column kernel of field f + 1 runs under the tail of field
f's row kernel instead of waiting for it.  Plane 0 and the head of plane 1 of each intermediate are kept in L2 and
discarded there by the row kernel.  Whatever the number of fields (one buffer, both, an odd tail), and however calls
follow each other on the stream, every field must have the bits of the single-field call.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

N = 2048


@pytest.fixture(scope='module')
def ops():
    if not torch.cuda.is_available():
        pytest.skip('needs a CUDA device')
    from prysm_b200 import _ops
    return _ops


def make_stack(b, n=N, seed=0):
    gen = torch.Generator(device='cuda').manual_seed(1000 + seed)
    return torch.complex(torch.randn((b, n, n), generator=gen, device='cuda'), torch.randn((b, n, n), generator=gen, device='cuda'))


def run(ops, x, d=-1):
    n = x.shape[-1]
    return ops.fft2_batch(x, (2 * n, 2 * n), dir=d, scale=1.0 / (2 * n), shift_in=True, shift_out=True,
                          out_kind=ops.capi.OUT_COMPLEX)


@pytest.mark.parametrize('d', [-1, 1])
@pytest.mark.parametrize('b', [1, 2, 3, 17])
def test_stack_fields_have_the_bits_of_single_calls(ops, b, d):
    x = make_stack(b, seed=b)
    got = run(ops, x, d)
    for f in range(b):
        assert torch.equal(got[f], run(ops, x[f:f + 1], d)[0]), f


@pytest.mark.parametrize('n', [512, 1024])
def test_smaller_sizes_keep_all_of_plane_1(ops, n):
    """At N <= 1024 the whole intermediate is kept in L2 and discarded: a stack still has the single-call bits."""
    x = make_stack(3, n, seed=n)
    for d in (-1, 1):
        got = run(ops, x, d)
        for f in range(3):
            assert torch.equal(got[f], run(ops, x[f:f + 1], d)[0]), (d, f)


def test_back_to_back_calls_match_synchronised_calls(ops):
    stacks = [make_stack(b, seed=20 + i) for i, b in enumerate((3, 2, 5, 1, 4))]
    dirs = [-1, 1, -1, 1, 1]
    ref = []
    for x, d in zip(stacks, dirs):
        ref.append(run(ops, x, d))
        torch.cuda.synchronize()
    got = [run(ops, x, d) for x, d in zip(stacks, dirs)]   # no synchronisation between the calls
    torch.cuda.synchronize()
    for i, (a, r) in enumerate(zip(got, ref)):
        assert torch.equal(a, r), i


def test_graph_of_two_consecutive_calls(ops):
    from prysm_b200 import graphs
    x, y = make_stack(3, seed=40), make_stack(2, seed=41)
    ref = (run(ops, x, -1), run(ops, y, 1))
    torch.cuda.synchronize()
    step = graphs.capture(lambda a, b: (run(ops, a, -1), run(ops, b, 1)), x, y)
    try:
        for _ in range(2):
            a, b = step(x, y)
            torch.cuda.synchronize()
            assert torch.equal(a, ref[0])
            assert torch.equal(b, ref[1])
        x2 = make_stack(3, seed=42)             # new inputs through the same graph
        a, _ = step(x2, y)
        torch.cuda.synchronize()
        assert torch.equal(a, run(ops, x2, -1))
    finally:
        step.close()
