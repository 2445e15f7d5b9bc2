"""GPU: the focus pipeline at N = 2048 (column + row kernel pair of csrc/fft_tuned.cu, one pair per field) gives the same
bits however a field reaches it.

In a call on a stack the column kernel of field 0 is a plain launch; those of fields 1, 2, ... are programmatic dependents
of the previous field's row kernel.  They gather their first tile before the wait when the host sees that the input stack
does not overlap the output stack (early input), and wait first when it does.  Every field of a stack must have the
bits of the single-field call, in both directions and for complex, intensity and accumulated-intensity outputs; so must
an output with padded strides, repeated calls, a CUDA-graph replay, and an input stack placed inside the output stack's
allocation.
"""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

N, B = 2048, 3


@pytest.fixture(scope='module')
def ops():
    if not torch.cuda.is_available():
        pytest.skip('needs a CUDA device')
    from prysm_b200 import _ops
    return _ops


@pytest.fixture(scope='module')
def stack(ops):
    gen = torch.Generator(device='cuda').manual_seed(7)
    return torch.complex(torch.randn((B, N, N), generator=gen, device='cuda'), torch.randn((B, N, N), generator=gen, device='cuda'))


def run(ops, x, d=-1, kind=None, out=None):
    kind = ops.capi.OUT_COMPLEX if kind is None else kind
    return ops.fft2_batch(x, (2 * N, 2 * N), dir=d, scale=1.0 / (2 * N), shift_in=True, shift_out=True, out_kind=kind, out=out)


def launches(ops, x, fn):
    """fn() and the number of kernels it launched on x's stream"""
    h = ops._ctx(x)[0]
    n0 = h.launch_count()
    res = fn()
    return res, h.launch_count() - n0


@pytest.mark.parametrize('d', [-1, 1])
def test_each_field_of_a_stack_has_the_bits_of_the_single_field_call(ops, stack, d):
    got, n = launches(ops, stack, lambda: run(ops, stack, d))
    assert n == 2 * B                 # one column + row kernel pair per field
    for b in range(B):
        assert torch.equal(got[b], run(ops, stack[b:b + 1], d)[0]), b


def test_intensity_and_accumulate_per_field(ops, stack):
    capi = ops.capi
    got = run(ops, stack, -1, capi.OUT_INTENSITY)
    for b in range(B):
        assert torch.equal(got[b], run(ops, stack[b:b + 1], -1, capi.OUT_INTENSITY)[0]), b
    gen = torch.Generator(device='cuda').manual_seed(8)
    acc = torch.rand((B, 2 * N, 2 * N), generator=gen, device='cuda')
    one = acc.clone()
    run(ops, stack, 1, capi.OUT_ACCUMULATE, out=acc)
    for b in range(B):
        run(ops, stack[b:b + 1], 1, capi.OUT_ACCUMULATE, out=one[b:b + 1])
        assert torch.equal(acc[b], one[b]), b


def test_padded_output_strides(ops, stack):
    big = torch.zeros((B, 2 * N + 3, 2 * N + 6), dtype=torch.complex64, device='cuda')   # padded field and row strides
    view = big[:, 1:2 * N + 1, 2:2 * N + 2]
    run(ops, stack, -1, out=view)
    assert torch.equal(view, run(ops, stack, -1))
    assert not big[:, 0].any() and not big[:, 2 * N + 1:].any() and not big[:, :, :2].any() and not big[:, :, 2 * N + 2:].any()


def test_repeated_calls_and_graph_replay(ops, stack):
    from prysm_b200 import graphs
    first = run(ops, stack, -1)
    assert torch.equal(first, run(ops, stack, -1))
    step = graphs.capture(lambda w: run(ops, w, -1), stack)
    try:
        assert torch.equal(step(stack), first)
        assert torch.equal(step(stack), first)
    finally:
        step.close()


@pytest.mark.parametrize('d', [-1, 1])
def test_input_inside_the_output_allocation(ops, stack, d):
    """The input stack lies in the never-written padding columns of the output stack's allocation, so the host sees
    overlapping ranges and the column kernels of fields 1, 2 wait before their first gather.  (_ops.fft2_batch copies
    strided inputs, hence the direct C-ABI call.)"""
    capi = ops.capi
    buf = torch.zeros((B, 2 * N, 3 * N), dtype=torch.complex64, device='cuda')
    out = buf[:, :, :2 * N]
    src = buf[:, :N, 2 * N:]          # row pitch 3N (even), 16-byte-aligned base
    src.copy_(stack)
    h, st = ops._ctx(buf)

    def call():
        h.check(capi.lib.pb_fft2_batch(h.ptr, capi.PB_C64, C.c_void_p(src.data_ptr()), capi.IN_COMPLEX, C.c_void_p(0),
                                       capi.AMP_NONE, 0.0, B, src.stride(0), 0, N, N, src.stride(1), 2 * N, 2 * N, d,
                                       1.0 / (2 * N), 1, 1, C.c_void_p(out.data_ptr()), capi.OUT_COMPLEX, 1.0, 2 * N,
                                       2 * N, out.stride(1), out.stride(0), st))

    _, n = launches(ops, buf, call)
    assert n == 2 * B
    assert torch.equal(src, stack)    # the input was not written over
    assert torch.equal(out, run(ops, stack, d))
