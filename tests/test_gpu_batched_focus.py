"""GPU: the batched focus call (pb_fft2_batch) gives, field for field, exactly what the single-field call gives --
the same kernels index one more dimension -- for every group size, for ragged last groups, on the fused shapes and on
the generic fallback, and for the fused phase-screen input."""
import ctypes as C

import numpy as np
import pytest
import torch

import prysm_oracle as O
from conftest import rel_linf
from gpu_fixtures import pb  # noqa: F401

pytestmark = pytest.mark.gpu


def crand(shape, seed, dt=torch.float32):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return torch.complex(torch.randn(shape, generator=g, device='cuda', dtype=dt), torch.randn(shape, generator=g, device='cuda', dtype=dt))


@pytest.mark.parametrize('n,batch', [(512, 1), (512, 5), (1024, 3), (2048, 9), (96, 4), (100, 3)])
def test_batched_equals_single(pb, n, batch):
    P = pb.propagation
    w = crand((batch, n, n), n + batch)
    got = P.focus(w, 2)                               # (B, 2n, 2n): fused kernels for 512/1024/2048, generic passes otherwise
    assert tuple(got.shape) == (batch, 2 * n, 2 * n)
    for b in range(batch):
        assert torch.equal(got[b], P.focus(w[b], 2)), b
    back = P.unfocus(w, 2)
    for b in (0, batch - 1):
        assert torch.equal(back[b], P.unfocus(w[b], 2))
    ref = O.focus(w[batch - 1].cpu().numpy().astype(np.complex128), 2)
    assert rel_linf(got[batch - 1].cpu().numpy(), ref) < 1e-6


def test_batched_complex128_and_strided_views(pb):
    P = pb.propagation
    w = crand((3, 64, 64), 7, torch.float64)
    got = P.focus(w, 2)
    for b in range(3):
        assert torch.equal(got[b], P.focus(w[b], 2))
    assert rel_linf(got[1].cpu().numpy(), O.focus(w[1].cpu().numpy(), 2)) < 1e-12


def test_batched_phase_screen_input_shared_amplitude(pb):
    """PB_IN_AMP_OPD through the batch entry point: one amplitude for all fields, one OPD per field."""
    from prysm_b200 import _ops
    n, batch = 512, 3
    g = torch.Generator(device='cuda').manual_seed(3)
    amp = torch.rand((n, n), generator=g, device='cuda') > 0.3
    opd = torch.randn((batch, n, n), generator=g, device='cuda') * 60.0
    k = 2 * np.pi / 0.6328 / 1e3
    got = _ops.fft2_batch(None, (2 * n, 2 * n), dir=-1, scale=1.0 / (2 * n), shift_in=True, shift_out=True, amp=amp, opd=opd, kscale=k)
    for b in range(batch):
        one = pb.propagation.psf_from_amp_and_phase(amp, opd[b], 0.6328, 2, field=True)
        assert torch.equal(got[b], one)
    amps = torch.stack([amp, ~amp, amp])
    got2 = _ops.fft2_batch(None, (2 * n, 2 * n), dir=-1, scale=1.0 / (2 * n), shift_in=True, shift_out=True, amp=amps, opd=opd, kscale=k)
    assert torch.equal(got2[1], pb.propagation.psf_from_amp_and_phase(~amp, opd[1], 0.6328, 2, field=True))


def test_wavefront_focus_on_a_stack(pb):
    """Wavefront.focus / unfocus accept a (B, N, N) stack: sample spacing from the last axis, fields batched."""
    P = pb.propagation
    w = crand((3, 512, 512), 11)
    wf = P.Wavefront(w, 0.6328, 10.0 / 512)
    psf = wf.focus(100.0, Q=2)
    one = P.Wavefront(w[1], 0.6328, 10.0 / 512).focus(100.0, Q=2)
    assert psf.dx == one.dx and psf.space == 'psf' and tuple(psf.data.shape) == (3, 1024, 1024)
    assert torch.equal(psf.data[1], one.data)
    back = psf.unfocus(100.0, Q=1)
    assert back.dx == pytest.approx(wf.dx) and tuple(back.data.shape) == (3, 1024, 1024)


def test_batched_fused_intensity(pb):
    P = pb.propagation
    w = crand((5, 512, 512), 21)
    got = P.focus_intensity(w, 2)
    assert got.dtype == torch.float32 and tuple(got.shape) == (5, 1024, 1024)
    for b in (0, 4):
        assert torch.equal(got[b], P.focus_intensity(w[b], 2))
    with pytest.raises(ValueError):
        P.focus_intensity(w, 2, weight=0.5)


WVL = 0.6328
KSCALE = 2 * np.pi / WVL / 1e3     # OPD [nm] -> radians


def screen_inputs(n, nb, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    mask = torch.rand((n, n), generator=g, device='cuda') > 0.3
    opd = torch.randn((nb, n, n), generator=g, device='cuda') * 60.0
    return mask, opd


@pytest.mark.parametrize('n', (512, 2048))
def test_phase_screen_input_equals_focus_of_the_field(pb, n):
    """The fused phase-screen input gives the bits of the same call on the field pb_phase_screen writes:
    psf_from_amp_and_phase against focus(Wavefront.from_amp_and_phase(...).data) as a field, |.|^2 and accumulated |.|^2;
    both directions of pb_fft2; a stack of 3 with one shared bool amplitude through pb_fft2_batch."""
    from prysm_b200 import _ops
    P = pb.propagation
    K = 2 * n
    mask, opd = screen_inputs(n, 3, n)
    field = P.Wavefront.from_amp_and_phase(mask, opd[0], WVL, 0.01).data
    assert torch.equal(P.psf_from_amp_and_phase(mask, opd[0], WVL, 2, field=True), P.focus(field, 2))
    assert torch.equal(P.psf_from_amp_and_phase(mask, opd[0], WVL, 2), P.focus_intensity(field, 2))
    acc0 = torch.rand((K, K), device='cuda')
    assert torch.equal(P.psf_from_amp_and_phase(mask, opd[0], WVL, 2, weight=0.375, out=acc0.clone()),
                       P.focus_intensity(field, 2, weight=0.375, out=acc0.clone()))
    for d in (-1, 1):
        kw = dict(dir=d, scale=1.0 / K, shift_in=True, shift_out=True)
        assert torch.equal(_ops.fft2(None, (K, K), amp=mask, opd=opd[1], kscale=KSCALE, **kw),
                           _ops.fft2(_ops.phase_screen(mask, opd[1], KSCALE), (K, K), **kw)), d
        got = _ops.fft2_batch(None, (K, K), amp=mask, opd=opd, kscale=KSCALE, **kw)
        fields = torch.stack([_ops.phase_screen(mask, opd[b], KSCALE) for b in range(3)])
        assert torch.equal(got, _ops.fft2_batch(fields, (K, K), **kw)), d


@pytest.mark.parametrize('n', (512, 2048))
def test_unaligned_input_equals_aligned(pb, n):
    """A complex input with a base off 16-byte alignment, an odd row pitch or an odd field pitch gives the bits of the
    same values passed contiguous and aligned, in both directions"""
    from prysm_b200 import _ops
    K = 2 * n
    w = crand((3, n, n), n + 7)
    flat = torch.empty(n * n + 1, dtype=torch.complex64, device='cuda')
    mis = flat[1:].view(n, n)
    mis.copy_(w[0])
    assert mis.data_ptr() % 16 == 8
    odd_ld = torch.zeros((n, n + 1), dtype=torch.complex64, device='cuda')[:, :n]
    odd_ld.copy_(w[1])
    bs = n * n + 1
    odd_bs = torch.zeros(3 * bs, dtype=torch.complex64, device='cuda').as_strided((3, n, n), (bs, n, 1))
    odd_bs.copy_(w)
    for d in (-1, 1):
        kw = dict(dir=d, scale=1.0 / K, shift_in=True, shift_out=True)
        assert torch.equal(_ops.fft2(mis, (K, K), **kw), _ops.fft2(w[0], (K, K), **kw)), d
        one = torch.empty((1, K, K), dtype=torch.complex64, device='cuda')
        h, st = _ops._ctx(one)
        for src, nb, in_bs, in_ld, ref in ((odd_ld, 1, 0, n + 1, w[1:2]), (odd_bs, 3, bs, n, w)):
            out = torch.empty((nb, K, K), dtype=torch.complex64, device='cuda')
            h.check(_ops.capi.lib.pb_fft2_batch(
                h.ptr, _ops.capi.PB_C64, C.c_void_p(src.data_ptr()), _ops.capi.IN_COMPLEX, C.c_void_p(0),
                _ops.capi.AMP_NONE, 0.0, nb, in_bs, 0, n, n, in_ld, K, K, d, 1.0 / K, 1, 1, C.c_void_p(out.data_ptr()),
                _ops.capi.OUT_COMPLEX, 1.0, K, K, K, K * K, st))
            assert torch.equal(out, _ops.fft2_batch(ref.contiguous(), (K, K), **kw)), (d, nb)


def test_captured_phase_screen_psf_replays_bit_identically(pb):
    """psf_from_amp_and_phase (phase-screen staging launch + the focus pair) captured in a CUDA graph replays to the
    eager bits, also on new OPD data"""
    P = pb.propagation
    mask, opd = screen_inputs(2048, 2, 5)
    step = pb.graphs.capture(lambda o: P.psf_from_amp_and_phase(mask, o, WVL, 2), opd[0])
    for o in (opd[0], opd[1], opd[0]):
        assert torch.equal(step(o).clone(), P.psf_from_amp_and_phase(mask, o, WVL, 2))
