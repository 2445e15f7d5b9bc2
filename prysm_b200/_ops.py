"""Thin tensor-level wrappers over the C ABI: each function takes CUDA torch tensors (or host
arrays, which are uploaded), allocates the output with torch's caching allocator and makes
exactly one library call on torch's current stream.  PyTorch is plumbing here (device memory,
streams); every kernel is in libprysm_b200.so.  A wrapper makes its call through `_call`, which supplies the handle
and stream and checks the status, and gets its output array from `_out`, which allocates it or validates the caller's.
"""
import math
import ctypes as C

import numpy as np
import torch

from . import _capi as capi
from ._capi import lib

_REAL_OF = {torch.complex64: torch.float32, torch.complex128: torch.float64}
_CPLX_OF = {torch.float32: torch.complex64, torch.float64: torch.complex128}
_CODE = {torch.complex64: capi.PB_C64, torch.complex128: capi.PB_C128,
         torch.float32: capi.PB_C64, torch.float64: capi.PB_C128}
# pb_elem code of typed storage; each wrapper still decides which of these its entry point takes
_ELEM = {torch.float32: capi.ELEM_F32, torch.float64: capi.ELEM_F64, torch.complex64: capi.ELEM_C64,
         torch.complex128: capi.ELEM_C128, torch.uint8: capi.ELEM_U8, torch.uint16: capi.ELEM_U16,
         torch.uint32: capi.ELEM_U32, torch.int32: capi.ELEM_I32, torch.int64: capi.ELEM_I64}

_default_device = None


def set_device(device=None):
    """Select the CUDA device new arrays are placed on (default: torch's current device)."""
    global _default_device
    _default_device = None if device is None else torch.device(device)


def device():
    if _default_device is not None:
        return _default_device
    if not torch.cuda.is_available():
        raise capi.B200Error('no CUDA device is visible: prysm_b200 has no CPU fallback')
    return torch.device('cuda', torch.cuda.current_device())


def torch_dtype(np_or_torch_dtype):
    if isinstance(np_or_torch_dtype, torch.dtype):
        return np_or_torch_dtype
    return {np.dtype('float32'): torch.float32, np.dtype('float64'): torch.float64,
            np.dtype('complex64'): torch.complex64, np.dtype('complex128'): torch.complex128,
            np.dtype('bool'): torch.bool, np.dtype('uint8'): torch.uint8,
            np.dtype('int64'): torch.int64, np.dtype('int32'): torch.int32}[np.dtype(np_or_torch_dtype)]


def asdevice(a, dtype=None):
    """Host array / scalar sequence / tensor -> contiguous CUDA tensor (no copy if already one)."""
    if isinstance(a, torch.Tensor):
        t = a if a.is_cuda else a.to(device(), non_blocking=True)
    else:
        t = torch.as_tensor(np.ascontiguousarray(a)).to(device(), non_blocking=True)
    if dtype is not None and t.dtype != dtype:
        t = t.to(dtype)
    return t.contiguous()


def asnumpy(t):
    return t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)


def ascomplex(t):
    """Promote a real / bool tensor to the complex dtype of matching precision."""
    if t.is_complex():
        return t
    if t.dtype == torch.float64:
        return t.to(torch.complex128)
    return t.to(torch.complex64)


def _ctx(t):
    stream = torch.cuda.current_stream(t.device).cuda_stream
    return capi.handle_for(t.device.index, stream), C.c_void_p(stream)


def _call(fn, like, *args):
    """fn(handle, *args, stream) on the handle and current stream of `like`'s device; a failed status raises."""
    h, st = _ctx(like)
    h.check(fn(h.ptr, *args, st))


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _check_out(out, shape, dtype, device, name='out'):
    """A caller-supplied output goes to the kernel as a raw pointer + row pitch: refuse anything the kernel would
    misread (wrong dtype / shape / device, rows that are not unit-stride) instead of writing out of bounds."""
    if not isinstance(out, torch.Tensor):
        raise TypeError(f'`{name}` must be a torch.Tensor, got {type(out).__name__}')
    if out.dtype != dtype:
        raise ValueError(f'`{name}` has dtype {out.dtype}, the operation writes {dtype}')
    if tuple(out.shape) != tuple(shape):
        raise ValueError(f'`{name}` has shape {tuple(out.shape)}, the operation writes {tuple(shape)}')
    if out.device != device:
        raise ValueError(f'`{name}` is on {out.device}, the input is on {device}')
    if out.ndim and out.stride(-1) != 1:
        raise ValueError(f'`{name}` must have unit stride along its last axis')
    return out


def _out(out, shape, dtype, device, contiguous=True, name='out'):
    """A new (shape) array of dtype on device, or the caller's `out` checked to be exactly that, and contiguous when
    `contiguous` (the kernel then writes a dense array; otherwise it takes the row pitch)."""
    if out is None:
        return torch.empty(shape, dtype=dtype, device=device)
    _check_out(out, shape, dtype, device, name)
    if contiguous and not out.is_contiguous():
        raise ValueError(f'`{name}` must be contiguous')
    return out


def _amp_operand(amp, rdtype):
    """(pb_amp_kind, tensor) of an optional amplitude: a bool / uint8 mask goes as bytes, anything else at rdtype."""
    if amp is None:
        return capi.AMP_NONE, None
    if amp.dtype in (torch.bool, torch.uint8):
        return capi.AMP_U8, amp.contiguous()
    return capi.AMP_REAL, amp.to(rdtype).contiguous()


def _field_operand(field):
    """(src, pb_in_kind, complex dtype) of a transform input: a complex field as is, a real one as IN_REAL (float32
    unless it is float64)."""
    if field.is_complex():
        return field, capi.IN_COMPLEX, field.dtype
    src = field if field.dtype in _CPLX_OF else field.to(torch.float32)
    return src, capi.IN_REAL, _CPLX_OF[src.dtype]


# Host arrays for the library.  numpy allocates at least one byte for an empty array, so an empty sequence still gives
# a valid pointer; the entry points read no element when its count is 0.
def _darr(v):
    v = np.ascontiguousarray(v, dtype=np.float64)
    return v, v.ctypes.data_as(C.POINTER(C.c_double))


def _iarr(v):
    v = np.ascontiguousarray(v, dtype=np.int32)
    return v, v.ctypes.data_as(C.POINTER(C.c_int))


def _nm(nms):
    """the two int32 host arrays (n, m) of a sequence of (n, m) pairs"""
    return _iarr([nm[0] for nm in nms]), _iarr([nm[1] for nm in nms])


# ------------------------------------------------------------------------------------------
def fft2(field, k=None, *, dir=-1, scale=1.0, shift_in=False, shift_out=False, crop=None,
         out_kind=capi.OUT_COMPLEX, weight=1.0, out=None, amp=None, opd=None, kscale=0.0):
    """pb_fft2.  Either `field` (complex or real 2-D tensor) or (amp, opd, kscale)."""
    if opd is not None:
        src, in_kind, cdtype = opd, capi.IN_AMP_OPD, _CPLX_OF[opd.dtype]
        amp_kind, amp_t = _amp_operand(amp, opd.dtype)
    else:
        src, in_kind, cdtype = _field_operand(field)
        amp_kind, amp_t = capi.AMP_NONE, None
    src = src.contiguous()
    ny, nx = src.shape
    ky, kx = (ny, nx) if k is None else k
    oy, ox = (ky, kx) if crop is None else crop
    odt = cdtype if out_kind == capi.OUT_COMPLEX else _REAL_OF[cdtype]
    if out is None and out_kind == capi.OUT_ACCUMULATE:
        raise ValueError('accumulate needs an existing `out` array')
    out = _out(out, (oy, ox), odt, src.device, contiguous=False)
    _call(lib.pb_fft2, src, _CODE[cdtype], _p(src), in_kind, _p(amp_t), amp_kind, float(kscale), ny, nx, nx, ky, kx,
          int(dir), float(scale), int(shift_in), int(shift_out), _p(out), out_kind, float(weight), oy, ox,
          out.stride(0))
    return out


def fft2_batch(fields, k=None, *, dir=-1, scale=1.0, shift_in=False, shift_out=False, out_kind=capi.OUT_COMPLEX, out=None,
               amp=None, opd=None, kscale=0.0, crop=None):
    """pb_fft2_batch over a (B, ny, nx) stack -> (B, ky, kx): either `fields` (complex or real) or `opd` (B, ny, nx)
    with an optional amplitude that is (ny, nx) (shared) or (B, ny, nx).  `crop` = (oy, ox) keeps the centred
    window of each transform, as fft2's does (the adjoints of focus / unfocus)."""
    if opd is not None:
        src = opd if opd.dtype in _CPLX_OF else opd.to(torch.float32)
        in_kind, cdtype = capi.IN_AMP_OPD, _CPLX_OF[src.dtype]
        amp_kind, amp_t = _amp_operand(amp, src.dtype)
    else:
        src, in_kind, cdtype = _field_operand(fields)
        amp_kind, amp_t = capi.AMP_NONE, None
    amp_bs = amp_t.stride(0) if amp_t is not None and amp_t.ndim == 3 else 0
    src = src.contiguous()
    nb, ny, nx = src.shape
    ky, kx = (ny, nx) if k is None else k
    oy, ox = (ky, kx) if crop is None else crop
    odt = cdtype if out_kind == capi.OUT_COMPLEX else _REAL_OF[cdtype]
    given = out is not None
    out = _out(out, (nb, oy, ox), odt, src.device, contiguous=False)
    if given and (out.stride(1) < ox or (nb > 1 and out.stride(0) < (oy - 1) * out.stride(1) + ox)):
        raise ValueError('`out` rows / fields overlap')
    _call(lib.pb_fft2_batch, src, _CODE[cdtype], _p(src), in_kind, _p(amp_t), amp_kind, float(kscale), nb,
          src.stride(0), amp_bs, ny, nx, src.stride(1), ky, kx, int(dir), float(scale), int(shift_in), int(shift_out),
          _p(out), out_kind, 1.0, oy, ox, out.stride(1), out.stride(0))
    return out


def fft1(a, n=None, axis=-1, dir=-1, scale=1.0):
    """pb_fft1: numpy fft(a, n, axis) on a 2-D complex tensor."""
    a = ascomplex(a).contiguous()
    ny, nx = a.shape
    axis = axis % 2
    if n is None:
        n = a.shape[axis]
    oshape = (n, nx) if axis == 0 else (ny, n)
    out = torch.empty(oshape, dtype=a.dtype, device=a.device)
    _call(lib.pb_fft1, a, _CODE[a.dtype], _p(a), ny, nx, nx, axis, int(n), int(dir), float(scale), _p(out), oshape[1])
    return out


def axis_dft(a, n, axis, dir=-1, scale=1.0, pre_e=None, pre_e_conj=False, pre_b=None, pre_b_conj=False,
             post_e=None, post_e_conj=False, post_b=None, post_b_conj=False, out_off=0, n_out=None, out=None):
    """pb_axis_dft: one DFT pass with fused multipliers and an output window; `out`: a contiguous array to write."""
    a = ascomplex(a).contiguous()
    ny, nx = a.shape
    axis = axis % 2
    if n_out is None:
        n_out = n - out_off
    oshape = (n_out, nx) if axis == 0 else (ny, n_out)
    out = _out(out, oshape, a.dtype, a.device)
    _call(lib.pb_axis_dft, a, _CODE[a.dtype], _p(a), ny, nx, nx, axis, int(n), int(dir), float(scale), _p(pre_e),
          int(pre_e_conj), _p(pre_b), int(pre_b_conj), _p(post_e), int(post_e_conj), _p(post_b), int(post_b_conj),
          int(out_off), int(n_out), _p(out), oshape[1])
    return out


def czt_plan(N, M, K, shift, alpha, sign, xc, f0, df, cdtype, dev):
    """pb_czt_plan: (b, post, H, Hadj) for one axis, built on the device."""
    b = torch.empty(N, dtype=cdtype, device=dev)
    post = torch.empty(M, dtype=cdtype, device=dev)
    H = torch.empty(K, dtype=cdtype, device=dev)
    Hadj = torch.empty(K, dtype=cdtype, device=dev)
    _call(lib.pb_czt_plan, b, _CODE[cdtype], int(N), int(M), int(K), float(shift), float(alpha), int(sign), float(xc),
          float(f0), float(df), _p(b), _p(post), _p(H), _p(Hadj))
    return b, post, H, Hadj


def polychromatic_czt(amp, opd, m, K, units, plane):
    """pb_polychromatic_czt: plane += sum_i weight_i |CZT_i(amp exp(i kscale_i opd))|^2 for the rows of `units`
    (host float64 array (n_units, 8): kscale, shift, alpha, xc, f0, df, norm, weight) -- one library call for the loop."""
    opd = opd.contiguous()
    n = opd.shape[0]
    if opd.ndim != 2 or opd.shape[1] != n:
        raise ValueError('a square OPD array is required')
    rdt = opd.dtype
    if rdt not in _CPLX_OF:
        raise ValueError('opd must be float32 or float64')
    amp_kind, amp_t = _amp_operand(amp, rdt)
    if amp_t is not None and tuple(amp_t.shape) != (n, n):
        raise ValueError('amplitude and OPD shapes differ')
    _out(plane, (m, m), rdt, opd.device, name='plane')
    units, up = _darr(units)
    if units.ndim != 2 or units.shape[1] != 8:
        raise ValueError('units must have shape (n_units, 8)')
    code = _CODE[_CPLX_OF[rdt]]
    nbytes = int(lib.pb_polychromatic_czt_work_bytes(code, n, int(m), int(K)))
    work = torch.empty(nbytes + 256, dtype=torch.uint8, device=opd.device)
    off = (-work.data_ptr()) % 256
    _call(lib.pb_polychromatic_czt, opd, code, _p(amp_t), amp_kind, _p(opd), n, int(m), int(K), int(units.shape[0]), up,
          work.data_ptr() + off, _p(plane))
    return plane


def czt_axis(a, K, axis, pre_e, H, post_e, out_off, n_out, scale=1.0, pre_conj=False, post_conj=False,
             out_kind=capi.OUT_COMPLEX, weight=1.0, out=None):
    """pb_czt_axis: (a*pre_e) -> FFT_K -> *H -> IFFT_K -> [out_off:out_off+n_out] -> *post_e*scale along `axis`.
    `a` may be a row-pitched view (a column slice of a larger array): only unit column stride is required."""
    a = ascomplex(a)
    if a.stride(1) != 1 or a.stride(0) < a.shape[1]:
        a = a.contiguous()
    ny, nx = a.shape
    axis = axis % 2
    oshape = (n_out, nx) if axis == 0 else (ny, n_out)
    if out_kind != capi.OUT_COMPLEX:     # |.|^2 (written or accumulated with `weight`) formed in the pass's store
        if out is None and out_kind == capi.OUT_ACCUMULATE:
            raise ValueError('accumulate needs an existing `out` array')
        out = _out(out, oshape, _REAL_OF[a.dtype], a.device, contiguous=False)
        _call(lib.pb_czt_axis_intensity, a, _CODE[a.dtype], _p(a), ny, nx, a.stride(0), axis, int(K), _p(pre_e),
              int(pre_conj), _p(H), _p(post_e), int(post_conj), int(out_off), int(n_out), float(scale), int(out_kind),
              float(weight), _p(out), out.stride(0))
        return out
    out = _out(out, oshape, a.dtype, a.device)
    _call(lib.pb_czt_axis, a, _CODE[a.dtype], _p(a), ny, nx, a.stride(0), axis, int(K), _p(pre_e), int(pre_conj), _p(H),
          _p(post_e), int(post_conj), int(out_off), int(n_out), float(scale), _p(out), oshape[1])
    return out


def angular_spectrum(field, k, ty=None, tx=None, tf=None, conj_tf=False, crop=None, screen=None, conj_screen=False,
                     out=None):
    """pb_angular_spectrum; with `screen` (complex, same shape as the field) pb_angular_spectrum_screen: the field is
    multiplied by the screen inside the first transform pass.  `out`: a contiguous array to write."""
    field = ascomplex(field).contiguous()
    ny, nx = field.shape
    ky, kx = k
    oy, ox = (ky, kx) if crop is None else crop
    out = _out(out, (oy, ox), field.dtype, field.device)
    if tf is not None:
        tf = tf.to(field.dtype).contiguous()
    if screen is not None:
        if tuple(screen.shape) != (ny, nx):
            raise ValueError(f'shape mismatch {(ny, nx)} vs {tuple(screen.shape)}')
        screen = ascomplex(screen).to(field.dtype).contiguous()
        _call(lib.pb_angular_spectrum_screen, field, _CODE[field.dtype], _p(field), _p(screen), int(conj_screen), ny,
              nx, ky, kx, _p(ty), _p(tx), _p(tf), int(conj_tf), _p(out), oy, ox)
        return out
    _call(lib.pb_angular_spectrum, field, _CODE[field.dtype], _p(field), ny, nx, ky, kx, _p(ty), _p(tx), _p(tf),
          int(conj_tf), _p(out), oy, ox)
    return out


_AS_VECTORS = {}     # (shape, wvl, dx, z, dtype, device, stream) -> (ty, tx); most recently used last


def angular_spectrum_vectors(shape, wvl, dx, z, cdtype, dev):
    """The two separable factors of the free-space transfer function (pb_angular_spectrum_vectors).  A plane-to-plane chain
    asks for the same pair at every step (same grid, wavelength and dz): the last few pairs are kept per stream (they are
    read-only, 8 or 16 bytes per sample of one axis), which takes two small launches out of every step of the chain.
    Skipped while a CUDA graph is being captured (a captured graph must own the launches that fill what it reads)."""
    ky, kx = shape
    dev = torch.device(dev)
    capturing = torch.cuda.is_current_stream_capturing() if dev.type == 'cuda' else False
    key = None
    if not capturing and dev.type == 'cuda':
        idx = dev.index if dev.index is not None else torch.cuda.current_device()
        key = (int(ky), int(kx), float(wvl), float(dx), float(z), cdtype, idx, torch.cuda.current_stream(dev).cuda_stream)
        hit = _AS_VECTORS.pop(key, None)
        if hit is not None:
            _AS_VECTORS[key] = hit
            return hit
    ty = torch.empty(ky, dtype=cdtype, device=dev)
    tx = torch.empty(kx, dtype=cdtype, device=dev)
    _call(lib.pb_angular_spectrum_vectors, ty, _CODE[cdtype], ky, kx, float(wvl), float(dx), float(z), _p(ty), _p(tx))
    if key is not None:
        _AS_VECTORS[key] = (ty, tx)
        while len(_AS_VECTORS) > 8:
            _AS_VECTORS.pop(next(iter(_AS_VECTORS)))
    return ty, tx


def mdft_basis(f, x, sign, cdtype, dev):
    """E[j, l] = exp(sign*2*pi*i*f[j]*x[l]) built on the device from fp64 host coordinates."""
    f, fp = _darr(f)
    x, xp = _darr(x)
    E = torch.empty((len(f), len(x)), dtype=cdtype, device=dev)
    _call(lib.pb_mdft_basis, E, _CODE[cdtype], fp, len(f), xp, len(x), int(sign), _p(E))
    return E


def cgemm(A, B, opA=capi.OP_N, opB=capi.OP_N, alpha=1.0):
    m = A.shape[0] if opA in (capi.OP_N, capi.OP_C) else A.shape[1]
    k = A.shape[1] if opA in (capi.OP_N, capi.OP_C) else A.shape[0]
    n = B.shape[1] if opB in (capi.OP_N, capi.OP_C) else B.shape[0]
    kb = B.shape[0] if opB in (capi.OP_N, capi.OP_C) else B.shape[1]
    if k != kb:
        raise ValueError(f'matmul: inner dimensions {k} and {kb} differ')
    A, B = A.contiguous(), B.contiguous()
    out = torch.empty((m, n), dtype=A.dtype, device=A.device)
    _call(lib.pb_cgemm, A, _CODE[A.dtype], opA, opB, m, n, k, float(alpha), _p(A), A.shape[1], _p(B), B.shape[1],
          _p(out), n)
    return out


def mdft_apply(Ey, Ex, a, norm, adjoint, left_first, out=None):
    my, ny = Ey.shape
    mx, nx = Ex.shape
    a = a.contiguous()
    want = (my, mx) if adjoint else (ny, nx)
    if tuple(a.shape) != want:
        raise ValueError(f'array of shape {tuple(a.shape)} does not match the executor ({want})')
    oshape = (ny, nx) if adjoint else (my, mx)
    out = _out(out, oshape, a.dtype, a.device)
    nwork = lib.pb_mdft_work_elems(my, ny, mx, nx, int(adjoint), int(left_first))
    work = torch.empty(nwork, dtype=a.dtype, device=a.device)
    _call(lib.pb_mdft_apply, a, _CODE[a.dtype], _p(Ey), _p(Ex), my, ny, mx, nx, _p(a), _p(out), float(norm),
          int(adjoint), int(left_first), _p(work))
    return out


def mdft_tc_supported(my, ny, mx, nx):
    return bool(lib.pb_mdft_tc_supported(my, ny, mx, nx))


def mdft_tc_expand(E):
    """complex64 basis (m, n) -> TF32-split real expansions (hi, lo), each (2m, 2n) float32."""
    m, n = E.shape
    hi = torch.empty((2 * m, 2 * n), dtype=torch.float32, device=E.device)
    lo = torch.empty_like(hi)
    _call(lib.pb_mdft_tc_expand, E, _p(E), m, n, _p(hi), _p(lo))
    return hi, lo


def _tc_aligned(a):
    """a contiguous, with a 16-byte aligned base: the tensor-core GEMM reads its input through TMA, which needs that.
    A contiguous view at an odd element offset (flat[1:].view(N, N)) is copied; anything else is passed as is."""
    a = a.contiguous()
    return a if a.data_ptr() % 16 == 0 else a.clone()


def mdft_tc_apply(ex_hi, ex_lo, ey_hi, ey_lo, a, norm, out=None):
    my, ny = ey_hi.shape[0] // 2, ey_hi.shape[1] // 2
    mx, nx = ex_hi.shape[0] // 2, ex_hi.shape[1] // 2
    a = _tc_aligned(a)
    if tuple(a.shape) != (ny, nx):
        raise ValueError(f'array of shape {tuple(a.shape)} does not match the executor ({(ny, nx)})')
    out = _out(out, (my, mx), a.dtype, a.device)
    work = torch.empty(lib.pb_mdft_tc_work_bytes(my, ny, mx, nx), dtype=torch.uint8, device=a.device)
    _call(lib.pb_mdft_tc_apply, a, _p(ex_hi), _p(ex_lo), _p(ey_hi), _p(ey_lo), my, ny, mx, nx, _p(a), _p(out),
          float(norm), _p(work))
    return out


def phase_screen(amp, opd, kscale):
    opd = opd.contiguous()
    if opd.dtype not in _CPLX_OF:
        opd = opd.to(torch.float32)
    amp_kind, amp_t = _amp_operand(amp, opd.dtype)
    out = torch.empty(opd.shape, dtype=_CPLX_OF[opd.dtype], device=opd.device)
    _call(lib.pb_phase_screen, opd, _CODE[opd.dtype], _p(amp_t), amp_kind, _p(opd), float(kscale), opd.numel(), _p(out))
    return out


def intensity(field, weight=1.0, out=None):
    field = field.contiguous()
    acc = out is not None
    out = _out(out, field.shape, _REAL_OF[field.dtype], field.device)
    _call(lib.pb_intensity, field, _CODE[field.dtype], _p(field), field.numel(), float(weight), int(acc), _p(out))
    return out


_BINOPS = {'mul': 0, 'truediv': 1, 'add': 2, 'sub': 3}


def binary(op, a, b, reverse=False):
    """a (op) b for complex tensor a and tensor-or-scalar b (pb_binary)."""
    a = a.contiguous()
    if isinstance(b, torch.Tensor):
        if b.shape != a.shape:
            raise ValueError(f'shape mismatch {tuple(a.shape)} vs {tuple(b.shape)}')
        b = b.to(a.dtype).contiguous()
        s = 0j
    else:
        s, b = complex(b), None
    out = torch.empty_like(a)
    _call(lib.pb_binary, a, _CODE[a.dtype], _BINOPS[op], _p(a), _p(b), s.real, s.imag, int(reverse), a.numel(), _p(out))
    return out


def mul_outer(a, vy=None, vx=None, conj_y=False, conj_x=False, scale=1.0, out=None):
    """a[y, x] * vy[y] * vx[x] * scale; `a` may be a strided (sliced) view with unit column stride."""
    if a.stride(1) != 1:
        a = a.contiguous()
    ny, nx = a.shape
    out = _out(out, (ny, nx), a.dtype, a.device, contiguous=False)
    _call(lib.pb_mul_outer, a, _CODE[a.dtype], _p(a), a.stride(0), ny, nx, _p(vy), int(conj_y), _p(vx), int(conj_x),
          float(scale), _p(out), out.stride(0))
    return out


def weighted_sum(modes, weights):
    modes = modes.contiguous()
    k = modes.shape[0]
    w, wp = _darr(weights)
    out = torch.empty(modes.shape[1:], dtype=modes.dtype, device=modes.device)
    _call(lib.pb_weighted_sum, modes, _CODE[modes.dtype], _p(modes), k, out.numel(), wp, _p(out))
    return out


def otf_normalize(D, which):
    D = D.contiguous()
    ny, nx = D.shape
    rd = _REAL_OF[D.dtype]
    mtf = torch.empty((ny, nx), dtype=rd, device=D.device) if which & 1 else None
    ptf = torch.empty((ny, nx), dtype=rd, device=D.device) if which & 2 else None
    otf = torch.empty((ny, nx), dtype=D.dtype, device=D.device) if which & 4 else None
    _call(lib.pb_otf_normalize, D, _CODE[D.dtype], _p(D), ny, nx, which, _p(mtf), _p(ptf), _p(otf))
    return mtf, ptf, otf


def encircled_energy(mtf, df, radii_mm):
    mtf = mtf.contiguous()
    ny, nx = mtf.shape
    r, rp = _darr(radii_mm)
    out = (C.c_double * len(r))()
    _call(lib.pb_encircled_energy, mtf, _CODE[mtf.dtype], _p(mtf), ny, nx, float(df), rp, len(r), out)
    return np.array(out[:])


def moments(data):
    data = data.contiguous()
    if data.dtype not in _CPLX_OF:
        data = data.to(torch.float32)
    ny, nx = data.shape
    sums = (C.c_double * 3)()
    _call(lib.pb_moments, data, _CODE[data.dtype], _p(data), ny, nx, sums)
    return sums[0], sums[1], sums[2]


def mask_multiply(a, m=None, *, b=None, w=None, conj=False, one_minus=False, real_out=False, scale=1.0, out=None):
    """out (+)= scale * (a - b) * f(m) * w in one pass (pb_mask_multiply).  `a`, `b` complex; `m` real or complex
    (f = conj(m) / 1 - m by flag); `w` real; real_out keeps the real part in a real tensor; a given `out` is
    accumulated into."""
    a = a.contiguous()
    rd = _REAL_OF[a.dtype]

    def same(t, name):
        if t is not None and tuple(t.shape) != tuple(a.shape):
            raise ValueError(f'shape mismatch: field {tuple(a.shape)} vs {name} {tuple(t.shape)}')
        return t
    kind = capi.MASK_REAL
    if m is not None:
        m = same(asdevice(m), 'mask')
        if m.is_complex():
            kind, m = capi.MASK_COMPLEX, m.to(a.dtype).contiguous()
        else:
            m = m.to(rd).contiguous()
    b = None if b is None else same(b, 'subtrahend').to(a.dtype).contiguous()
    w = None if w is None else same(asdevice(w), 'window').to(rd).contiguous()
    flags = (capi.MASK_CONJ if conj else 0) | (capi.MASK_ONE_MINUS if one_minus else 0) | \
            (capi.MASK_REAL_OUT if real_out else 0)
    if out is not None:
        flags |= capi.MASK_ACCUMULATE
    out = _out(out, a.shape, rd if real_out else a.dtype, a.device)
    _call(lib.pb_mask_multiply, a, _CODE[a.dtype], _p(a), _p(b), _p(m), kind, flags, _p(w), float(scale), a.numel(),
          _p(out))
    return out


def field_adjoint(mode, field, bar, opd, kscale):
    """Adjoints of from_amp_and_phase (pb_field_adjoint): mode 0 phase (complex out), 1 / 2 amplitude (real out)."""
    bar = bar.contiguous()
    rd = _REAL_OF[bar.dtype]
    field = None if field is None else field.to(bar.dtype).contiguous()
    opd = None if opd is None else asdevice(opd).to(rd).contiguous()
    out = torch.empty(bar.shape, dtype=bar.dtype if mode == 0 else rd, device=bar.device)
    _call(lib.pb_field_adjoint, bar, _CODE[bar.dtype], int(mode), _p(field), _p(bar), _p(opd), float(kscale),
          bar.numel(), _p(out))
    return out


def component(which, field):
    """re / im / angle / abs of a complex tensor as a contiguous real tensor (pb_component)."""
    field = field.contiguous()
    out = torch.empty(field.shape, dtype=_REAL_OF[field.dtype], device=field.device)
    _call(lib.pb_component, field, _CODE[field.dtype], {'real': 0, 'imag': 1, 'angle': 2, 'abs': 3}[which], _p(field),
          field.numel(), _p(out))
    return out


def dot(a, b, w=None):
    """sum w * a * conj(b) as a Python complex (pb_dot; fp64 accumulation)."""
    a = a.contiguous()
    b = b.to(a.dtype).contiguous()
    if a.shape != b.shape:
        raise ValueError(f'shape mismatch {tuple(a.shape)} vs {tuple(b.shape)}')
    w = None if w is None else asdevice(w).to(_REAL_OF[a.dtype]).contiguous()
    out = (C.c_double * 2)()
    _call(lib.pb_dot, a, _CODE[a.dtype], _p(a), _p(b), _p(w), a.numel(), out)
    return complex(out[0], out[1])


def mode_projection(modes, bar):
    """tensordot(modes(k, m, n), bar(m, n)) over the trailing axes (pb_mode_projection) -> host array (k,)."""
    modes = modes.contiguous()
    k = modes.shape[0]
    cplx = bar.is_complex()
    bar = bar.to(_CPLX_OF[modes.dtype] if cplx else modes.dtype).contiguous()
    if tuple(bar.shape) != tuple(modes.shape[1:]):
        raise ValueError(f'shape mismatch: modes {tuple(modes.shape)} vs gradient {tuple(bar.shape)}')
    out = (C.c_double * (2 * k))()
    _call(lib.pb_mode_projection, modes, _CODE[modes.dtype], _p(modes), k, bar.numel(), _p(bar), int(cplx), out)
    v = np.array(out[:]).reshape(k, 2)
    return v[:, 0] + 1j * v[:, 1] if cplx else v[:, 0].copy()


def otf_adjoint_seed(which, bar, D):
    """k-space gradient of mtf (1) / ptf (2) / otf (4) _from_psf_adjoint (pb_otf_adjoint_seed)."""
    D = D.contiguous()
    ny, nx = D.shape
    bar = asdevice(bar)
    bar = bar.to(D.dtype if which == 4 else _REAL_OF[D.dtype]).contiguous()
    if tuple(bar.shape) != (ny, nx):
        raise ValueError(f'shape mismatch: gradient {tuple(bar.shape)} vs transform {(ny, nx)}')
    out = torch.empty_like(D)
    _call(lib.pb_otf_adjoint_seed, D, _CODE[D.dtype], int(which), _p(bar), _p(D), ny, nx, _p(out))
    return out


def encircled_energy_adjoint_seed(shape, df, radii_mm, ee_bar, rdtype, dev):
    ny, nx = shape
    r, rp = _darr(radii_mm)
    b, bp = _darr(ee_bar)
    if len(r) != len(b):
        raise ValueError('one gradient value per radius is required')
    out = torch.empty((ny, nx), dtype=rdtype, device=dev)
    _call(lib.pb_encircled_energy_adjoint_seed, out, _CODE[rdtype], ny, nx, float(df), rp, bp, len(r), _p(out))
    return out


def vortex_phase(charge, xf, yf):
    xf = xf.contiguous()
    yf = yf.to(xf.dtype).contiguous()
    out = torch.empty(xf.shape, dtype=_CPLX_OF[xf.dtype], device=xf.device)
    _call(lib.pb_vortex_phase, xf, _CODE[xf.dtype], int(charge), _p(xf), _p(yf), xf.numel(), _p(out))
    return out


def resample_bilinear(cmap, xf, yf, cx, cy, dx, fill):
    """Bilinear, edge-replicating resampling of a complex map at focal coordinates; `fill` (tensor or scalar) outside."""
    xf = xf.contiguous()
    yf = yf.to(xf.dtype).contiguous()
    cd = _CPLX_OF[xf.dtype]
    cmap = cmap.to(cd).contiguous()
    ny, nx = cmap.shape
    fill_t, fs = None, 0j
    if isinstance(fill, torch.Tensor):
        fill_t = ascomplex(fill).to(cd).expand(xf.shape).contiguous()
    else:
        fs = complex(fill)
    out = torch.empty(xf.shape, dtype=cd, device=xf.device)
    _call(lib.pb_resample_bilinear, xf, _CODE[cd], _p(cmap), ny, nx, _p(xf), _p(yf), xf.numel(), float(cx), float(cy),
          float(dx), _p(fill_t), fs.real, fs.imag, _p(out))
    return out


def radial_window(shape, fdx, shift, here, nxt, rdtype, dev):
    """(window, xf, yf) of one multi-resolution level (pb_radial_window); here / nxt = (a, b) or None."""
    ny, nx = shape
    win, xf, yf = (torch.empty((ny, nx), dtype=rdtype, device=dev) for _ in range(3))
    a0, b0 = here if here is not None else (-1.0, 0.0)
    a1, b1 = nxt if nxt is not None else (-1.0, 0.0)
    _call(lib.pb_radial_window, win, _CODE[rdtype], ny, nx, float(fdx), float(shift), float(a0), float(b0), float(a1),
          float(b1), _p(win), _p(xf), _p(yf))
    return win, xf, yf


def xy_grid(shape, dx, rdtype, dev, want='xy'):
    """Any of x, y, r, t of make_xy_grid / cart_to_polar from one kernel (pb_xy_grid); returns a dict."""
    ny, nx = shape
    out = {k: torch.empty((ny, nx), dtype=rdtype, device=dev) for k in want}
    any_t = next(iter(out.values()))
    _call(lib.pb_xy_grid, any_t, _CODE[rdtype], ny, nx, float(dx), _p(out.get('x')), _p(out.get('y')), _p(out.get('r')),
          _p(out.get('t')))
    return out


def cart_to_polar(x, y):
    x = x.contiguous()
    y = y.to(x.dtype).contiguous()
    r, t = torch.empty_like(x), torch.empty_like(x)
    _call(lib.pb_cart_to_polar, x, _CODE[x.dtype], _p(x), _p(y), x.numel(), _p(r), _p(t))
    return r, t


def circle(r, radius, aa_dx=0.0):
    """bool mask r - radius <= 0, or with aa_dx > 0 the one-sample grey-edge coverage (pb_circle)."""
    r = r.contiguous()
    out = torch.empty(r.shape, dtype=r.dtype if aa_dx > 0 else torch.bool, device=r.device)
    _call(lib.pb_circle, r, _CODE[r.dtype], _p(r), r.numel(), float(radius), float(aa_dx), _p(out))
    return out


def jacobi_seq(ns, alpha, beta, x):
    x = x.contiguous()
    ns = [int(n) for n in ns]
    nmax = max(ns) if ns else 0
    slots = np.full(nmax + 1, -1, dtype=np.int32)
    for i, n in enumerate(ns):
        slots[n] = i
    _, sp = _iarr(slots)
    out = torch.empty((len(ns),) + tuple(x.shape), dtype=x.dtype, device=x.device)
    if not ns:
        return out
    _call(lib.pb_jacobi_seq, x, _CODE[x.dtype], _p(x), x.numel(), nmax, float(alpha), float(beta), sp, _p(out))
    return out


def zernike_seq(nms, a, b, norm, polar):
    a = a.contiguous()
    b = b.to(a.dtype).contiguous()
    k = len(nms)
    out = torch.empty((k,) + tuple(a.shape), dtype=a.dtype, device=a.device)
    if k == 0:
        return out
    (n, nptr), (m, mptr) = _nm(nms)
    _call(lib.pb_zernike_seq, a, _CODE[a.dtype], int(polar), _p(a), _p(b), a.numel(), k, nptr, mptr, int(bool(norm)),
          _p(out))
    return out


def zernike_sum(coefs, nms, a, b, norm, polar):
    a = a.contiguous()
    b = b.to(a.dtype).contiguous()
    k = len(nms)
    out = torch.empty(a.shape, dtype=a.dtype, device=a.device)
    (n, nptr), (m, mptr) = _nm(nms)
    c, cptr = _darr(np.asarray(coefs, dtype=np.float64)[:k])
    _call(lib.pb_zernike_sum, a, _CODE[a.dtype], int(polar), _p(a), _p(b), a.numel(), k, nptr, mptr, cptr,
          int(bool(norm)), _p(out))
    return out


def balance_scale(a, b):
    """Device scalar s = sqrt(sum a^2 / sum b^2) (pb_balance_scale); stays on the device."""
    a = a.contiguous()
    b = b.to(a.dtype).contiguous()
    s = torch.empty(1, dtype=torch.float64, device=a.device)
    _call(lib.pb_balance_scale, a, _CODE[a.dtype], _p(a), _p(b), a.numel(), _p(s))
    return s


def pack_complex(re, im=None, im_scale=None):
    re = re.contiguous()
    if re.dtype not in _CPLX_OF:
        re = re.to(torch.float32)
    im = None if im is None else im.to(re.dtype).contiguous()
    out = torch.empty(re.shape, dtype=_CPLX_OF[re.dtype], device=re.device)
    _call(lib.pb_pack_complex, re, _CODE[re.dtype], _p(re), _p(im), _p(im_scale), re.numel(), _p(out))
    return out


def packed_spectrum_product(Z, scale=1.0, im_scale=None):
    """O*H from Z = FFT2(o + i*s*h) of two real arrays (pb_packed_spectrum_product)."""
    Z = Z.contiguous()
    ny, nx = Z.shape
    out = torch.empty_like(Z)
    _call(lib.pb_packed_spectrum_product, Z, _CODE[Z.dtype], _p(Z), ny, nx, float(scale), _p(im_scale), _p(out))
    return out


def _real2d(a):
    a = asdevice(a)
    if a.dtype not in _CPLX_OF:
        a = a.to(torch.float32)
    return a.contiguous()


def bindown(a, fy, fx, mean):
    a = _real2d(a)
    ny, nx = a.shape
    out = torch.empty((ny // max(fy, 1), nx // max(fx, 1)), dtype=a.dtype, device=a.device)
    _call(lib.pb_bindown, a, _CODE[a.dtype], _p(a), ny, nx, int(fy), int(fx), int(bool(mean)), _p(out))
    return out


def tile(a, fy, fx, scale):
    a = _real2d(a)
    ny, nx = a.shape
    out = torch.empty((ny * fy, nx * fx), dtype=a.dtype, device=a.device)
    _call(lib.pb_tile, a, _CODE[a.dtype], _p(a), ny, nx, int(fy), int(fx), float(scale), _p(out))
    return out


def separable_tf(kind, fx, fy, wx, wy):
    fx = _real2d(fx).reshape(-1)
    fy = _real2d(fy).to(fx.dtype).reshape(-1)
    out = torch.empty((fy.numel(), fx.numel()), dtype=fx.dtype, device=fx.device)
    _call(lib.pb_separable_tf, fx, _CODE[fx.dtype], int(kind), _p(fx), _p(fy), fy.numel(), fx.numel(), float(wx),
          float(wy), _p(out))
    return out


def _real_or_complex2d(a):
    """2-D real (float32 / float64) or complex tensor, contiguous; returns (tensor, is_complex)."""
    a = asdevice(a)
    if a.ndim != 2:
        raise ValueError(f'a 2-D array is required, got shape {tuple(a.shape)}')
    if a.is_complex():
        return a.contiguous(), True
    return _real2d(a), False


def spline_prefilter(a):
    """float64 cubic B-spline coefficients of a real 2-D array (of the real part of a complex one), mirror boundary
    (pb_spline_prefilter; scipy.ndimage.spline_filter(a, 3, output=float64, mode='mirror'))."""
    a, cplx_in = _real_or_complex2d(a)
    ny, nx = a.shape
    out = torch.empty((ny, nx), dtype=torch.float64, device=a.device)
    _call(lib.pb_spline_prefilter, a, _CODE[a.dtype], _p(a), int(cplx_in), ny, nx, _p(out))
    return out


def warp(img, xc=None, yc=None, matrix=None, shape=None, scale=1.0, out=None):
    """scale * map_coordinates(real(img), (yc, xc), order=3, mode='constant', cval=0) (pb_warp).  Either the
    coordinate arrays (same shape; float32 or float64) or a host 3 x 3 `matrix` mapping each output pixel (x, y, 1)
    of an output of `shape` (default: the input's) to input coordinates.  The result has img's real dtype."""
    img, cplx_in = _real_or_complex2d(img)
    ny, nx = img.shape
    rd = _REAL_OF.get(img.dtype, img.dtype)
    mp = None
    if matrix is not None:
        m, mp = _darr(np.asarray(matrix, dtype=np.float64).reshape(9))
        oshape = (ny, nx) if shape is None else tuple(shape)
        cdt, xc_t, yc_t = capi.PB_C128, None, None
    else:
        xc_t, yc_t = asdevice(xc), asdevice(yc)
        if tuple(xc_t.shape) != tuple(yc_t.shape):
            raise ValueError(f'coordinate arrays differ in shape: {tuple(xc_t.shape)} vs {tuple(yc_t.shape)}')
        cd = torch.float64 if torch.float64 in (xc_t.dtype, yc_t.dtype) else torch.float32
        xc_t, yc_t = xc_t.to(cd).contiguous(), yc_t.to(cd).contiguous()
        oshape, cdt = tuple(xc_t.shape), _CODE[cd]
    out = _out(out, oshape, rd, img.device)
    oy, ox = (oshape[0], int(np.prod(oshape[1:]))) if len(oshape) else (1, 1)
    _call(lib.pb_warp, img, _CODE[img.dtype], _p(img), int(cplx_in), ny, nx, _p(xc_t), _p(yc_t), cdt, mp, oy, ox,
          float(scale), _p(out))
    return out


def dm_scatter(act, shape, lattice):
    """poke grid of `shape`: actuators on the lattice (y0, sy, x0, sx), zero elsewhere (pb_dm_scatter)."""
    act = act.contiguous()
    nay, nax = act.shape
    ny, nx = shape
    y0, sy, x0, sx = lattice
    out = torch.empty((ny, nx), dtype=act.dtype, device=act.device)
    _call(lib.pb_dm_scatter, act, _CODE[act.dtype], _p(act), nay, nax, ny, nx, y0, sy, x0, sx, _p(out))
    return out


def dm_gather(a, nact, lattice):
    """real(a) at the lattice points (y0 + k sy, x0 + l sx) -> (nact_y, nact_x) (pb_dm_gather)."""
    a, cplx_in = _real_or_complex2d(a)
    ny, nx = a.shape
    nay, nax = nact
    y0, sy, x0, sx = lattice
    out = torch.empty((nay, nax), dtype=_REAL_OF.get(a.dtype, a.dtype), device=a.device)
    _call(lib.pb_dm_gather, a, _CODE[a.dtype], _p(a), int(cplx_in), ny, nx, nay, nax, y0, sy, x0, sx, _p(out))
    return out


def _real_pair(x, y):
    x = asdevice(x)
    y = None if y is None else asdevice(y)
    rd = torch.float64 if torch.float64 in (x.dtype, getattr(y, 'dtype', None)) else torch.float32
    return x.to(rd).contiguous(), (None if y is None else y.to(rd).contiguous())


def sdf(kind, x, y, params=(), verts=None, mask=False):
    """One signed-distance shape (pb_sdf) on a pair of (ny, nx) grids, or on the separable row (nx values) and
    column (ny values) that optimize_xy_separable reduces them to; y is None for the annulus (x is then r, any
    shape).  Returns the real distance in the coordinates' dtype, or the bool mask sdf <= 0."""
    x, y = _real_pair(x, y)
    if y is None or tuple(x.shape) == tuple(y.shape):
        oshape = tuple(x.shape)
        separable, ny = 0, (oshape[0] if len(oshape) > 1 else 1)
        nx = x.numel() // ny if ny else 0
    else:
        if x.ndim > 2 or y.ndim > 2 or (x.ndim == 2 and x.shape[0] != 1) or (y.ndim == 2 and y.shape[1] != 1):
            raise ValueError(f'x {tuple(x.shape)} and y {tuple(y.shape)} are neither one grid shape nor a row and a column')
        ny, nx = y.numel(), x.numel()
        oshape, separable = (ny, nx), 1
    out = torch.empty(oshape, dtype=torch.bool if mask else x.dtype, device=x.device)
    p, pp = _darr(np.asarray(params, dtype=np.float64).reshape(-1))
    v = np.zeros(0) if verts is None else np.asarray(verts, dtype=np.float64).reshape(-1)
    if len(v) // 2 > capi.SDF_MAX_VERTICES:
        raise ValueError(f'{len(v) // 2} polygon vertices or spider vanes: at most {capi.SDF_MAX_VERTICES} are '
                         'supported')
    v, vp = _darr(v)
    _call(lib.pb_sdf, x, _CODE[x.dtype], int(kind), _p(x), _p(y), separable, int(ny), int(nx), pp, len(p), vp,
          len(v) // 2, int(bool(mask)), _p(out))
    return out


def sdf_combine(op, a, b):
    """min(a, b) / max(a, b) / max(a, -b) of two signed distances (pb_sdf_combine); the two arrays broadcast
    against each other as numpy's minimum / maximum do."""
    a, b = _real_pair(a, b)
    if a.shape != b.shape:
        a, b = (t.contiguous() for t in torch.broadcast_tensors(a, b))
    out = torch.empty_like(a)
    _call(lib.pb_sdf_combine, a, _CODE[a.dtype], int(op), _p(a), _p(b), a.numel(), _p(out))
    return out


def hex_segments(x, y, tiles, seg, geo, nverts, dx, total):
    """Coverage, local x, local y of every segment window, packed (`total` samples each), and the amplitude
    (pb_hex_segments).  tiles = (tiles_y, tiles_x, tile_ptr, tile_seg); seg / geo are the device tables."""
    ny, nx = x.shape
    ty, tx, ptr, lst = tiles
    cover, lx, ly = (torch.empty(total, dtype=x.dtype, device=x.device) for _ in range(3))
    amp = torch.empty((ny, nx), dtype=x.dtype, device=x.device)
    _call(lib.pb_hex_segments, x, _CODE[x.dtype], _p(x), _p(y), ny, nx, ty, tx, _p(ptr), _p(lst), _p(seg), _p(geo),
          int(nverts), float(dx), _p(cover), _p(lx), _p(ly), _p(amp))
    return cover, lx, ly, amp


def segment_compose(tiles, seg, masks, bases, nmodes, coefs, ncoef, out):
    """out += the masked per-segment modal sums of the first `ncoef` segments (pb_segment_compose); coefs is a
    contiguous (n, nmodes) float64 device tensor."""
    ny, nx = out.shape
    ty, tx, ptr, lst = tiles
    _call(lib.pb_segment_compose, out, _CODE[out.dtype], ny, nx, ty, tx, _p(ptr), _p(lst), _p(seg), _p(masks),
          _p(bases), int(nmodes), _p(coefs), int(nmodes), int(ncoef), _p(out))
    return out


def segment_compose_adjoint(seg, nseg, masks, bases, nmodes, opdbar, max_window):
    """(nseg, nmodes) = per-segment windowed projections of opdbar * mask onto the basis (pb_segment_compose_adjoint)."""
    ny, nx = opdbar.shape
    nchunk = max(1, -(-int(max_window) // capi.SEGMENT_CHUNK))
    out = torch.empty((nseg, nmodes), dtype=opdbar.dtype, device=opdbar.device)
    _call(lib.pb_segment_compose_adjoint, opdbar, _CODE[opdbar.dtype], ny, nx, int(nseg), _p(seg), _p(masks), _p(bases),
          int(nmodes), _p(opdbar), nchunk, _p(out))
    return out


def jones_planar(src, cdtype, out=None):
    """A (rows, cols, 2, 2) device tensor of any strides, real or complex -> its 4 element planes (4, rows, cols) at
    `cdtype` (pb_jones_planar)."""
    rows, cols = src.shape[:2]
    out = _out(out, (4, rows, cols), cdtype, src.device)
    _call(lib.pb_jones_planar, src, _CODE[cdtype], _p(src), _ELEM[src.dtype], rows, cols, *src.stride(), _p(out))
    return out


def jones_product(mode, n, a, b, out, consts=None):
    """out = op(A) (x) op(B) over n pixels (pb_jones_product); a / b = (kind, tensor or None, op), consts = 4 + 4
    complex values of the constant operands."""
    (ak, at, ao), (bk, bt, bo) = a, b
    c = np.zeros(16) if consts is None else np.asarray(consts, dtype=np.complex128).view(np.float64)
    c, cp = _darr(c)
    _call(lib.pb_jones_product, out, _CODE[out.dtype], int(mode), int(n), int(ak), _p(at), int(ao), int(bk), _p(bt),
          int(bo), cp, _p(out))
    return out


def jones_elements(kind, n, params, out, plane=None):
    """4 planes of one Jones constructor over n pixels (pb_jones_elements); plane: optional real device tensor."""
    p, pp = _darr(np.asarray(params, dtype=np.float64).reshape(-1))
    ptype = _ELEM[plane.dtype] if plane is not None else 0
    _call(lib.pb_jones_elements, out, _CODE[out.dtype], int(kind), int(n), _p(plane), ptype, pp, len(p), _p(out))
    return out


def jones_reduce(kind, n, a, out, b=None):
    """Mueller (16 real planes), Kronecker (16 complex planes) or Pauli (4 planes) of 4-plane operands (pb_jones_reduce)."""
    _call(lib.pb_jones_reduce, a, _CODE[a.dtype], int(kind), int(n), _p(a), _p(b), _p(out))
    return out


def lp_modes(r, t, a, plan, out=None):
    """(P, *r.shape) LP / single-mode fiber fields of the real radius (and angle) grids (pb_lp_modes); plan is a
    (P, 6) host array of l, ld, U, W, rule, az rows."""
    r = r.contiguous()
    t = None if t is None else t.to(r.dtype).contiguous()
    plan, pp = _darr(np.asarray(plan, dtype=np.float64).reshape(-1, 6))
    P = plan.shape[0]
    out = _out(out, (P, *r.shape), r.dtype, r.device, contiguous=False)
    _call(lib.pb_lp_modes, r, _CODE[r.dtype], _p(r), _p(t), r.numel(), float(a), P, pp, _p(out))
    return out


def overlap(E, modes, ip=None, ie=None, want_c=False):
    """eta_p = |sum conj(M_p) E|^2 / (I_p I_E) for every mode (pb_overlap), as one (P,) device tensor of E's real
    type, and sqrt(I_E eta_0) as a 0-d device tensor when want_c.  `modes` is one packed (P, *E.shape) tensor or a
    sequence of P tensors of E's shape (passed as pointers, never gathered); ip (P,) / ie (1,) are optional fp64 device
    tensors of the intensity sums."""
    E = E.contiguous()
    rd = _REAL_OF[E.dtype]
    n = E.numel()
    if isinstance(modes, torch.Tensor):
        packed, ptrs, P, first = modes.contiguous(), None, modes.shape[0], modes
        if tuple(packed.shape[1:]) != tuple(E.shape):
            raise ValueError(f'modes {tuple(packed.shape)} do not match the field {tuple(E.shape)}')
        keep = (packed,)
    else:
        keep = tuple(m.contiguous() for m in modes)
        P, first = len(keep), keep[0]
        packed = None
        for m in keep:
            if tuple(m.shape) != tuple(E.shape) or m.dtype != first.dtype or m.device != E.device:
                raise ValueError('every mode must be a device tensor of the field\'s shape, all of one dtype')
        ptrs = (C.c_void_p * P)(*[m.data_ptr() for m in keep])
    mc = first.is_complex()
    if (_REAL_OF[first.dtype] if mc else first.dtype) != rd:
        raise ValueError(f'modes of {first.dtype} with a field of {E.dtype}')
    eta = torch.empty(P, dtype=rd, device=E.device)
    c = torch.empty((), dtype=rd, device=E.device) if want_c else None
    _call(lib.pb_overlap, E, _CODE[E.dtype], _p(E), n, P, _p(packed), ptrs, int(mc), _p(ip), _p(ie), _p(eta), _p(c))
    del keep
    return eta, c


def wfs_combine(a, alpha=1.0, b=None, beta=1.0, alpha_scale=None, beta_scale=None, real_out=False):
    """alpha a + beta b, or |alpha a + beta b|^2 with real_out (pb_wfs_combine); alpha / beta are host complex numbers,
    each optionally times a 0-d real device tensor."""
    a = a.contiguous()
    if b is not None:
        if tuple(b.shape) != tuple(a.shape):
            raise ValueError(f'shape mismatch {tuple(a.shape)} vs {tuple(b.shape)}')
        b = b.to(a.dtype).contiguous()
    rd = _REAL_OF[a.dtype]
    al, be = complex(alpha), complex(beta)
    k, kp = _darr([al.real, al.imag, be.real, be.imag])
    sa = None if alpha_scale is None else alpha_scale.to(rd).contiguous()
    sb = None if beta_scale is None else beta_scale.to(rd).contiguous()
    out = torch.empty(a.shape, dtype=rd if real_out else a.dtype, device=a.device)
    _call(lib.pb_wfs_combine, a, _CODE[a.dtype], a.numel(), _p(a), _p(b), kp, _p(sa), _p(sb), int(real_out), _p(out))
    return out


def grating(kind, x, params, shift=0.0, E=None):
    """E * g(x + shift), or g itself when E is None (pb_grating); x real, the arithmetic in fp64."""
    x = x.contiguous()
    if E is not None:
        E = E.to(_CPLX_OF[x.dtype]).contiguous()
        if tuple(E.shape) != tuple(x.shape):
            raise ValueError(f'shape mismatch {tuple(E.shape)} vs grid {tuple(x.shape)}')
    p, pp = _darr(params)
    out = torch.empty(x.shape, dtype=x.dtype if E is None else E.dtype, device=x.device)
    _call(lib.pb_grating, x, _CODE[x.dtype], int(kind), x.numel(), _p(x), float(shift), pp, len(p), _p(E), _p(out))
    return out


def psi(frames, s, c, num_dtype, phase_dtype, want_num=True, want_phase=True):
    """num = sum s_k g_k, den = sum c_k g_k and phase = atan2(num, den) in one pass over the frames (pb_psi): a (N, ...)
    tensor or a sequence of N tensors of one shape and dtype (passed as pointers, never stacked)."""
    if isinstance(frames, torch.Tensor):
        stack, ptrs, N, f0 = frames.contiguous(), None, frames.shape[0], frames[0]
        keep = (stack,)
    else:
        keep = tuple(f.contiguous() for f in frames)
        N, f0, stack = len(keep), keep[0], None
        for f in keep:
            if f.shape != f0.shape or f.dtype != f0.dtype or f.device != f0.device:
                raise ValueError('every frame must have one shape, dtype and device')
        ptrs = (C.c_void_p * N)(*[f.data_ptr() for f in keep])
    if f0.dtype not in (torch.float32, torch.float64, torch.uint16, torch.int32):
        raise ValueError(f'frames of {f0.dtype} are not supported (float32, float64, uint16, int32)')
    shape, n = tuple(f0.shape), f0.numel()
    s, sp = _darr(s)
    c, cp = _darr(c)
    if len(s) != N or len(c) != N:
        raise ValueError(f'{N} frames but {len(s)} / {len(c)} weights')
    num = torch.empty(shape, dtype=num_dtype, device=f0.device) if want_num else None
    den = torch.empty(shape, dtype=num_dtype, device=f0.device) if want_num else None
    phase = torch.empty(shape, dtype=phase_dtype, device=f0.device) if want_phase else None
    _call(lib.pb_psi, f0, _ELEM[f0.dtype], N, ptrs, _p(stack), n, n, sp, cp, _ELEM[num_dtype], _p(num), _p(den),
          _ELEM[phase_dtype], _p(phase))
    del keep
    return num, den, phase


_CODE_BYTES = {torch.uint8: 1, torch.uint16: 2, torch.uint32: 4}


def rows_view(m, shape):
    """(map, row stride, column stride) through which an operand broadcast against `shape` is read as the (rows, last
    axis) view of that shape: a broadcast dimension is stride 0, never materialised.  An operand whose broadcast cannot
    be read that way is made contiguous at `shape`."""
    nx = shape[-1] if shape else 1
    rows = math.prod(shape[:-1]) if shape else 1
    e = m.expand(shape) if shape else m.reshape(())
    try:
        v = e.view(rows, nx) if shape else e.reshape(1, 1)
    except RuntimeError:
        v = e.contiguous().view(rows, nx)
    return v, v.stride(0), v.stride(1)


def _flags_read(flags, words):
    """The call's one synchronisation: the first `words` uint32 of the device flag buffer, to the host."""
    return [int(v) & 0xFFFFFFFF for v in flags[:words].cpu().tolist()]


def expose(aerial, prnu, dcnu, params, frames, key, code_dtype, lut=None):
    """(frames, *shape) detector frames of code_dtype (or of the LUT's dtype) in one launch (pb_expose); returns
    (out, flags) where flags are the host copy of the kernel's error words."""
    shape = tuple(aerial.shape)
    n = math.prod(shape)
    nx = shape[-1] if shape else 1
    mp = [prnu, dcnu]
    views = []
    for m in mp:
        views.append(None if m is None else rows_view(m, shape))
    lut_t = None if lut is None else lut.contiguous()
    odt = code_dtype if lut_t is None else lut_t.dtype
    out = torch.empty((frames, *shape), dtype=odt, device=aerial.device)
    flags = torch.zeros(2, dtype=torch.int32, device=aerial.device)
    if n == 0:
        return out, [0, 0]
    pp, pr, pc = views[0] or (None, 0, 0)
    dp, dr, dc = views[1] or (None, 0, 0)
    prm, prmp = _darr(params)
    _call(lib.pb_expose, aerial, _CODE[aerial.dtype], _p(aerial), n, nx, _p(pp), pr, pc, _p(dp), dr, dc, prmp,
          int(frames), int(key), _CODE_BYTES[code_dtype], _p(lut_t), 0 if lut_t is None else lut_t.numel(),
          odt.itemsize, _p(out), _p(flags))
    return out, _flags_read(flags, 2 if lut_t is not None else 1)


def apply_lut(codes, lut, check):
    """np.take(lut, codes) for unsigned codes (pb_apply_lut); returns (out, largest out-of-range code or None)."""
    codes = codes.contiguous()
    lut = lut.contiguous()
    out = torch.empty(codes.shape, dtype=lut.dtype, device=codes.device)
    flags = torch.zeros(2, dtype=torch.int32, device=codes.device) if check else None
    _call(lib.pb_apply_lut, codes, _CODE_BYTES[codes.dtype], _p(codes), codes.numel(), _p(lut), lut.numel(),
          lut.dtype.itemsize, int(bool(check)), _p(out), _p(flags))
    if check and codes.numel():
        f = _flags_read(flags, 2)
        if f[0] & 4:
            return out, f[1]
    return out, None


def pixel(x, y, wx, wy):
    """(x <= wx) & (x >= -wx) & (y <= wy) & (y >= -wy) as a bool tensor of the broadcast shape (pb_pixel)."""
    shape = tuple(torch.broadcast_shapes(x.shape, y.shape))
    xv, xr, xc = rows_view(x, shape)
    yv, yr, yc = rows_view(y, shape)
    out = torch.empty(shape, dtype=torch.uint8, device=x.device)
    n = math.prod(shape)
    if n:
        _call(lib.pb_pixel, x, _CODE[x.dtype], _p(xv), xr, xc, _p(yv), yr, yc, n, shape[-1] if shape else 1, float(wx),
              float(wy), _p(out))
    return out.view(torch.bool)


def bayer_interleave(planes, half, out):
    """out[site s] = planes[s] at (y, x), or at (y / 2, x / 2) with half (pb_bayer_interleave); planes are 2-D tensors
    of out's dtype with unit column stride (or None for a site the output does not have)."""
    M, N = out.shape
    ptrs = (C.c_void_p * 4)(*[None if p is None else p.data_ptr() for p in planes])
    lds = (C.c_longlong * 4)(*[0 if p is None else p.stride(0) for p in planes])
    _call(lib.pb_bayer_interleave, out, out.element_size(), ptrs, lds, int(half), M, N, _p(out), out.stride(0))
    return out


def demosaic_deinterlace(img, bggr, out_dtype):
    m, n = img.shape
    out = torch.empty((m // 2, n // 2, 3), dtype=out_dtype, device=img.device)
    _call(lib.pb_demosaic_deinterlace, img, _ELEM[img.dtype], _p(img), m, n, img.stride(0), int(bggr),
          _ELEM[out_dtype], _p(out))
    return out


def white_balance(a, kind, gains, sat=None):
    """a *= gain in place (pb_white_balance): per CFA site (kind 0, a 2-D mosaic) or per channel (kind 1, (..., 3));
    with `sat` the gains are first descaled on the device so that no plane exceeds its saturation."""
    g, gp = _darr(gains)
    s, sp = (None, None) if sat is None else _darr(sat)
    _call(lib.pb_white_balance, a, _CODE[a.dtype], _p(a), a.numel(), a.shape[-1] if kind == 0 else 3, int(kind), gp, sp)
    return a


def demosaic_malvar(img, bggr, out_dtype):
    m, n = img.shape
    out = torch.empty((m, n, 3), dtype=out_dtype, device=img.device)
    _call(lib.pb_demosaic_malvar, img, _ELEM[img.dtype], _p(img), m, n, img.stride(0), int(bggr),
          _ELEM[out_dtype], _p(out))
    return out


def bayer_assemble(rp, g2p, bp, g1, out):
    _call(lib.pb_bayer_assemble, g1, _CODE[g1.dtype], _p(rp), _p(g2p), _p(bp), _p(g1), g1.numel(), _p(out))
    return out


def lenslet_screen(x, y, centres, cand, kind, params, two_efl, kphase, ncols, nrows):
    """The complex Shack-Hartmann screen of x's precision in one launch (pb_lenslet_screen); centres (fp64) and cand
    (int32) are the device tables shack_hartmann builds."""
    H, W = x.shape
    out = torch.empty((H, W), dtype=_CPLX_OF[x.dtype], device=x.device)
    prm, prmp = _darr(params)
    _call(lib.pb_lenslet_screen, x, _CODE[x.dtype], _p(x), _p(y), H, W, int(ncols), int(nrows), _p(centres), _p(cand),
          int(kind), prmp, float(two_efl), float(kphase), _p(out))
    return out


def subaperture_centroids(frames, dtab, itab, ncols, nrows, threshold, scale=1.0):
    """(disp (F, 2, nrows, ncols) times scale, flux (F, nrows, ncols)) of an (F, H, W) stack in one launch
    (pb_subaperture_centroids); float64 for float64 frames, float32 otherwise."""
    if frames.dtype not in (torch.float32, torch.float64, torch.uint16, torch.int32):
        raise ValueError(f'frames of {frames.dtype} are not supported (float32, float64, uint16, int32)')
    frames = frames.contiguous()
    F, H, W = frames.shape
    odt = torch.float64 if frames.dtype == torch.float64 else torch.float32
    disp = torch.empty((F, 2, nrows, ncols), dtype=odt, device=frames.device)
    flux = torch.empty((F, nrows, ncols), dtype=odt, device=frames.device)
    _call(lib.pb_subaperture_centroids, frames, _ELEM[frames.dtype], _p(frames), F, H, W, H * W, int(ncols),
          int(nrows), _p(dtab), _p(itab), float(threshold), float(scale), _ELEM[odt], _p(disp), _p(flux))
    return disp, flux


def sh_reconstruct(slopes, idx, ref, R, frame_shape):
    """out[f, k] = sum_m R[k, m] (slopes[f].flat[idx[m]] - ref[m]) for an (F, *frame_shape) slope stack
    (pb_sh_reconstruct).  idx is a device gather table the kernel cannot bound-check, so the stack's shape is checked
    here against the frame_shape the table was built for."""
    if not isinstance(slopes, torch.Tensor) or slopes.dtype not in (torch.float32, torch.float64):
        raise ValueError(f'slopes must be a float32 or float64 tensor, got {getattr(slopes, "dtype", type(slopes))}')
    if slopes.ndim != 1 + len(frame_shape) or tuple(slopes.shape[1:]) != tuple(frame_shape):
        raise ValueError(f'slopes must be (F, {", ".join(map(str, frame_shape))}), got {tuple(slopes.shape)}')
    slopes = slopes.contiguous()
    F = slopes.shape[0]
    K, M = R.shape
    out = torch.empty((F, K), dtype=slopes.dtype, device=slopes.device)
    _call(lib.pb_sh_reconstruct, slopes, _ELEM[slopes.dtype], _p(slopes), F, math.prod(frame_shape), _p(idx),
          _p(ref), _p(R), K, M, _p(out))
    return out


def qpoly_seq(family, kind, ns, ms, a, b=None):
    """Forbes basis planes (len(ns), *a.shape) of a's dtype in one launch (pb_qpoly_seq): values, or d/dx of Q-bfs /
    Q-con, or (d/dr, d/dt) / (d/dx, d/dy) of 2D-Q as a pair.  ms is None for Q-bfs / Q-con."""
    a = a.contiguous()
    if b is not None:
        b = b.to(a.dtype).contiguous()
    k = len(ns)
    pair = family == capi.QPOLY_2D and kind != capi.QPOLY_VALUE
    out0 = torch.empty((k,) + tuple(a.shape), dtype=a.dtype, device=a.device)
    out1 = torch.empty_like(out0) if pair else None
    if k == 0:
        return (out0, out1) if pair else out0
    n, nptr = _iarr(ns)
    m, mptr = _iarr(ms) if ms is not None else (None, C.POINTER(C.c_int)())
    _call(lib.pb_qpoly_seq, a, _CODE[a.dtype], int(family), int(kind), _p(a), _p(b), a.numel(), k, nptr, mptr, _p(out0),
          _p(out1))
    return (out0, out1) if pair else out0


def qpoly_sum(family, ns, ms, coefs, u, t=None, want_der=False):
    """The Forbes sag z (and with want_der dz/du, plus dz/dt for 2D-Q) of coefficient list (ns, ms, coefs) in one
    launch (pb_qpoly_sum)."""
    u = u.contiguous()
    if t is not None:
        t = t.to(u.dtype).contiguous()
    z = torch.empty_like(u)
    dr = torch.empty_like(u) if want_der else None
    dt = torch.empty_like(u) if want_der and family == capi.QPOLY_2D else None
    k = len(ns)
    n, nptr = _iarr(ns)
    m, mptr = _iarr([] if ms is None else ms)      # read for 2D-Q only
    c, cptr = _darr(coefs)
    _call(lib.pb_qpoly_sum, u, _CODE[u.dtype], int(family), _p(u), _p(t), u.numel(), k, nptr, mptr, cptr, _p(z), _p(dr),
          _p(dt))
    return z, dr, dt


def qpoly_tables(family, m, nmax):
    """(nmax + 1, 7) fp64 recurrence tables from the host C++ the kernels are planned with (pb_qpoly_tables)."""
    out, op = _darr(np.zeros((nmax + 1, 7)))
    rc = lib.pb_qpoly_tables(int(family), int(m), int(nmax), op)
    if rc != 0:
        raise ValueError(f'pb_qpoly_tables(family={family}, m={m}, nmax={nmax}) failed with status {rc}')
    return out


def poly_seq(family, kind, ns, x, alpha=0.0, beta=0.0):
    """1-D family planes of x's dtype in one launch (pb_poly_seq): (len(ns), *x.shape) of values (POLY_VALUE) or
    derivatives (POLY_DER), or with POLY_VALUE_DER the pair (values, derivatives).  An empty ns launches nothing."""
    x = x.contiguous()
    k = len(ns)
    both = kind == capi.POLY_VALUE_DER
    out = torch.empty(((2 if both else 1) * k,) + tuple(x.shape), dtype=x.dtype, device=x.device)
    if k:
        n, nptr = _iarr(ns)
        _call(lib.pb_poly_seq, x, _CODE[x.dtype], int(family), int(kind), float(alpha), float(beta), _p(x), x.numel(),
              k, nptr, _p(out))
    return (out[:k], out[k:]) if both else out


def jacobi_radial_sum(coefs, ns, alpha, beta, x, y, radius, want_der):
    """z (and dz/dx, dz/dy) of sum_q coefs[q] P_{ns[q]}(2 (x^2 + y^2) / R^2 - 1) in one launch (pb_jacobi_radial_sum)."""
    x = x.contiguous()
    y = y.to(x.dtype).contiguous()
    z = torch.empty_like(x)
    dx = torch.empty_like(x) if want_der else None
    dy = torch.empty_like(x) if want_der else None
    k = len(ns)
    n, nptr = _iarr(ns)
    c, cptr = _darr(coefs)
    _call(lib.pb_jacobi_radial_sum, x, _CODE[x.dtype], float(alpha), float(beta), _p(x), _p(y), x.numel(), k, nptr,
          cptr, float(radius), _p(z), _p(dx), _p(dy))
    return z, dx, dy


def jacobi_clenshaw(s, alpha, beta, x, j, table, out=None):
    """Clenshaw's alphas for sum_n s[n] P_n^(alpha,beta)(x) in one launch (pb_jacobi_clenshaw): with table the whole
    (j + 1, max(len(s), 2), *x.shape) table (into `out` when given), otherwise the sum alone."""
    x = x.contiguous()
    N = max(len(s), 2)
    shape = ((j + 1, N) + tuple(x.shape)) if table else tuple(x.shape)
    out = _out(out, shape, x.dtype, x.device)
    c, cptr = _darr(s)
    _call(lib.pb_jacobi_clenshaw, x, _CODE[x.dtype], float(alpha), float(beta), _p(x), x.numel(), len(s), cptr, int(j),
          int(bool(table)), _p(out))
    return out


def zernike_der(nms, a, b, norm, cartesian):
    """(k, 2, *a.shape): (dZ/dr, dZ/dt) of (r, t), or (dZ/dx, dZ/dy) of (x, y) (pb_zernike_der)."""
    a = a.contiguous()
    b = b.to(a.dtype).contiguous()
    k = len(nms)
    out = torch.empty((k, 2) + tuple(a.shape), dtype=a.dtype, device=a.device)
    if k == 0:
        return out
    (n, nptr), (m, mptr) = _nm(nms)
    _call(lib.pb_zernike_der, a, _CODE[a.dtype], int(bool(cartesian)), _p(a), _p(b), a.numel(), k, nptr, mptr,
          int(bool(norm)), _p(out))
    return out


def zernike_sum_der_xy(coefs, nms, x, y, norm):
    """(3, *x.shape): W, dW/dx, dW/dy of sum coefs[q] Z_q(x, y) (pb_zernike_sum_der_xy)."""
    x = x.contiguous()
    y = y.to(x.dtype).contiguous()
    k = len(nms)
    out = torch.empty((3,) + tuple(x.shape), dtype=x.dtype, device=x.device)
    (n, nptr), (m, mptr) = _nm(nms)
    c, cptr = _darr(coefs)
    _call(lib.pb_zernike_sum_der_xy, x, _CODE[x.dtype], _p(x), _p(y), x.numel(), k, nptr, mptr, cptr, int(bool(norm)),
          _p(out))
    return out


def xy_seq(ms, ns, kinds, x, y, shape, separable):
    """XY-monomial planes (len(ms), *shape) (pb_xy_seq); separable: x is the row of nx = shape[-1] values and y the
    column, otherwise x and y hold one value per sample."""
    x = x.contiguous()
    y = y.to(x.dtype).contiguous()
    k = len(ms)
    out = torch.empty((k,) + tuple(shape), dtype=x.dtype, device=x.device)
    if k == 0:
        return out
    m, mptr = _iarr(ms)
    n, nptr = _iarr(ns)
    kd, kptr = _iarr(kinds)
    _call(lib.pb_xy_seq, x, _CODE[x.dtype], _p(x), _p(y), math.prod(shape), int(shape[-1]) if separable else 1,
          int(bool(separable)), k, mptr, nptr, kptr, _p(out))
    return out


def tensor_sum(basis, coefs, ms, ns, x, y, shape, separable, want_der, x_norm=1.0, y_norm=1.0):
    """z (and dz/dx / x_norm, dz/dy / y_norm) of sum coefs[q] P_{ms[q]}(x) P_{ns[q]}(y) in one launch (pb_tensor_sum)."""
    x = x.contiguous()
    y = y.to(x.dtype).contiguous()
    z = torch.empty(tuple(shape), dtype=x.dtype, device=x.device)
    dx = torch.empty_like(z) if want_der else None
    dy = torch.empty_like(z) if want_der else None
    k = len(ms)
    m, mptr = _iarr(ms)
    n, nptr = _iarr(ns)
    c, cptr = _darr(coefs)
    _call(lib.pb_tensor_sum, x, _CODE[x.dtype], int(basis), _p(x), _p(y), math.prod(shape),
          int(shape[-1]) if separable else 1, int(bool(separable)), k, mptr, nptr, cptr, float(x_norm), float(y_norm),
          _p(z), _p(dx), _p(dy))
    return z, dx, dy


def tf_layout(ops):
    """(broadcast calculation shape, collapsed shape, (len(ops), 5) int64 host strides) of the six thin-film operands
    (wavelength, angle, ambient index, substrate index, layer index, layer thickness: fp64 / complex128 device tensors,
    the last two with a leading layer axis) and of any operands after them (per sample only).  Dims that are contiguous in every operand are merged; a broadcast that
    still needs more than TF_DIMS dims is refused with ValueError."""
    calc = [tuple(t.shape[1:]) if q in (capi.TF_IN_N, capi.TF_IN_D) else tuple(t.shape) for q, t in enumerate(ops)]
    bshape = np.broadcast_shapes(*calc)
    nd = len(bshape)
    st = []
    for q, (t, c) in enumerate(zip(ops, calc)):
        tst = t.stride()[1:] if q in (capi.TF_IN_N, capi.TF_IN_D) else t.stride()
        pad = nd - len(c)
        st.append([0 if j < pad or c[j - pad] == 1 else tst[j - pad] for j in range(nd)])
    dims, cst = [], [[] for _ in ops]
    for j in range(nd):
        if bshape[j] == 1:
            continue
        if dims and all(s[-1] == st[q][j] * bshape[j] for q, s in enumerate(cst)):
            dims[-1] *= bshape[j]
            for q, s in enumerate(cst):
                s[-1] = st[q][j]
            continue
        dims.append(bshape[j])
        for q, s in enumerate(cst):
            s.append(st[q][j])
    if len(dims) > capi.TF_DIMS:
        raise ValueError(f'thin-film operands broadcast to {bshape}, which needs {len(dims)} dims after merging the '
                         f'contiguous ones; at most {capi.TF_DIMS} are supported')
    strides = np.zeros((len(ops), capi.TF_DIMS + 1), dtype=np.int64)
    for q, s in enumerate(cst):
        strides[q, :len(s)] = s
        if q in (capi.TF_IN_N, capi.TF_IN_D) and ops[q].shape[0] != 1:
            strides[q, capi.TF_DIMS] = ops[q].stride(0)
    return bshape, dims, strides


def tf_nlayers(ops):
    """layers of the thin-film operands: the index and thickness layer axes broadcast"""
    return max(int(ops[capi.TF_IN_N].shape[0]), int(ops[capi.TF_IN_D].shape[0])) \
        if min(ops[capi.TF_IN_N].shape[0], ops[capi.TF_IN_D].shape[0]) else 0


def _tf_args(ops):
    """(broadcast shape, ndim, shape, strides, operands) of the thin-film operands and any coating-design operands after
    them, as the C ABI takes them: host arrays of CM_NOPS operand slots, the slots past len(ops) NULL."""
    bshape, dims, strides = tf_layout(ops)
    shp = (C.c_longlong * max(len(dims), 1))(*(dims or [1]))
    st = (C.c_longlong * (capi.CM_NOPS * (capi.TF_DIMS + 1)))(*strides.ravel().tolist())
    ins = (C.c_void_p * capi.CM_NOPS)(*[t.data_ptr() for t in ops])
    return bshape, len(dims), shp, st, ins


def stack_eval(mode, pol, ops, outputs, rdtype, theta_scale=1.0):
    """{TF_OUT_* code: device array} for the codes in `outputs`, from one pb_stack_eval launch: r, t, eta0, eta_sub
    complex of the broadcast shape, E, H, Esq (N + 1, *shape), REFL, TRANS (shape), ABS (N, *shape), in rdtype's
    precision."""
    nlayers = tf_nlayers(ops)
    bshape, nd, shp, stp, inp = _tf_args(ops)
    cdtype = _CPLX_OF[rdtype]
    lead = {capi.TF_OUT_E: nlayers + 1, capi.TF_OUT_H: nlayers + 1, capi.TF_OUT_ESQ: nlayers + 1,
            capi.TF_OUT_ABS: nlayers}
    cplx = (capi.TF_OUT_R, capi.TF_OUT_T, capi.TF_OUT_E, capi.TF_OUT_H, capi.TF_OUT_ETA0, capi.TF_OUT_ETASUB)
    dev = ops[0].device
    res = {}
    for code in outputs:
        shape = ((lead[code],) if code in lead else ()) + tuple(bshape)
        res[code] = torch.empty(shape, dtype=cdtype if code in cplx else rdtype, device=dev)
    live = [q for q in res if res[q].numel()]        # an empty output (no layers, or no samples) is not written
    if not live:
        return res
    outs = (C.c_void_p * capi.TF_NOUT)(*[res[q].data_ptr() if q in live else None for q in range(capi.TF_NOUT)])
    flags = sum(1 << q for q in live)
    _call(lib.pb_stack_eval, ops[0], _CODE[rdtype], int(mode), int(pol), flags, nlayers, nd, shp, stp, inp,
          float(theta_scale), C.cast(outs, C.POINTER(C.c_void_p)))
    return res


def stack_grad(pol, kinds, ops, E, H, seeds, rdtype):
    """(N,) thickness or index gradient, or (2, N) both, summed over the samples (pb_stack_grad).  E, H: the complex128
    boundary fields of stack_eval; seeds: dR, dT, dA, dEsq as contiguous fp64 device arrays of the full shapes, or
    None."""
    nlayers = tf_nlayers(ops)
    bshape, nd, shp, stp, inp = _tf_args(ops)
    both = kinds == capi.TF_GRAD_THICKNESS | capi.TF_GRAD_INDEX
    grad = torch.empty(((2,) if both else ()) + (nlayers,), dtype=rdtype, device=E.device)
    if nlayers == 0:
        return grad
    sp = (C.c_void_p * 4)(*[None if s is None else s.data_ptr() for s in seeds])
    _call(lib.pb_stack_grad, E, _CODE[rdtype], int(pol), int(kinds), nlayers, nd, shp, stp, inp, _p(E), _p(H),
          C.cast(sp, C.POINTER(C.c_void_p)), _p(grad))
    return grad


def coating_merit(quantity, pol, flags, ops, b0=0, b1=0, blist=None, value=None, residuals=None, grad=None,
                  rdtype=torch.float64):
    """One merit term (pb_coating_merit) over ops = the six thin-film operands, target and weight: the fp64 value
    into `value` (a one-element device array), sqrt(w) (q - target) into `residuals` (count, rdtype) and the
    gradient into `grad` (rdtype), each as `flags` (CM_OUT_*, CM_ACCUMULATE) asks."""
    nlayers = tf_nlayers(ops)
    bshape, nd, shp, stp, inp = _tf_args(ops)
    nb = 0 if blist is None else blist.numel() // 2
    _call(lib.pb_coating_merit, ops[0], _CODE[rdtype], int(quantity), int(pol), int(flags), nlayers, nd, shp, stp, inp,
          int(b0), int(b1), _p(blist), nb, _p(value), _p(residuals), _p(grad))


def needle(quantity, pol, ops, zpart, zlist, P, accumulate):
    """P(z) of an R or T term (pb_needle): ops = the six thin-film operands, target, weight and the needle index;
    zpart (2, nz) fp64 partial thicknesses, zlist the per-layer depth runs (int32), P (nz) written or added to."""
    nlayers = tf_nlayers(ops)
    bshape, nd, shp, stp, inp = _tf_args(ops)
    _call(lib.pb_needle, ops[0], _CODE[P.dtype], int(quantity), int(pol), nlayers, nd, shp, stp, inp, _p(zpart),
          int(zpart.shape[1]), _p(zlist), _p(P), int(bool(accumulate)))


def monitor_runs(strategy, mode, pol, ops, runs, per_cand, err, levels, n_points, start, max_factor, turning_index,
                 rdtype):
    """(runs, N) as-built thicknesses in rdtype from one pb_monitor_runs launch: ops = wavelength, angle, ambient and
    substrate index (ncand each), layer indices (N, ncand) and nominal thicknesses (N), dense fp64 / complex128 device
    arrays; err (runs, N) and levels (ncand, N) fp64 or None."""
    nlayers = int(ops[capi.TF_IN_D].shape[0])
    out = torch.empty((runs, nlayers), dtype=rdtype, device=ops[0].device)
    ins = (C.c_void_p * capi.TF_NOPS)(*[t.data_ptr() for t in ops])
    _call(lib.pb_monitor_runs, ops[0], _CODE[rdtype], int(strategy), int(mode), int(pol), nlayers,
          int(ops[capi.TF_IN_WVL].numel()), ins, int(runs), int(per_cand), _p(err), _p(levels), int(n_points),
          float(start), float(max_factor), int(turning_index), _p(out))
    return out


def monitor_cut(strategy, d, sig, level=0.0, target=float('nan')):
    """level_cut (a one-element device array) or turning_points (a device array and a device int64 count) of a trace
    (pb_monitor_cut): d and sig of one real dtype."""
    d, sig = d.contiguous(), sig.contiguous()
    n = d.numel()
    out = torch.empty(max(n, 1), dtype=d.dtype, device=d.device)
    count = torch.zeros(1, dtype=torch.int64, device=d.device)
    _call(lib.pb_monitor_cut, d, _CODE[d.dtype], int(strategy), _p(d), _p(sig), n, float(level), float(target),
          _p(out), _p(count))
    return out, count


def monitor_jacobian(Rr, ncand, nlayers, eps, rdtype, want_J=True):
    """J (ncand, W, N) and score (ncand) in rdtype from the realized reflectance Rr (ncand (N + 1), W) fp64
    (pb_monitor_jacobian)."""
    nw = int(Rr.shape[1])
    J = torch.empty((ncand, nw, nlayers), dtype=rdtype, device=Rr.device) if want_J else None
    score = torch.empty(ncand, dtype=rdtype, device=Rr.device)
    _call(lib.pb_monitor_jacobian, Rr, _CODE[rdtype], int(ncand), int(nlayers), nw, _p(Rr), float(eps), _p(J),
          _p(score))
    return J, score


def field_at_depth(pol, z, zb, n, n0, wvl, theta0, Eb, Hb, cdtype):
    """E, H (complex, like z) at depths z inside a stack (pb_field_at_depth): z, zb fp64, n, Eb, Hb complex128."""
    z = z.contiguous()
    E = torch.empty(z.shape, dtype=cdtype, device=z.device)
    H = torch.empty_like(E)
    n0 = complex(n0)
    _call(lib.pb_field_at_depth, z, _CODE[cdtype], int(pol), int(n.shape[0]), _p(z), z.numel(), _p(zb), _p(n),
          n0.real, n0.imag, float(wvl), float(theta0), _p(Eb), _p(Hb), _p(E), _p(H))
    return E, H


def _analysis_data(data, types):
    """data as a dense 2-D tensor of one of `types`; anything else is refused before any launch"""
    if not isinstance(data, torch.Tensor) or data.ndim != 2:
        raise ValueError(f'data must be a 2-D CUDA tensor, got {getattr(data, "shape", type(data))}')
    if data.dtype not in types:
        raise ValueError(f'data of {data.dtype} is not supported ({", ".join(str(t) for t in types)})')
    return data.contiguous()


def interp2d_linear(data, xax, yax, px=None, py=None, rmax=None, fill=0.0, ld=None):
    """Linear interpolation of (ny, nx) data on the fp64 axes xax, yax (pb_interp2d_linear): at the fp64 points (px, py)
    -- out has px's shape -- or, with rmax, on the (ny, nx) polar lattice of uniform_cart_to_polar.  `ld` is the row
    pitch of a strided data view (one row or column of a larger array)."""
    if ld is None:
        data = _analysis_data(data, (torch.float32, torch.float64, torch.complex64, torch.complex128))
        ld = data.shape[1]
    ny, nx = data.shape
    if rmax is not None:
        out = torch.empty((ny, nx), dtype=data.dtype, device=data.device)
        _call(lib.pb_interp2d_linear, data, _ELEM[data.dtype], _p(data), ny, nx, ld, _p(xax), _p(yax),
              capi.INTERP_POLAR, None, None, 0, float(rmax), 0.0, _p(out))
        return out
    shape = px.shape
    px, py = px.reshape(-1).contiguous(), py.reshape(-1).contiguous()
    out = torch.empty(shape, dtype=data.dtype, device=data.device)
    _call(lib.pb_interp2d_linear, data, _ELEM[data.dtype], _p(data), ny, nx, ld, _p(xax), _p(yax), capi.INTERP_POINTS,
          _p(px), _p(py), px.numel(), 0.0, float(fill), _p(out))
    return out


def azimuthal_stats(data, xax, yax, rmax, stats):
    """(6, nx) of data's dtype: rows count, mean, var, min, max, median over phi of each rho column of the polar lattice,
    the rows `stats` (a mask of AZ_*) asks for filled, in one launch (pb_azimuthal_stats)."""
    data = _analysis_data(data, (torch.float32, torch.float64))
    ny, nx = data.shape
    if ny > capi.AZ_MAX_NY:
        raise ValueError(f'azimuthal statistics hold a column on chip: at most {capi.AZ_MAX_NY} phi samples (rows), '
                         f'got {ny}')
    out = torch.full((6, nx), float('nan'), dtype=data.dtype, device=data.device)
    _call(lib.pb_azimuthal_stats, data, _ELEM[data.dtype], _p(data), ny, nx, _p(xax), _p(yax), float(rmax), int(stats),
          _p(out))
    return out


def polar_crossings(data, xax, yax, rmax, metric, relative, last):
    """(rows that cross, mean crossing radius) of estimate_size on the polar lattice (pb_polar_crossings); the call
    waits for the device."""
    data = _analysis_data(data, (torch.float32, torch.float64))
    ny, nx = data.shape
    res = (C.c_double * 2)()
    _call(lib.pb_polar_crossings, data, _ELEM[data.dtype], _p(data), ny, nx, _p(xax), _p(yax), float(rmax),
          float(metric), int(bool(relative)), int(bool(last)), res)
    return int(res[0]), res[1]


def analytic_radial(kind, x, a, b, out_dtype):
    """f(x) of one AR_* kind elementwise in fp64, stored as out_dtype (pb_analytic_radial); a = wavelength, b = F/#."""
    if x.dtype not in (torch.float32, torch.float64):
        x = x.to(torch.float64)
    x = x.contiguous()
    out = torch.empty(x.shape, dtype=out_dtype, device=x.device)
    _call(lib.pb_analytic_radial, x, _ELEM[x.dtype], _ELEM[out_dtype], int(kind), _p(x), x.numel(), float(a), float(b),
          _p(out))
    return out


# ---- interferometric metrology (pb_nan_stats ... pb_metro_pointwise) --------------------------------------------------
def metro_data(data):
    """data as a dense real CUDA tensor the metrology entry points take (fp32 / fp64; anything else is refused)"""
    if not isinstance(data, torch.Tensor) or not data.is_cuda:
        raise ValueError('metrology data must be a CUDA tensor')
    if data.dtype not in (torch.float32, torch.float64):
        raise ValueError(f'metrology data of {data.dtype} is not supported (torch.float32, torch.float64)')
    return data.contiguous()


def nan_stats(x):
    """(9,) fp64 host array: finite count, sum, min, max, sum of squares, NaN count, mean, sum |x - mean|,
    sum (x - mean)^2 over the finite values of x (pb_nan_stats: two launches, one copy to the host)."""
    x = metro_data(x)
    res = torch.empty(9, dtype=torch.float64, device=x.device)
    _call(lib.pb_nan_stats, x, _CODE[x.dtype], _p(x), x.numel(), _p(res))
    return res.cpu().numpy()


def masked_gram(modes, data):
    """The packed upper triangle of [A d]^T [A d] over the finite pixels of data (pb_masked_gram), as a host fp64
    array; modes is a sequence of tensors shaped like data (dtype data's), None for the constant 1."""
    data = metro_data(data)
    k = len(modes)
    if not 1 <= k <= capi.GRAM_MAX_K:
        raise ValueError(f'a masked least-squares fit takes 1 to {capi.GRAM_MAX_K} modes, got {k}')
    keep = [None if m is None else m.to(data.dtype).contiguous() for m in modes]
    for m in keep:
        if m is not None and m.numel() != data.numel():
            raise ValueError(f'mode of {m.numel()} samples against data of {data.numel()}')
    ptrs = (C.c_void_p * k)(*[None if m is None else m.data_ptr() for m in keep])
    out = torch.empty((k + 1) * (k + 2) // 2, dtype=torch.float64, device=data.device)
    _call(lib.pb_masked_gram, data, _CODE[data.dtype], C.cast(ptrs, C.POINTER(C.c_void_p)), k, _p(data), data.numel(),
          _p(out))
    return out.cpu().numpy()


def _same_shape(name, t, shape):
    """refuse an operand the kernel would index densely over `shape` but which has another shape"""
    if t is not None and tuple(t.shape) != tuple(shape):
        raise ValueError(f'{name} of shape {tuple(t.shape)} does not match the data shape {tuple(shape)}')


def psd_prologue(height, kind, user=None, dx=1.0, alpha=4.0, rmax=1.0, corners=None, want_shifted=True,
                 want_window=False, shape=None, dtype=None):
    """(shifted, window, s2) of pb_psd_prologue: fftshift(height * w) and / or w (None where not asked for), and the
    device fp64 scalar sum w^2.  A user window must have height's shape."""
    like = height if height is not None else user
    if height is not None:
        _same_shape('window', user, height.shape)
        height = metro_data(height)
        shape, dtype = height.shape, height.dtype
    ny, nx = shape
    dev = device() if like is None else like.device
    if user is not None:
        user = user.to(dtype).contiguous()
    shifted = torch.empty((ny, nx), dtype=dtype, device=dev) if want_shifted else None
    window = torch.empty((ny, nx), dtype=dtype, device=dev) if want_window else None
    s2 = torch.empty(1, dtype=torch.float64, device=dev)
    flags = torch.empty(4, dtype=torch.int32, device=dev)
    cor, cp = _iarr(np.zeros(16) if corners is None else corners)
    _call(lib.pb_psd_prologue, s2, _CODE[dtype], _p(height), ny, nx, int(kind), _p(user), float(dx), float(alpha),
          float(rmax), cp if corners is not None else None, _p(shifted), _p(window), _p(s2), _p(flags))
    return shifted, window, s2


def psd_epilogue(F, s2, fs):
    """ifftshift(|F|^2) / (s2 fs^2) (pb_psd_epilogue) of the complex transform F."""
    ny, nx = F.shape
    out = torch.empty((ny, nx), dtype=_REAL_OF[F.dtype], device=F.device)
    _call(lib.pb_psd_epilogue, F, _CODE[F.dtype], _p(F), ny, nx, _p(s2), float(fs), _p(out))
    return out


def band_trapz(psd, r=None, fx=None, fy=None, flow=0.0, fhigh=np.inf):
    """sum w_i w_j psd over flow <= r <= fhigh with trapezoid edge weights (pb_band_trapz), a host float; r is an
    array like psd or None for hypot of the fp64 axes fx, fy.  1-D psd: one trapezoid."""
    _same_shape('r', r, psd.shape)
    psd = metro_data(psd)
    twod = psd.ndim == 2
    if twod and r is None and (fx.numel() != psd.shape[1] or fy.numel() != psd.shape[0]):
        raise ValueError(f'frequency axes of {fx.numel()} and {fy.numel()} samples for a PSD of shape {tuple(psd.shape)}')
    ny, nx = psd.shape if twod else (psd.numel(), 1)
    if r is not None:
        r = r.to(psd.dtype).contiguous()
    res = torch.empty(1, dtype=torch.float64, device=psd.device)
    _call(lib.pb_band_trapz, psd, _CODE[psd.dtype], _p(psd), _p(r), _p(fx), _p(fy), ny, nx, int(twod), float(flow),
          float(fhigh), _p(res))
    return float(res.cpu()[0])


def filter_h(shape, parts, dtype, dev, r=None, dx=1.0, fcn0=0.0, fcn1=None):
    """hann2d (FILT_W), ideal_lpf_iir2d (FILT_H) or their product over shape (pb_filter_h); with fcn1 a second array
    at that cut-off from the same launch."""
    ny, nx = shape
    _same_shape('r', r, shape)
    if r is not None:
        r = r.to(dtype).contiguous()
    out0 = torch.empty((ny, nx), dtype=dtype, device=dev)
    out1 = torch.empty((ny, nx), dtype=dtype, device=dev) if fcn1 is not None else None
    _call(lib.pb_filter_h, out0, _CODE[dtype], _p(r), ny, nx, int(parts), float(dx), float(fcn0),
          float(0.0 if fcn1 is None else fcn1), _p(out0), _p(out1))
    return out0, out1


def filter_apply(typ, Hl, Hh=None, D=None):
    """D *= H in place (returns D), or with D None the real H (pb_filter_apply)."""
    for t in (Hh, D):
        if t is not None and (t.dtype != Hl.dtype or t.shape != Hl.shape):
            raise ValueError(f'filter transforms of {t.dtype} {tuple(t.shape)} and {Hl.dtype} {tuple(Hl.shape)} differ')
    Hout = None if D is not None else torch.empty(Hl.shape, dtype=_REAL_OF[Hl.dtype], device=Hl.device)
    _call(lib.pb_filter_apply, Hl, _CODE[Hl.dtype], _p(D), _p(Hl), _p(Hh), Hl.numel(), int(typ), _p(Hout))
    return D if D is not None else Hout


def gradient2d(f, dx):
    """(gx, gy, hypot(gx, gy)) of np.gradient(f, dx) (pb_gradient2d)."""
    f = metro_data(f)
    ny, nx = f.shape
    if ny < 2 or nx < 2:
        raise ValueError('Shape of array too small to calculate a numerical gradient, at least (edge_order + 1) '
                         'elements are required.')
    gx, gy, gr = (torch.empty_like(f) for _ in range(3))
    _call(lib.pb_gradient2d, f, _CODE[f.dtype], _p(f), ny, nx, float(dx), _p(gx), _p(gy), _p(gr))
    return gx, gy, gr


def finite_bounds(x):
    """(first finite row, rows after the last finite one, first finite column, columns after the last finite one);
    all zero without a finite sample (pb_finite_bounds, one launch, the call waits)."""
    x = metro_data(x)
    ny, nx = x.shape
    box = (C.c_int * 4)()
    _call(lib.pb_finite_bounds, x, _CODE[x.dtype], _p(x), ny, nx, box)
    if box[0] == 0:
        return 0, 0, 0, 0
    return ny - box[0], ny - box[1], nx - box[2], nx - box[3]


def metro_pointwise(op, x=None, u=None, v=None, m=None, a=0.0, b=0.0, out=None, shape=None, dtype=None):
    """One PW_* op of pb_metro_pointwise; out may be x (in place).  u, v are cast to the output's dtype."""
    like = x if x is not None else u
    if dtype is None:
        dtype = _REAL_OF.get(like.dtype, like.dtype) if like is not None else None
    if shape is None:
        shape = like.shape
    dev = like.device if like is not None else device()
    n = int(np.prod(shape))
    for name, t, want in (('data', x, 2 * n if op == capi.PW_REAL else n), ('u', u, n), ('v', v, n), ('mask', m, n)):
        if t is not None and t.numel() != want:
            raise ValueError(f'{name} of {t.numel()} elements for an operation over {want} (shape {tuple(shape)})')
    if x is not None:
        x = x.contiguous()
    u = None if u is None else u.to(dtype).contiguous()
    v = None if v is None else v.to(dtype).contiguous()
    if m is not None:
        m = m.contiguous()
        m = m.view(torch.uint8) if m.dtype == torch.bool else m.to(torch.uint8)
    out = _out(out, tuple(shape), dtype, dev)
    ny, nx = (shape[0], shape[1]) if len(shape) == 2 else (1, int(np.prod(shape)))
    _call(lib.pb_metro_pointwise, out, _CODE[dtype], int(op), _p(x), _p(u), _p(v), _p(m), ny, nx, float(a), float(b),
          _p(out))
    return out


def launch_count(dev=None):
    dev = device() if dev is None else torch.device(dev)
    return capi.launch_count(dev.index)


def ceil_half(d):
    return math.ceil(d / 2)
