"""Fourier tools on the H100 engine -- same names and semantics as prysm.fttools
(reference prysm/fttools.py), arrays are CUDA tensors, every transform is a libprysm_b200 call.

Executors (MDFT / CZT / FFTDFT) keep the reference constructor `(x, y, fx, fy, sign, norm)`,
`__call__`, `.adjoint` and `.nbytes()`; holding an instance is the caching mechanism
(prysm/fttools.py:181-183).  Coordinates are taken on the host in fp64 and every basis /
chirp argument is range-reduced in fp64 before the sincos, so the complex64 executors track
the reference's *fp64* output (the reference's own fp32 chirps are only good to ~1e-4 at
2048^2, BASELINE.md section 3).
"""
import math

import numpy as np
import torch

from . import _ops
from ._capi import OUT_INTENSITY, OUT_ACCUMULATE
from ._capi import OP_N, OP_T, OP_H, OP_C  # noqa: F401
from .conf import config


def _host(v):
    """1-D coordinate vector -> host float64."""
    if isinstance(v, torch.Tensor):
        v = v.detach().cpu().numpy()
    return np.asarray(v, dtype=np.float64)


def fftrange(n, dtype=None):
    """FFT-aligned integer grid, zero at index n//2 (prysm/fttools.py:13-15).  Device tensor."""
    dt = config.real_dtype if dtype is None else _ops.torch_dtype(dtype)
    return torch.arange(-(n // 2), -(n // 2) + n, dtype=dt, device=_ops.device())


def next_fast_len(n):
    """Next transform length the radix kernels run natively: a power of two
    (the reference asks its FFT backend, prysm/fttools.py:23-31; any K >= N+M-1 is valid for CZT)."""
    return 1 << max(0, math.ceil(math.log2(n)))


def fftfreq(n, d=1.0):
    """DFT sample frequencies, numpy ordering, at config.precision (prysm/fttools.py:34-40)."""
    return _ops.asdevice(np.fft.fftfreq(n, d).astype(config.precision))


def forward_ft_unit(dx, samples, shift=True):
    """prysm/fttools.py:128-152."""
    u = np.fft.fftfreq(samples, dx).astype(config.precision)
    return _ops.asdevice(np.fft.fftshift(u) if shift else u)


def pad2d(array, Q=2, value=0, mode='constant', out_shape=None):
    """Centred pad; offsets ceil((out-in)/2) (prysm/fttools.py:43-100).  Q == 1 returns the input."""
    if Q == 1 and out_shape is None:
        return array
    if mode != 'constant':
        raise NotImplementedError("only mode='constant' is on the propagation path")
    array = _ops.asdevice(array)
    in_shape = tuple(array.shape)
    if out_shape is None:
        out_shape = [math.ceil(s * Q) for s in in_shape]
    elif isinstance(out_shape, int):
        out_shape = [out_shape] * array.ndim
    offs = [math.ceil((o - i) / 2) for o, i in zip(out_shape, in_shape)]
    if value != 0:
        out = torch.full(tuple(out_shape), value, dtype=array.dtype, device=array.device)
    else:
        out = torch.zeros(tuple(out_shape), dtype=array.dtype, device=array.device)
    view = out[offs[0]:offs[0] + in_shape[0], offs[1]:offs[1] + in_shape[1]]
    if array.is_complex():
        _ops.mul_outer(array, out=view)
    else:
        view.copy_(array)
    return out


def crop_center(img, out_shape):
    """Centred window starting at ceil((in-out)/2): a view (prysm/fttools.py:103-125)."""
    if isinstance(out_shape, int):
        out_shape = (out_shape, out_shape)
    left = [math.ceil((i - o) / 2) for i, o in zip(img.shape, out_shape)]
    return img[left[0]:left[0] + out_shape[0], left[1]:left[1] + out_shape[1]]


def _prep(ary, cdtype):
    ary = _ops.asdevice(ary)
    if ary.dtype != cdtype:
        ary = ary.to(cdtype)
    return ary


class MDFT:
    """Matrix DFT: out = norm * Ey @ ary @ Ex.T with Ex = exp(sign*2*pi*i*outer(fx, x))
    (prysm/fttools.py:155-232).  complex64 runs on the wgmma tensor cores when the shape
    allows, otherwise (and always for complex128) on the fp32 / fp64 CUDA-core GEMM."""

    def __init__(self, x, y, fx, fy, sign=-1, norm=1.0, use_tensor_cores=True):
        x, y, fx, fy = _host(x), _host(y), _host(fx), _host(fy)
        cd = config.complex_dtype
        dev = _ops.device()
        self.Ex = _ops.mdft_basis(fx, x, sign, cd, dev)  # (len(fx), len(x))
        self.Ey = _ops.mdft_basis(fy, y, sign, cd, dev)  # (len(fy), len(y))
        self.norm = norm
        Nx, Ny, Mx, My = len(x), len(y), len(fx), len(fy)
        self._forward_left_first = My * Nx * (Ny + Mx) <= Ny * Mx * (Nx + My)
        self._adjoint_left_first = Ny * Mx * (My + Nx) <= My * Nx * (Mx + Ny)
        # tensor-core plan: TF32-split real expansions of both bases, built once (4x the basis bytes)
        self._tc = None
        if cd == torch.complex64 and use_tensor_cores and _ops.mdft_tc_supported(My, Ny, Mx, Nx):
            self._tc = _ops.mdft_tc_expand(self.Ex) + _ops.mdft_tc_expand(self.Ey)
        # the adjoint Ey^H @ g @ conj(Ex) is the same two-GEMM form with the bases Ey^H = basis(y, fy, -sign)
        # and Ex^H, so it runs on the tensor cores too when the swapped shape allows
        self._tc_adj = None
        if cd == torch.complex64 and use_tensor_cores and _ops.mdft_tc_supported(Ny, My, Nx, Mx):
            self._tc_adj = (_ops.mdft_tc_expand(_ops.mdft_basis(x, fx, -sign, cd, dev))
                            + _ops.mdft_tc_expand(_ops.mdft_basis(y, fy, -sign, cd, dev)))

    def __call__(self, ary):
        return self._forward(ary)

    def adjoint(self, grad):
        return self._adjoint(grad)

    # _forward / _adjoint write into a given contiguous `out` (one plane of a stack, prysm_b200.polarization)
    def _forward(self, ary, out=None):
        ary = _prep(ary, self.Ey.dtype)
        if self._tc is not None:
            return _ops.mdft_tc_apply(*self._tc, ary, self.norm, out=out)
        return _ops.mdft_apply(self.Ey, self.Ex, ary, self.norm, False, self._forward_left_first, out=out)

    def _adjoint(self, grad, out=None):
        grad = _prep(grad, self.Ey.dtype)
        if self._tc_adj is not None:
            return _ops.mdft_tc_apply(*self._tc_adj, grad, self.norm, out=out)
        return _ops.mdft_apply(self.Ey, self.Ex, grad, self.norm, True, self._adjoint_left_first, out=out)

    def _out_shape(self, adjoint):
        return (self.Ey.shape[1], self.Ex.shape[1]) if adjoint else (self.Ey.shape[0], self.Ex.shape[0])

    @property
    def _dtype(self):
        return self.Ey.dtype

    def nbytes(self):
        return self.Ex.numel() * self.Ex.element_size() + self.Ey.numel() * self.Ey.element_size()


def _expi(turns):
    """exp(2*pi*i*turns) for a host fp64 vector with the argument reduced first."""
    fr = turns - np.rint(turns)
    return np.exp(2j * np.pi * fr)


_ENGINE_MAX_K = 4096     # longest Bluestein length the register-resident axis engine runs (csrc/fft_tuned.cu)


class _CztAxis:
    """Per-axis Bluestein pieces (prysm/fttools.py:372-389), built in fp64 on the host."""

    def __init__(self, N, M, shift, alpha, sign, xc, f):
        K = next_fast_len(N + M - 1)
        n = np.arange(-(N // 2), -(N // 2) + N, dtype=np.float64)
        m = np.arange(-(M // 2), -(M // 2) + M, dtype=np.float64)
        q = m + shift
        half = 0.5 * sign * alpha                       # exp(sign*i*pi*alpha*t^2) = expi(half*t^2)
        a = _expi(half * q * q)
        b = _expi(half * n * n)
        d = np.arange(m[0] - n[-1], m[-1] - n[0] + 1, dtype=np.float64)
        h = np.zeros(K, dtype=np.complex128)
        h[:len(d)] = _expi(-half * (d + shift) * (d + shift))
        H = np.fft.fft(h)
        phase = _expi(sign * xc * f)                    # exp(sign*2*pi*i*x[N//2]*f)
        k = np.arange(K, dtype=np.float64)
        self.N, self.M, self.K = N, M, K
        self.b = b                                      # applied before the forward FFT
        self.H = H                                      # kernel spectrum
        self.post = a * phase                           # applied to the M kept samples
        # adjoint: embedding at offset N-1 is a linear phase on the spectrum
        self.Hadj = np.conj(H) * _expi(-(N - 1) * k / K)


def czt_axis_scalars(xv, fv, sign=-1):
    """The plan of one chirp-z axis as scalars: [(input offset, (n, M, K, shift, alpha, sign, xc, f0, df)), ...] -- one
    entry, or two half-length ones when N + M - 1 exceeds the register engine's longest transform (see CZT.__init__).
    prysm/fttools.py:257-291 builds the same quantities as arrays on the host."""
    N, M = len(xv), len(fv)
    d, df = float(xv[1] - xv[0]), float(fv[1] - fv[0])
    K = next_fast_len(N + M - 1)
    if K > _ENGINE_MAX_K and N % 2 == 0 and next_fast_len(N // 2 + M - 1) <= _ENGINE_MAX_K:
        parts = [(0, N // 2), (N // 2, N // 2)]
    else:
        parts = [(0, N)]
    out = []
    for start, n in parts:
        sub = xv[start:start + n]
        out.append((start, (n, M, next_fast_len(n + M - 1), float(fv[M // 2]) / df, d * df, sign, float(sub[n // 2]), float(fv[0]), df)))
    return out


class CZT:
    """Chirp-z transform with the MDFT interface (prysm/fttools.py:235-369).  Each axis is two
    fused passes: (chirp * data -> FFT_K -> * H) and (IFFT_K -> slice -> * chirp * phase)."""

    def __init__(self, x, y, fx, fy, sign=-1, norm=1.0):
        if sign not in (-1, 1):
            raise ValueError(f'sign must be -1 or +1, got {sign}')
        x, y, fx, fy = _host(x), _host(y), _host(fx), _host(fy)
        self.sign, self.norm = sign, norm
        Nx, Mx, Ny, My = len(x), len(fx), len(y), len(fy)
        dx, dfx = float(x[1] - x[0]), float(fx[1] - fx[0])
        dy, dfy = float(y[1] - y[0]), float(fy[1] - fy[0])
        cd = config.complex_dtype
        dev = _ops.device()
        # One Bluestein plan per axis -- or TWO half-length plans when N + M - 1 exceeds the longest transform of the
        # register-resident engine (4096): sum_n a[n] exp(s 2 pi i x_n f_m) splits exactly into the sums over the two halves
        # of the input, each a CZT of length N/2 on its own sub-grid (own centre coordinate), and N/2 + M - 1 <= 4096 keeps
        # both on the fast kernels (C5's final focus 4096 -> 512: 2 x K = 4096 instead of K = 8192 on the generic kernel).
        # The chirps, phase ramps and kernel spectra are built on the device from ten scalars per plan (fp64 phases):
        # constructing an executor per wavelength costs no host maths and no uploads.
        px, py = czt_axis_scalars(x, fx, sign), czt_axis_scalars(y, fy, sign)
        built = {}

        def build(params):
            if params not in built:      # square, centred geometry (every BASELINE config): one plan serves both axes
                built[params] = _ops.czt_plan(*params, cd, dev)
            return built[params]
        # per axis: list of (input offset, n, K, b, post, H, Hadj)
        self._ax = [(s, p[0], p[2]) + tuple(build(p)) for s, p in px]
        self._ay = [(s, p[0], p[2]) + tuple(build(p)) for s, p in py]
        self._Nx, self._Ny, self._Mx, self._My = Nx, Ny, Mx, My
        Kx, Ky = self._ax[0][2], self._ay[0][2]
        self._bx = self._ax[0][3]
        x_first_cost = Ny * Kx * math.log2(Kx) * len(self._ax) + Mx * Ky * math.log2(Ky) * len(self._ay)
        y_first_cost = Nx * Ky * math.log2(Ky) * len(self._ay) + My * Kx * math.log2(Kx) * len(self._ax)
        self._x_first = x_first_cost <= y_first_cost

    def _forward_axis(self, o, axis, parts, M, scale, out=None):
        # ONE fused call per part: chirp -> FFT_K -> kernel spectrum -> IFFT_K -> slice -> chirp*phase.
        # (the row chirp by[y] of the reference's `out *= brow` commutes with the x pass: it is the y pass's pre_e)
        acc = None
        for start, n, K, b, post, H, _ in parts:
            piece = o[:, start:start + n] if axis == 1 else o[start:start + n]
            r = _ops.czt_axis(piece, K, axis, b, H, post, n - 1, M, scale, out=out if len(parts) == 1 else None)
            acc = r if acc is None else _ops.binary('add', acc, r)
        if out is not None and acc is not out:     # a split axis adds its halves into a new array
            out.copy_(acc)
        return acc if out is None else out

    def _adjoint_axis(self, o, axis, parts, scale, out=None):
        # conj(post) -> FFT_K -> conj(H) with the embedding offset folded in -> IFFT_K -> [:n] -> conj(chirp), per part
        if out is not None and len(parts) == 1:
            _, n, K, b, post, _, Hadj = parts[0]
            return _ops.czt_axis(o, K, axis, post, Hadj, b, 0, n, scale, pre_conj=True, post_conj=True, out=out)
        outs = [_ops.czt_axis(o, K, axis, post, Hadj, b, 0, n, scale, pre_conj=True, post_conj=True)
                for _, n, K, b, post, _, Hadj in parts]
        if out is not None:
            return torch.cat(outs, dim=axis, out=out)
        return outs[0] if len(outs) == 1 else torch.cat(outs, dim=axis)

    def __call__(self, ary):
        return self._forward(ary)

    def _forward(self, ary, out=None):
        o = _prep(ary, self._bx.dtype)
        if tuple(o.shape) != (self._Ny, self._Nx):
            raise ValueError(f'array of shape {tuple(o.shape)} does not match the executor')
        if self._x_first:
            return self._forward_axis(self._forward_axis(o, 1, self._ax, self._Mx, 1.0), 0, self._ay, self._My, self.norm, out)
        return self._forward_axis(self._forward_axis(o, 0, self._ay, self._My, 1.0), 1, self._ax, self._Mx, self.norm, out)

    def _out_shape(self, adjoint):
        return (self._Ny, self._Nx) if adjoint else (self._My, self._Mx)

    @property
    def _dtype(self):
        return self._bx.dtype

    def intensity(self, ary, weight=1.0, out=None):
        """|self(ary)|^2, written to a new real array or, with `out`, accumulated as out += weight * |.|^2: the modulus
        is formed in the store of the last axis pass, the complex focal field is never written (one wavelength of an
        incoherent sum; prysm/propagation/wavefront.py:147-151 + prysm/polynomials/fitting.py:37)."""
        o = _prep(ary, self._bx.dtype)
        if tuple(o.shape) != (self._Ny, self._Nx):
            raise ValueError(f'array of shape {tuple(o.shape)} does not match the executor')
        first = (1, self._ax, self._Mx) if self._x_first else (0, self._ay, self._My)
        last = (0, self._ay, self._My) if self._x_first else (1, self._ax, self._Mx)
        if len(last[1]) != 1:      # split last axis: the two halves add as fields, so the modulus cannot be fused
            return _ops.intensity(self(ary), weight=weight, out=out)
        mid = self._forward_axis(o, first[0], first[1], first[2], 1.0)
        _, n, K, b, post, H, _ = last[1][0]
        kind = OUT_INTENSITY if out is None else OUT_ACCUMULATE
        return _ops.czt_axis(mid, K, last[0], b, H, post, n - 1, last[2], self.norm, out_kind=kind, weight=weight, out=out)

    def adjoint(self, grad):
        return self._adjoint(grad)

    def _adjoint(self, grad, out=None):
        o = _prep(grad, self._bx.dtype)
        if tuple(o.shape) != (self._My, self._Mx):
            raise ValueError(f'array of shape {tuple(o.shape)} does not match the executor')
        if self._x_first:  # undo y then x
            return self._adjoint_axis(self._adjoint_axis(o, 0, self._ay, 1.0), 1, self._ax, self.norm, out)
        return self._adjoint_axis(self._adjoint_axis(o, 1, self._ax, 1.0), 0, self._ay, self.norm, out)

    def nbytes(self):
        vs = {id(v): v for part in self._ax + self._ay for v in part[3:]}
        return sum(v.numel() * v.element_size() for v in vs.values())


def _uniform_spacing(values, name):
    """prysm/fttools.py:484-497 (same messages)."""
    if len(values) < 2:
        raise ValueError(f'{name} must contain at least two samples')
    spacing = float(values[1] - values[0])
    if spacing == 0:
        raise ValueError(f'{name} must have nonzero spacing')
    tolerance = 32 * np.finfo(config.precision).eps
    scale = max(1.0, abs(float(values[0])), abs(float(values[-1])), abs(spacing))
    if not bool(np.allclose(np.diff(values), spacing, rtol=tolerance, atol=tolerance * scale)):
        raise ValueError(f'{name} must be uniformly spaced')
    return spacing


def _fft_compatible_length(alpha, N, M, name):
    """prysm/fttools.py:500-514 (same messages)."""
    inv_alpha = 1 / abs(alpha)
    K = round(inv_alpha)
    tolerance = 32 * np.finfo(config.precision).eps
    if not math.isclose(inv_alpha, K, rel_tol=tolerance, abs_tol=tolerance):
        raise ValueError(f'{name} spacings are not FFT-compatible: '
                         'abs(input spacing * output spacing) must be 1/integer')
    if K < max(N, M):
        raise ValueError(f'{name} requires FFT length {K}, smaller than input/output length {max(N, M)}')
    return K


class FFTDFT:
    """DFT as one FFT per axis when dx*dfx = +-1/K (prysm/fttools.py:392-481): phase ramp ->
    FFT_K -> crop, with the ramps fused into the two passes."""

    def __init__(self, x, y, fx, fy, sign=-1, norm=1.0):
        if sign not in (-1, 1):
            raise ValueError(f'sign must be -1 or +1, got {sign}')
        x, y, fx, fy = _host(x), _host(y), _host(fx), _host(fy)
        Nx, Ny, Mx, My = len(x), len(y), len(fx), len(fy)
        dx, dy = _uniform_spacing(x, 'x'), _uniform_spacing(y, 'y')
        dfx, dfy = _uniform_spacing(fx, 'fx'), _uniform_spacing(fy, 'fy')
        Kx = _fft_compatible_length(dx * dfx, Nx, Mx, 'x/fx')
        Ky = _fft_compatible_length(dy * dfy, Ny, My, 'y/fy')
        cd = config.complex_dtype
        up = lambda v: _ops.asdevice(v.astype(config.precision_complex), cd)  # noqa: E731
        self._pre_x = up(_expi(sign * np.arange(Nx) * dx * float(fx[0])))
        self._pre_y = up(_expi(sign * np.arange(Ny) * dy * float(fy[0])))
        self._post_x = up(_expi(sign * float(x[0]) * fx))
        self._post_y = up(_expi(sign * float(y[0]) * fy))
        self._Nx, self._Ny, self._Mx, self._My, self._Kx, self._Ky = Nx, Ny, Mx, My, Kx, Ky
        self._x_direction = sign if dx * dfx > 0 else -sign
        self._y_direction = sign if dy * dfy > 0 else -sign
        self.norm = norm
        x_first_cost = Ny * Kx * math.log2(Kx) + Mx * Ky * math.log2(Ky)
        y_first_cost = Nx * Ky * math.log2(Ky) + My * Kx * math.log2(Kx)
        self._x_first = x_first_cost <= y_first_cost

    def __call__(self, ary):
        return self._forward(ary)

    def adjoint(self, grad):
        return self._adjoint(grad)

    def _out_shape(self, adjoint):
        return (self._Ny, self._Nx) if adjoint else (self._My, self._Mx)

    @property
    def _dtype(self):
        return self._pre_x.dtype

    def _forward(self, ary, out=None):
        o = _prep(ary, self._pre_x.dtype)
        if tuple(o.shape) != (self._Ny, self._Nx):
            raise ValueError(f'array of shape {tuple(o.shape)} does not match the executor')
        if self._x_first:
            o = _ops.axis_dft(o, self._Kx, 1, self._x_direction, pre_e=self._pre_x, pre_b=self._pre_y,
                              n_out=self._Mx, post_e=self._post_x)
            o = _ops.axis_dft(o, self._Ky, 0, self._y_direction, n_out=self._My, post_e=self._post_y, scale=self.norm,
                              out=out)
        else:
            o = _ops.axis_dft(o, self._Ky, 0, self._y_direction, pre_e=self._pre_y, pre_b=self._pre_x,
                              n_out=self._My, post_e=self._post_y)
            o = _ops.axis_dft(o, self._Kx, 1, self._x_direction, n_out=self._Mx, post_e=self._post_x, scale=self.norm,
                              out=out)
        return o

    def _adjoint(self, grad, out=None):
        o = _prep(grad, self._pre_x.dtype)
        if tuple(o.shape) != (self._My, self._Mx):
            raise ValueError(f'array of shape {tuple(o.shape)} does not match the executor')
        if self._x_first:
            o = _ops.axis_dft(o, self._Ky, 0, -self._y_direction, pre_e=self._post_y, pre_e_conj=True,
                              pre_b=self._post_x, pre_b_conj=True, n_out=self._Ny, post_e=self._pre_y, post_e_conj=True)
            o = _ops.axis_dft(o, self._Kx, 1, -self._x_direction, n_out=self._Nx, post_e=self._pre_x, post_e_conj=True,
                              scale=self.norm, out=out)
        else:
            o = _ops.axis_dft(o, self._Kx, 1, -self._x_direction, pre_e=self._post_x, pre_e_conj=True,
                              pre_b=self._post_y, pre_b_conj=True, n_out=self._Nx, post_e=self._pre_x, post_e_conj=True)
            o = _ops.axis_dft(o, self._Ky, 0, -self._y_direction, n_out=self._Ny, post_e=self._pre_y, post_e_conj=True,
                              scale=self.norm, out=out)
        return o

    def nbytes(self):
        return sum(v.numel() * v.element_size() for v in (self._pre_x, self._pre_y, self._post_x, self._post_y))


def _resample_geometry(shape, zoom):
    """(zoom pair, output shape) of fourier_resample, with the reference's checks (prysm/fttools.py:562-576)."""
    if isinstance(zoom, (float, int)):
        zoom = (zoom, zoom)
    elif not isinstance(zoom, tuple):
        zoom = tuple(float(z) for z in zoom)
    if len(zoom) != 2 or any(z <= 0 for z in zoom):
        raise ValueError('zoom must contain two positive values')
    m, n = shape
    M, N = int(m * zoom[0]), int(n * zoom[1])
    if M < 1 or N < 1:
        raise ValueError('zoom produces an empty output')
    return zoom, (M, N)


class FourierResampler:
    """The fixed part of fourier_resample for one input shape and zoom, built once: calling it on an (m, n) array runs
    the centred FFT and the matrix DFT and returns the COMPLEX (int(m*zoom), int(n*zoom)) result."""

    def __init__(self, shape, zoom):
        zoom, (M, N) = _resample_geometry(shape, zoom)
        m, n = shape
        rng = lambda k: np.arange(-(k // 2), -(k // 2) + k, dtype=np.float64)      # noqa: E731  (fftrange on the host)
        self.shape, self.out_shape = (m, n), (M, N)
        self._op = MDFT(rng(n), rng(m), rng(N) * (1.0 / zoom[1] / n), rng(M) * (1.0 / zoom[0] / m), sign=+1,
                        norm=1.0 / (m * n))

    def __call__(self, f):
        F = _ops.fft2(f, self.shape, dir=-1, shift_in=True, shift_out=True)
        return self._op(F)


def fourier_resample(f, zoom):
    """Resample f by Fourier methods: centred FFT, then a sign=+1 matrix DFT onto int(m*zoom) x int(n*zoom)
    samples spaced 1/zoom, scaled by 1/(m n) (prysm/fttools.py:538-593).  Real in -> real out."""
    if zoom == 1:
        return f
    _resample_geometry(tuple(f.shape), zoom)
    f = _ops.asdevice(f)
    out = FourierResampler(tuple(f.shape), zoom)(f)
    return out if f.is_complex() else out.real
