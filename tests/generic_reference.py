"""Extended-precision reference and launch rules of the generic axis pass (csrc/axis_pass.cu) and of Bluestein's
algorithm on top of it (csrc/fft2.cu: axis_dft, get_chirp, get_chirp_filter, bluestein_len).

The reference is scipy.fft on np.clongdouble: an 80-bit FFT on x86-64 (eps 1.1e-19), four orders of magnitude below
a correct complex128 transform (about 1e-15), so a figure against it is the device's own error.  A host whose long
double is just a double would compare fp64 against fp64 and pass anything: importing this module fails there.

The numpy models of the device's Bluestein (`bluestein_model`) follow the C++ rules step by step, with optional
defects, so that tests/test_host_generic_reference.py can show that the ceilings of the GPU test catch each defect.
"""
import numpy as np
import scipy.fft as sfft

from accuracy import ld

LD = np.clongdouble
PI_LD = np.longdouble('3.14159265358979323846264338327950288')
PB_C64, PB_C128 = 0, 1
CPLX = {PB_C64: np.complex64, PB_C128: np.complex128}
DT_NAME = {PB_C64: 'c64', PB_C128: 'c128'}
CEILING = {PB_C64: 1e-6, PB_C128: 1e-14}     # hard ceilings of the bounds: a figure above one is a finding
SMEM_OPTIN_H100 = 232448                       # cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100
CSIZE = {PB_C64: 8, PB_C128: 16}


# ---- the C++ rules --------------------------------------------------------------------------------------------------
def bluestein_len(n):
    """bluestein_len: the least power of two M >= 2n - 1"""
    m = 1
    while m < 2 * n - 1:
        m <<= 1
    return m


def is_pow2(n):
    return n > 0 and n & (n - 1) == 0


def max_pow2_len(dtype, cap=SMEM_OPTIN_H100):
    """generic_max_len: the largest power-of-two line that fits one CTA's shared memory"""
    L = 1
    while 2 * L * CSIZE[dtype] <= cap:
        L <<= 1
    return L


def accepts(n, dtype, cap=SMEM_OPTIN_H100):
    """axis_dft's test: a power of two up to max_pow2_len, any other length whose Bluestein M fits"""
    lmax = max_pow2_len(dtype, cap)
    return n <= lmax and (is_pow2(n) or bluestein_len(n) <= lmax)


def max_len(dtype, cap=SMEM_OPTIN_H100):
    """the largest length of any kind (non-power-of-two lengths stop at half the power-of-two limit)"""
    return max_pow2_len(dtype, cap) // 2


def axis_launches(n, dtype, cols):
    """{(L, dtype, cols): generic launches} of one logical axis of length n: one pass at L = n for a power of two, two
    at L = bluestein_len(n) otherwise"""
    if is_pow2(n):
        return {(n, dtype, int(cols)): 1}
    return {(bluestein_len(n), dtype, int(cols)): 2}


def merge(*counts):
    out = {}
    for c in counts:
        for k, v in c.items():
            out[k] = out.get(k, 0) + v
    return out


# ---- the long-double reference --------------------------------------------------------------------------------------
def fft_ld(a, n=None, axis=-1, inverse=False):
    """numpy's fft(a, n, axis) (inverse: unnormalised, sign +) in long double"""
    a = ld(a)
    if inverse:
        n_ = a.shape[axis] if n is None else n
        return sfft.ifft(a, n, axis=axis) * n_
    return sfft.fft(a, n, axis=axis)


def centred_ft2_ld(a, k, inverse=False, crop=None, shift=True):
    """fft2 of `a` zero-padded to k at offset ceil((k - n)/2), with ifftshift before and fftshift after when `shift`
    (unnormalised), cropped to the centred window `crop`"""
    a = ld(a)
    ky, kx = k
    ny, nx = a.shape
    p = np.zeros((ky, kx), dtype=LD)
    oy, ox = -(-(ky - ny) // 2), -(-(kx - nx) // 2)
    p[oy:oy + ny, ox:ox + nx] = a
    if shift:
        p = sfft.ifftshift(p)
    f = sfft.ifft2(p) * (ky * kx) if inverse else sfft.fft2(p)
    if shift:
        f = sfft.fftshift(f)
    if crop is not None:
        cy, cx = crop
        y0, x0 = -(-(ky - cy) // 2), -(-(kx - cx) // 2)
        f = f[y0:y0 + cy, x0:x0 + cx]
    return f


def expi_ld(turns):
    """exp(2 pi i turns) in long double, turns reduced to [-1/2, 1/2] first (exact)"""
    t = np.asarray(turns, dtype=np.longdouble)
    t = t - np.round(t)
    ang = 2 * PI_LD * t
    return np.cos(ang) + 1j * np.sin(ang).astype(LD)


def phase_field_ld(opd, kscale, amp=None):
    """the amplitude / OPD input kind: turns = (kscale / 2 pi) * opd formed in double exactly as the kernel does, then
    amp * exp(2 pi i turns) in long double (a u8 / bool amplitude is 0 or 1)"""
    kturns = float(kscale) / (2.0 * np.pi)
    turns = kturns * np.asarray(opd).astype(np.float64)
    e = expi_ld(turns)
    if amp is not None:
        amp = np.asarray(amp)
        a = (amp != 0).astype(np.longdouble) if amp.dtype in (np.bool_, np.uint8) else amp.astype(np.longdouble)
        e = e * a
    return e


def ramp_ld(m, p, K, sign):
    """exp(sign 2 pi i m p / K) with the product m p reduced mod K in integers"""
    r = (np.asarray(m, dtype=np.int64) * int(p)) % K
    ang = sign * 2 * PI_LD * r.astype(np.longdouble) / K
    return np.cos(ang) + 1j * np.sin(ang).astype(LD)


def impulse_centred_ft2(n, k, pixels, values, inverse=False, crop=None):
    """centred_ft2_ld (shift=True) of an n = (ny, nx) array that is zero but for values[i] at pixels[i], in closed
    form: an impulse at padded position P of a K-point axis becomes exp(-+2 pi i (m - K//2)(P - K//2) / K)"""
    (ny, nx), (ky, kx) = n, k
    cy, cx = (ky, kx) if crop is None else crop
    s = 1 if inverse else -1
    my = np.arange(cy) + -(-(ky - cy) // 2) - ky // 2
    mx = np.arange(cx) + -(-(kx - cx) // 2) - kx // 2
    out = np.zeros((cy, cx), dtype=LD)
    for (a, b), v in zip(pixels, values):
        ey = ramp_ld(my % ky, a + -(-(ky - ny) // 2) - ky // 2, ky, s)
        ex = ramp_ld(mx % kx, b + -(-(kx - nx) // 2) - kx // 2, kx, s)
        out += LD(v) * np.outer(ey, ex)
    return out


def rel_linf(a, b):
    den = float(np.abs(b).max())
    return float(np.abs(ld(a) - b).max()) / (den if den > 0 else 1.0)


def rel_l2(a, b):
    den = float(np.sqrt(np.sum(np.abs(b) ** 2)))
    return float(np.sqrt(np.sum(np.abs(ld(a) - b) ** 2))) / (den if den > 0 else 1.0)


# ---- numpy models of the device's Bluestein ---------------------------------------------------------------------
DEFECTS = ('unreduced', 'angle32', 'twiddle32', 'mirror_off', 'filter_conj', 'window_off', 'jj32')


def _expi_pi(r, n, sign, angle32=False):
    """exp(sign pi i r / n), as the host tables form it: the angle in long double, then rounded to double"""
    ang = sign * PI_LD * np.asarray(r, dtype=np.longdouble) / n
    if angle32:
        ang = ang.astype(np.float32).astype(np.longdouble)
    return (np.cos(ang) + 1j * np.sin(ang).astype(LD)).astype(np.complex128)


def _fft_pow2(a, sign, cdt, twiddle32=False):
    """the generic kernel's transform: radix-2 decimation in time over bit-reversed input, in cdt arithmetic, with the
    twiddle table exp(-2 pi i k / L) rounded once to cdt (twiddle32: from fp32-rounded angles)"""
    L = a.shape[-1]
    lg = L.bit_length() - 1
    k = np.arange(L // 2 if L > 1 else 1)
    ang = -2 * PI_LD * k.astype(np.longdouble) / L
    if twiddle32:
        ang = ang.astype(np.float32).astype(np.longdouble)
    tw = (np.cos(ang) + 1j * np.sin(ang).astype(LD)).astype(cdt)
    if sign > 0:
        tw = np.conj(tw)
    rev = np.zeros(L, dtype=np.int64)
    for b in range(lg):
        rev |= ((np.arange(L) >> b) & 1) << (lg - 1 - b)
    x = a.astype(cdt)[..., rev]
    h = 1
    while h < L:
        x = x.reshape(x.shape[:-1] + (L // (2 * h), 2, h))
        w = tw[(np.arange(h) * (L // (2 * h)))]
        t = x[..., 1, :] * w
        u = x[..., 0, :]
        x = np.stack((u + t, u - t), axis=-2).reshape(x.shape[:-3] + (L,))
        h *= 2
    return x


def bluestein_model(x, dtype, defect=None, dir=-1):
    """axis_dft on a non-power-of-two length n, modelled on the host: chirp c[j] = exp(dir pi i (j^2 mod 2n) / n),
    filter g[d mod M] = conj(c[|d|]) transformed in double, stage 1 FFT_M(x c) G, stage 2 IFFT_M / M times c on
    k < n -- in the arithmetic of dtype (PB_C64: float32, PB_C128: float64).  `defect` is one of DEFECTS."""
    assert defect in (None,) + DEFECTS
    cdt = CPLX[dtype]
    n = x.shape[-1]
    M = bluestein_len(n)
    j = np.arange(n, dtype=np.int64)
    if defect == 'jj32':
        r = np.float32(j.astype(np.float32) * j.astype(np.float32)).astype(np.float64) % (2 * n)
    else:
        r = (j * j) % (2 * n)
    c = _expi_pi(r, n, dir, angle32=defect == 'angle32')
    if defect == 'unreduced':        # the angle pi j^2 / n of an unreduced square, formed and taken in double
        ang = dir * np.pi * (j.astype(np.float64) * j.astype(np.float64)) / n
        c = np.cos(ang) + 1j * np.sin(ang)
    g = np.zeros(M, dtype=np.complex128)
    v = _expi_pi((j * j) % (2 * n), n, -dir)
    if defect == 'filter_conj':
        v = np.conj(v)
    g[:n] = v
    if defect == 'mirror_off':
        g[(M - j[1:] + 1) % M] = v[1:]
    else:
        g[M - j[1:]] = v[1:]
    G = sfft.fft(g).astype(cdt)                         # host_fft_pow2 in double, rounded to the table's type
    c = c.astype(cdt)
    u = np.zeros(x.shape[:-1] + (M,), dtype=cdt)
    u[..., :n] = x.astype(cdt) * c
    tw32 = defect == 'twiddle32'
    U = _fft_pow2(u, -1, cdt, tw32) * G
    V = _fft_pow2(U, +1, cdt, tw32)
    k = j + 1 if defect == 'window_off' else j
    return V[..., k % M] * c * cdt(1.0 / M).real
