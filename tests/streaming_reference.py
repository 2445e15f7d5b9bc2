"""Plain high-precision references, launch geometry and defect models of the streaming kernels: the adjoint seeds and
elementwise twins of csrc/adjoint_ops.cu, the non-transform kernels of csrc/elementwise.cu and the image chain of
csrc/imagechain.cu.

Reductions are summed in long double (np.longdouble / np.clongdouble, 80-bit on x86-64) and return, beside the value,
the condition denominator sum|terms|: a device reduction that accumulates in fp64 lands within a few fp64 ulps of
that denominator whatever the cancellation, so |got - ref| / sum|terms| is the figure.  Elementwise references are
formed in fp64 or long double from the very values handed to the device (for float32 runs, the float32-rounded
inputs), so a figure is the kernel's own rounding.

The launch rules are mirrored from the C++ so that a test can build shapes that put each kernel on both sides of its
grid cap from the device's SM count, and count the launches an entry point makes.

The `defect` models (numpy versions of a kernel with one deliberate fault) are used by
tests/test_host_streaming_reference.py only, to show that the GPU test's ceilings would catch each fault.
"""
import math

import numpy as np
import scipy.fft as sfft
import scipy.ndimage as ndi
import scipy.special as sps

import generic_reference as G
from accuracy import LDBL, THREADS, grid_for, ld, sweep  # noqa: F401
from generic_reference import LD, PB_C64, PB_C128, expi_ld, phase_field_ld, centred_ft2_ld  # noqa: F401

RDT = {PB_C64: np.float32, PB_C128: np.float64}
CDT = {PB_C64: np.complex64, PB_C128: np.complex128}
DT_NAME = G.DT_NAME
CEIL_ELEM = G.CEILING                 # relative L-inf of an elementwise output: a few ulps of R
CEIL_RED = 1e-13                      # |got - ref| / sum|terms| of an fp64-accumulated reduction, both dtypes
CEIL_EE = 1e-12                       # encircled energy: the same over ee_ref's majorant, j1 error included


# ---- launch geometry (mirrors of the C++) --------------------------------------------------------------------------
PB_MAX_MODES = 64                     # csrc/elementwise.cu: #define PB_MAX_MODES 64 (weights per weighted_sum launch)


def reduction_grid(n, sm_count, threads=THREADS):
    """the grid of pb_dot, pb_otf_adjoint_seed, pb_balance_scale and pb_encircled_energy (csrc/common.cuh fold_blocks:
    min(ceil(n/256), sm_count*4))"""
    return min((n + threads - 1) // threads, sm_count * 4)


def mode_projection_gx(n, k, sm_count, threads=THREADS):
    """pb_mode_projection (csrc/adjoint_ops.cu): blocks per mode, min(ceil(n/256), max(1, sm_count*4 // k))"""
    return min((n + threads - 1) // threads, max(1, sm_count * 4 // k))


def reduction_cap(sm_count):
    return sm_count * 4 * THREADS


def shapes(sm_count):
    """{name: (ny, nx)} of the streaming tests: element counts of cap - 1, cap and cap + 1 for both caps (alternating
    1 x n and n x 1), 1 x 1, 1 x n, n x 1, a partial warp, an odd shape, and two that take many sweeps"""
    out = {'1x1': (1, 1), '1xn': (1, 1000), 'nx1': (1000, 1), '31x33': (31, 33), '1023x769': (1023, 769),
           '2048sq': (2048, 2048), '4096sq': (4096, 4096)}
    for tag, cap in (('red', reduction_cap(sm_count)), ('elem', sweep(sm_count))):
        out.update({f'{tag}-1': (1, cap - 1), tag: (cap, 1), f'{tag}+1': (1, cap + 1)})
    return out


SHAPE_NAMES = ('1x1', '1xn', 'nx1', '31x33', '1023x769', '2048sq', '4096sq', 'red-1', 'red', 'red+1', 'elem-1', 'elem',
               'elem+1')


# ---- figures --------------------------------------------------------------------------------------------------------
def rel_linf(got, ref):
    """max|got - ref| / max|ref| (NaN anywhere in got: infinity)"""
    got = np.asarray(got)
    if not np.all(np.isfinite(got)):
        return math.inf
    den = float(np.abs(ref).max())
    return float(np.abs(ld(got) - ref).max()) / (den if den > 0 else 1.0)


def red_fig(got, ref, cond):
    """|got - ref| / sum|terms| elementwise over a vector of reductions, max"""
    got, ref, cond = np.atleast_1d(got), np.atleast_1d(ref), np.atleast_1d(cond)
    if not np.all(np.isfinite(got)):
        return math.inf
    cond = np.where(cond > 0, cond, 1)
    return float(np.max(np.abs(ld(got) - ref) / cond))


# ---- reductions -----------------------------------------------------------------------------------------------------
def dot_ref(a, b, w=None):
    """sum w * a * conj(b) and sum |w| |a| |b|"""
    t = ld(a) * np.conj(ld(b))
    if w is not None:
        t = t * ld(w)
    return t.sum(), np.abs(t).sum()


def mode_projection_ref(modes, bar):
    """tensordot(modes, bar) over the trailing axes, and the per-mode sum|terms|"""
    m = ld(modes).reshape(modes.shape[0], -1)
    g = ld(bar).reshape(-1)
    return m @ g, np.abs(m) @ np.abs(g)


def moments_ref(d):
    """(sum v, sum v y, sum v x) and (sum |v|, sum |v| y, sum |v| x)"""
    d = ld(d)
    y = np.arange(d.shape[0], dtype=LDBL)[:, None]
    x = np.arange(d.shape[1], dtype=LDBL)[None, :]
    a = np.abs(d)
    return np.array([d.sum(), (d * y).sum(), (d * x).sum()]), np.array([a.sum(), (a * y).sum(), (a * x).sum()])


def balance_ref(a, b):
    """pb_balance_scale: sqrt(sum a^2 / sum b^2), 1 where either is zero or not finite"""
    sa, sb = (ld(a) ** 2).sum(), (ld(b) ** 2).sum()
    ok = sa > 0 and sb > 0 and np.isfinite(sa) and np.isfinite(sb)
    return (np.sqrt(sa / sb) if ok else LDBL(1)), (sa, sb)


def ee_nu(shape, df):
    """the fftrange * df frequency radius of the EE kernels, nu(0) -> 1e-16"""
    ny, nx = shape
    fy = (np.arange(ny) - ny // 2) * df
    fx = (np.arange(nx) - nx // 2) * df
    nu = np.hypot(fx[None, :], fy[:, None])
    return np.where(nu == 0, 1e-16, nu)


def ee_ref(mtf, df, radii):
    """Baliga & Cohn: r * sum(mtf * j1(2 pi r nu) / nu) * df^2 (scipy.special.j1, long-double sum), and the condition
    denominator r * sum(|mtf| min(pi r nu, 0.582) / nu) * df^2: |j1(x)| <= min(x/2, 0.582), so each term of it bounds
    that term, and an absolute j1 error enters relative to it"""
    nu = ee_nu(mtf.shape, df)
    m = ld(mtf)
    out, cond = [], []
    for r in radii:
        t = m * ld(sps.j1(2 * np.pi * r * nu) / nu)
        out.append(t.sum() * LDBL(r) * LDBL(df) ** 2)
        cond.append((np.abs(m) * ld(np.minimum(np.pi * r * nu, 0.582) / nu)).sum() * LDBL(r) * LDBL(df) ** 2)
    return np.array(out), np.array(cond)


def ee_adjoint_seed_ref(shape, df, radii, ee_bar):
    """mtf_bar = sum_r eebar[r] r j1(2 pi r nu) / nu df^2 (fp64 per term, summed in long double)"""
    nu = ee_nu(shape, df)
    acc = np.zeros(shape, dtype=LDBL)
    for r, g in zip(radii, ee_bar):
        acc += ld(g * r * (sps.j1(2 * np.pi * r * nu) / nu) * df * df)
    return acc


# ---- OTF path -------------------------------------------------------------------------------------------------------
def centre_index(shape):
    """pb_otf_normalize / pb_otf_adjoint_seed: (ny // 2, nx // 2)"""
    return shape[0] // 2, shape[1] // 2


def otf_normalize_ref(D):
    """(mtf, ptf, otf) of D / D[centre] in long double"""
    D = ld(D)
    q = D / D[centre_index(D.shape)]
    return np.abs(q), np.arctan2(q.imag, q.real), q


def otf_adjoint_seed_ref(which, bar, D, defect=None):
    """gradient at the k-space plane of mtf (1) / ptf (2) / otf (4) = f(D / D[centre]) under the pairing
    Re sum conj(seed) dD; returns (seed, S, sum|terms of S|).  Long double.  Defects: 'no_centre' drops the centre
    correction; 'centre_nm1' takes the centre at ((ny-1)//2, (nx-1)//2)."""
    D = ld(D)
    g = ld(bar)
    cy, cx = ((D.shape[0] - 1) // 2, (D.shape[1] - 1) // 2) if defect == 'centre_nm1' else centre_index(D.shape)
    c = D[cy, cx]
    if which == 1:
        a = np.abs(c)
        seed = g * D / np.abs(D) / a
        t = g * np.abs(D)
        S = t.sum()
        corr = S * c / a ** 3
    elif which == 2:
        seed = g * 1j * D / np.abs(D) ** 2
        t = g
        S = t.sum()
        corr = S * 1j * c / np.abs(c) ** 2
    else:
        seed = g / np.conj(c)
        t = np.conj(D) * g
        S = t.sum()
        corr = S / np.conj(c) ** 2
    if defect != 'no_centre':
        seed[cy, cx] -= corr
    return seed, S, np.abs(t).sum()


def transform_psf_ld(psf):
    """fftshift(fft2(ifftshift(psf))) in long double (prysm otf.transform_psf)"""
    return centred_ft2_ld(psf, psf.shape)


def transform_psf_adjoint_ld(g):
    """fftshift(ifft2(ifftshift(g), norm='forward')) in long double"""
    return centred_ft2_ld(g, g.shape, inverse=True)


def mtf_ptf_otf_from_psf_ld(psf):
    return otf_normalize_ref(transform_psf_ld(psf))


def otf_from_psf_adjoint_ld(which, bar, psf):
    """the composite reverse map psf_bar = Re transform_psf_adjoint(seed)"""
    seed, _, _ = otf_adjoint_seed_ref(which, bar, transform_psf_ld(psf))
    return transform_psf_adjoint_ld(seed).real


def encircled_energy_ld(psf, dx, radii_mm):
    mtf = mtf_ptf_otf_from_psf_ld(psf)[0]
    df = 1000 / (psf.shape[0] * dx)
    return ee_ref(np.asarray(mtf, dtype=np.float64), df, radii_mm)[0]


def encircled_energy_adjoint_ld(ee_bar, psf, dx, radii_mm):
    df = 1000 / (psf.shape[0] * dx)
    mtf_bar = ee_adjoint_seed_ref(psf.shape, df, radii_mm, ee_bar)
    return otf_from_psf_adjoint_ld(1, mtf_bar, psf)


# ---- elementwise ----------------------------------------------------------------------------------------------------
def mask_multiply_ref(a, m=None, b=None, w=None, conj=False, one_minus=False, real_out=False, scale=1.0, out0=None,
                      rdt=np.float64, defect=None):
    """out (+)= scale * (a - b) * f(m) * w, f = m, conj(m), 1 - m or conj(1 - m); scale is rounded to R as the kernel
    gets it.  Defect 'one_minus_re': 1 - m formed on the real part only (the imaginary part kept)."""
    v = ld(a)
    if b is not None:
        v = v - ld(b)
    if m is not None:
        f = ld(m).astype(LD)
        if one_minus:
            f = (1 - f.real) + 1j * f.imag if defect == 'one_minus_re' else 1 - f
        if conj:
            f = np.conj(f)
        v = v * f
    s = ld(rdt(scale))
    if w is not None:
        s = s * ld(w)
    v = v * s
    if real_out:
        v = v.real
    if out0 is not None:
        v = v + ld(out0)
    return v


def field_adjoint_ref(mode, f, bar, opd, k):
    """0: i k imag(bar conj(f)) (complex);  1: real(bar conj(f)) / |f|, 0 where f = 0;  2: real(bar conj(exp(i k opd)))"""
    g = ld(bar)
    if mode == 0:
        return 1j * LDBL(k) * (g * np.conj(ld(f))).imag
    if mode == 1:
        p = ld(f)
        mod = np.abs(p)
        return np.where(mod > 0, (g * np.conj(p)).real / np.where(mod > 0, mod, 1), 0)
    return (g * np.conj(phase_field_ld(opd, k))).real


def component_ref(which, v):
    v = ld(v)
    return {'real': v.real, 'imag': v.imag, 'angle': np.arctan2(v.imag, v.real), 'abs': np.abs(v)}[which]


def binary_ref(op, a, b, reverse=False):
    x, y = ld(a), ld(b)
    if reverse:
        x, y = y, x
    return {'mul': lambda: x * y, 'truediv': lambda: x / y, 'add': lambda: x + y, 'sub': lambda: x - y}[op]()


def div_model(x, y, rdt, defect=None):
    """the kernels' complex division in numpy: x conj(y) / |y|^2 with |y|^2 formed in fp64 and the quotient rounded
    once to rdt; defect 'den_r' forms everything in rdt (float32 overflows past |y| ~ 1.8e19)"""
    wt = rdt if defect == 'den_r' else np.float64
    with np.errstate(all='ignore'):
        xr, xi = x.real.astype(wt), x.imag.astype(wt)
        yr, yi = y.real.astype(wt), y.imag.astype(wt)
        d = yr * yr + yi * yi
        qr = (xr * yr + xi * yi) / d
        qi = (xi * yr - xr * yi) / d
        return (qr.astype(rdt) + 1j * qi.astype(rdt)).astype(np.complex64 if rdt == np.float32 else np.complex128)


def intensity_ref(v, weight=1.0, out0=None, rdt=np.float64):
    r = np.abs(ld(v)) ** 2 * ld(rdt(weight))
    return r if out0 is None else r + ld(out0)


def mul_outer_ref(a, vy=None, vx=None, conj_y=False, conj_x=False, scale=1.0, rdt=np.float64):
    v = ld(a)
    if vy is not None:
        v = v * (np.conj(ld(vy)) if conj_y else ld(vy))[:, None]
    if vx is not None:
        v = v * (np.conj(ld(vx)) if conj_x else ld(vx))[None, :]
    return v * ld(rdt(scale))


def weighted_sum_ref(modes, weights, rdt=np.float64):
    """sum_k w_k modes_k with the weights rounded to R, as the kernel gets them"""
    w = ld(np.asarray(weights, dtype=np.float64).astype(rdt))
    return np.tensordot(w, ld(modes), axes=1)


def weighted_sum_model(modes, weights, defect=None):
    """the chunked fp64 launch sequence of pb_weighted_sum; defect 'no_accumulate': each chunk overwrites"""
    out = np.zeros(modes.shape[1:])
    for k0 in range(0, len(weights), PB_MAX_MODES):
        acc = out if (k0 > 0 and defect != 'no_accumulate') else np.zeros_like(out)
        for m in range(k0, min(len(weights), k0 + PB_MAX_MODES)):
            acc = acc + weights[m] * modes[m]
        out = acc
    return out


def vortex_ref(charge, xf, yf):
    """exp(i charge atan2(y, x)) in long double"""
    th = np.arctan2(ld(yf), ld(xf))
    return expi_ld(LDBL(charge) * th / (2 * G.PI_LD))


def resample_ref(cmap, xf, yf, cx, cy, dx, fill, defect=None):
    """map_coordinates(order=1, mode='nearest') at row = (yf - cy)/dx + ny//2, col = (xf - cx)/dx + nx//2 (fp64), and
    `fill` outside [0, n-1] on either axis or at a NaN coordinate.  Defect 'clamp_m1': the last row / column counts as
    outside."""
    ny, nx = cmap.shape
    col = (np.asarray(xf, np.float64) - cx) / dx + nx // 2
    row = (np.asarray(yf, np.float64) - cy) / dx + ny // 2
    hi_r, hi_c = (ny - 2, nx - 2) if defect == 'clamp_m1' else (ny - 1, nx - 1)
    with np.errstate(invalid='ignore'):
        inside = (row >= 0) & (row <= hi_r) & (col >= 0) & (col <= hi_c)
    rr, cc = np.where(inside, row, 0), np.where(inside, col, 0)
    m = np.asarray(cmap, np.complex128)
    re = ndi.map_coordinates(m.real, [rr.ravel(), cc.ravel()], order=1, mode='nearest').reshape(rr.shape)
    im = ndi.map_coordinates(m.imag, [rr.ravel(), cc.ravel()], order=1, mode='nearest').reshape(rr.shape)
    fillv = np.broadcast_to(np.asarray(fill, np.complex128), rr.shape)
    return np.where(inside, re + 1j * im, fillv)


def radial_axes_ref(shape, fdx, shift, rdt):
    """the focal grids of one multi-resolution level as numpy forms them in R: (i - n//2) * fdx + shift, two roundings"""
    ny, nx = shape
    x = (np.arange(nx) - nx // 2).astype(rdt) * rdt(fdx) + rdt(shift)
    y = (np.arange(ny) - ny // 2).astype(rdt) * rdt(fdx) + rdt(shift)
    return np.broadcast_to(x[None, :], shape), np.broadcast_to(y[:, None], shape)


def smootherstep(t):
    t = np.clip(t, 0, 1)
    return t * t * t * (t * (t * 6 - 15) + 10)


def radial_window_ref(xf, yf, here, nxt):
    """taper(here) - taper(nxt), taper = 1 - smootherstep((r - a)/(b - a)); None: 1 (outer) / 0 (inner)"""
    r = np.hypot(ld(xf), ld(yf))
    a = LDBL(1) if here is None else 1 - smootherstep((r - here[0]) / LDBL(here[1] - here[0]))
    b = LDBL(0) if nxt is None else 1 - smootherstep((r - nxt[0]) / LDBL(nxt[1] - nxt[0]))
    return a - b + np.zeros(r.shape, dtype=LDBL)


# ---- image chain ----------------------------------------------------------------------------------------------------
def mirror(n, defect=None):
    """index of -k on an n-point DFT axis: (n - k) % n; defect 'mirror_nm1' uses n - 1 - k"""
    k = np.arange(n)
    return n - 1 - k if defect == 'mirror_nm1' else (n - k) % n


def packed_product_ref(Z, scale=1.0, im_scale=1.0, defect=None):
    """O H = (Z[k]^2 - conj(Z[-k])^2) / (4i) * scale / im_scale, long double"""
    Z = ld(Z)
    ny, nx = Z.shape
    Zm = Z[mirror(ny, defect)][:, mirror(nx, defect)]
    return (Z * Z - np.conj(Zm) ** 2) / (4j) * LDBL(scale) / LDBL(im_scale)


def ft2_ld(a):
    return G.fft_ld(G.fft_ld(a, axis=1), axis=0)


def conv_ref(obj, psf):
    """circular convolution ifft2(fft2(obj) fft2(psf)) in long double (real part)"""
    return sfft.ifft2(ft2_ld(obj) * ft2_ld(psf)).real


def bindown_ref(a, fy, fx, mean):
    ny, nx = a.shape
    s = ld(a).reshape(ny // fy, fy, nx // fx, fx).sum(axis=(1, 3))
    return s / (fy * fx) if mean else s


def tile_ref(a, fy, fx, scale, rdt=np.float64):
    return np.repeat(np.repeat(ld(a), fy, axis=0), fx, axis=1) * ld(rdt(scale))


def separable_tf_ref(kind, fx, fy, wx, wy):
    """0: sinc(fx wx) sinc(fy wy) (numpy's normalised sinc);  1: cos(2 wx fx) cos(2 wy fy); arguments in fp64"""
    ax = ld(np.asarray(fx, np.float64) * wx)
    ay = ld(np.asarray(fy, np.float64) * wy)
    if kind == 0:
        def sinc(t):
            pt = G.PI_LD * t
            return np.where(t == 0, LDBL(1), np.sin(pt) / np.where(t == 0, 1, pt))
        return sinc(ay)[:, None] * sinc(ax)[None, :]
    return np.cos(2 * ay)[:, None] * np.cos(2 * ax)[None, :]


# ---- the fp64 weighted dot as the kernel forms it, for the conj defect ----------------------------------------------
def dot_model(a, b, w=None, defect=None):
    """sum w a conj(b) in fp64; defect 'conj_swap' conjugates a instead of b"""
    t = np.conj(a) * b if defect == 'conj_swap' else a * np.conj(b)
    if w is not None:
        t = t * w
    return t.sum()
