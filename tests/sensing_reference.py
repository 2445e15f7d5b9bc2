"""Plain high-precision references, launch rules and defect models of the wavefront-sensing kernels: the fiber modes,
coupling, combine, grating and PSI passes of csrc/wfs.cu and the lenslet screen, centroids and reconstructor of
csrc/shack_hartmann.cu.

References are written from the documented definitions (DESIGN 4.12 / 4.14, the spot_centroids docstring), not from
the engine's host code.  Sums are in long double (80-bit on x86-64) and return, beside the value, the sum of the terms'
magnitudes: a device reduction that accumulates in fp64 lands within a few fp64 ulps of that sum whatever the
cancellation.  Integer PSI sums are exact (int64).

The launch rules are mirrored from the C++ so that the GPU test can put each kernel on both sides of every chunk, vector
route and per-launch split, and count what it launched.  The Bessel reference values are a committed fixture
(tests/golden/wfs_bessel*.npz) computed at 40 digits with mpmath by `write_bessel_fixture`; nothing else here imports
mpmath.

The `defect` models (numpy versions of a kernel with one deliberate fault) are used by
tests/test_host_sensing_reference.py only, to show that the GPU test's ceilings would catch each fault.
"""
import math
import os

import numpy as np
import scipy.special as sps

from accuracy import LDBL

# ---- launch rules (mirrors of csrc/wfs.cu and csrc/shack_hartmann.cu) ----------------------------------------------
THREADS = 256                   # kThreads of both files
OVERLAP_CHUNK = 4096            # PB_OVERLAP_CHUNK: pixels per stage-1 block of pb_overlap
OV_GROUP = 8                    # kOvGroup: modes per stage-1 block
OV_MAX = 256                    # kOvMax: mode pointers per pb_overlap launch
LP_MAX = 64                     # kLpMax: mode plans per pb_lp_modes launch
PSI_MAX = 64                    # kPsiMax: frames of pb_psi
CENTROID_VEC = 4                # kCentroidVec: grid columns per thread of the vector centroid route
CENTROID_SMEM = 48 * 1024       # kCentroidSmemMax: bytes of dynamic shared memory of a centroid CTA
GRID_Y_MAX = 65535              # frames per centroid / reconstruct launch (gridDim.y)

ELEM_SIZE = {'float32': 4, 'float64': 8, 'uint16': 2, 'int32': 4}


def overlap_chunks(n):
    return -(-n // OVERLAP_CHUNK)


def overlap_launches(P):
    """stage-1 launches of 256 modes each, then one stage-2 launch"""
    return -(-P // OV_MAX) + 1


def lp_launches(P):
    return -(-P // LP_MAX)


def centroid_smem(ncols, V):
    return (5 * ncols + 3 * THREADS * V) * 8


def centroid_route(W, ncols, aligned=True, elem_size=4):
    """V of pb_subaperture_centroids (4 or 1), or None when it refuses the lenslet row: V = 4 needs W % 4 == 0, a frame
    start and stride aligned to 4 elements, and 5 ncols + 3 * 256 * 4 doubles within 48 KB (ncols <= 614); V = 1 needs
    ncols <= 1075."""
    if W % CENTROID_VEC == 0 and aligned and centroid_smem(ncols, CENTROID_VEC) <= CENTROID_SMEM:
        return CENTROID_VEC
    return 1 if centroid_smem(ncols, 1) <= CENTROID_SMEM else None


CENTROID_NCOLS_V4 = max(k for k in range(4096) if centroid_smem(k, CENTROID_VEC) <= CENTROID_SMEM)    # 614
CENTROID_NCOLS_MAX = max(k for k in range(4096) if centroid_smem(k, 1) <= CENTROID_SMEM)              # 1075


def psi_width(dtype):
    """samples per thread of the vector PSI route: one 16-byte load"""
    return 16 // ELEM_SIZE[np.dtype(dtype).name]


def psi_route(n, dtype, aligned=True):
    """V of pb_psi: the vector width when every frame and output is 16-byte aligned and n is a multiple of it, else 1"""
    v = psi_width(dtype)
    return v if aligned and n % v == 0 else 1


# ---- edge lists ----------------------------------------------------------------------------------------------------
OVERLAP_N = (1, 4095, 4096, 4097, 1024 ** 2, 1024 ** 2 + 1, 2048 ** 2)
OVERLAP_P = (1, 7, 8, 9, 255, 256, 257, 513)
LP_P = (1, 64, 65, 129)
PSI_FRAMES = (1, 13, 64)
PSI_TYPES = ('float32', 'float64', 'uint16', 'int32')
CENTROID_W = tuple(sorted({THREADS * v + d for v in (1, CENTROID_VEC) for d in (-1, 0, 1)} | {4096}))
CENTROID_NCOLS = (CENTROID_NCOLS_V4, CENTROID_NCOLS_V4 + 1, CENTROID_NCOLS_MAX, CENTROID_NCOLS_MAX + 1)
CENTROID_TYPES = ('float32', 'float64', 'uint16', 'int32')
RECON_M = (1, 255, 256, 257, 8192)
RECON_K = (1, 10, 300)
RECON_F = (1, 16, GRID_Y_MAX)
BESSEL_ORDERS = (0, 1, 2, 3, 5, 8, 13, 20, 30, 40, 60)


def overlap_cases():
    """(n, P) pairs: every n with a few P, every P with a small and a chunk-crossing n; the product stays below 2^27
    samples so that a case fits a test's time"""
    out = []
    for n in OVERLAP_N:
        for P in (1, 9) if n > 4097 else (1, 8, 9):
            out.append((n, P))
    for P in OVERLAP_P:
        for n in (4097, 3 * OVERLAP_CHUNK + 5):
            if (n, P) not in out:
                out.append((n, P))
    return out


# ---- coupling ------------------------------------------------------------------------------------------------------
def overlap_ref(E, modes):
    """eta_p = |sum conj(M_p) E|^2 / (I_p I_E) in long double, the Cauchy-Schwarz majorant (sum|M_p||E|)^2 / (I_p I_E)
    of its error scale (<= 1), and I_p, I_E.  E (n,), modes (P, n), real or complex."""
    E = np.asarray(E).reshape(-1)
    M = np.asarray(modes).reshape(len(modes), -1)
    ie, ip, ov, am = LDBL(0), np.zeros(len(M), LDBL), np.zeros(len(M), np.clongdouble), np.zeros(len(M), LDBL)
    for k0 in range(0, E.size, 1 << 18):                   # blocks keep the long-double copies small
        e = E[k0:k0 + (1 << 18)].astype(np.clongdouble)
        m = M[:, k0:k0 + (1 << 18)]
        m = m.astype(np.clongdouble if np.iscomplexobj(m) else LDBL)
        ie += np.sum(e.real * e.real + e.imag * e.imag)
        ip += np.sum(m.real * m.real + m.imag * m.imag, axis=1)
        ov += np.conj(m) @ e
        am += np.abs(m) @ np.abs(e)
    eta = (ov.real ** 2 + ov.imag ** 2) / (ip * ie)
    return eta, am ** 2 / (ip * ie), ip, ie


def coupling_c_ref(eta0, ie):
    """SRI's c = (I_E eta_0)^(1/2)"""
    return np.sqrt(LDBL(ie) * LDBL(eta0))


def overlap_model(E, modes, defect=None):
    """the device's two-stage reduction in numpy fp64 (chunk partials, then a sum of the partials), or with one fault:
    'f32' (every sum in float32), 'drop_last_chunk', 'stage2_256' (stage 2 reads only the first 256 chunks),
    'e_twice' (every stage-1 launch after the first adds |E|^2 again)"""
    acc = np.float32 if defect == 'f32' else np.float64
    e = np.asarray(E).reshape(-1)
    m = np.asarray(modes).reshape(len(modes), -1)
    n, P = e.size, m.shape[0]
    nch = overlap_chunks(n)
    if defect == 'drop_last_chunk' and nch > 1:
        nch -= 1
    part = np.zeros((P, nch, 3), acc)
    part_e = np.zeros(nch, acc)
    for k in range(nch):
        sl = slice(k * OVERLAP_CHUNK, min(n, (k + 1) * OVERLAP_CHUNK))
        ec = e[sl].astype(np.complex64 if acc is np.float32 else np.complex128)
        mc = m[:, sl].astype(ec.dtype)
        ov = np.conj(mc) @ ec
        part[:, k, 0], part[:, k, 1] = ov.real, ov.imag
        part[:, k, 2] = np.sum(np.abs(mc) ** 2, axis=1, dtype=acc)
        part_e[k] = np.sum(np.abs(ec) ** 2, dtype=acc)
    if defect == 'e_twice':
        part_e = part_e * (1 + (P - 1) // OV_MAX)
    k2 = min(nch, THREADS) if defect == 'stage2_256' else nch
    t = part[:, :k2].sum(axis=1, dtype=acc)
    ie = part_e[:k2].sum(dtype=acc)
    return (t[:, 0] ** 2 + t[:, 1] ** 2) / (t[:, 2] * ie)


def overlap_fig(got, eta, maj):
    """max_p |eta_got - eta_ref| / majorant_p"""
    return float(np.max(np.abs(np.asarray(got, LDBL) - eta) / maj))


# ---- combine and grating -------------------------------------------------------------------------------------------
def combine_ref(a, alpha, b=None, beta=0.0, real_out=False):
    """alpha a + beta b (or its |.|^2) in long double from the values handed to the device"""
    z = np.asarray(a).astype(np.clongdouble) * np.clongdouble(alpha)
    if b is not None:
        z = z + np.asarray(b).astype(np.clongdouble) * np.clongdouble(beta)
    return z.real ** 2 + z.imag ** 2 if real_out else z


def grating_rect_ref(x, shift, period, edge, hi, lo, mid, eps):
    """pb_grating's rectangle: np.mod(x + shift, period) of the same fp64 values, hi below edge else lo, mid within
    eps of 0"""
    xw = np.mod(np.asarray(x, np.float64) + np.float64(shift), np.float64(period))
    g = np.where(xw < edge, hi, lo)
    return np.where(np.abs(xw) < eps, mid, g).astype(np.float64)


def grating_sin_ref(x, shift, prefix):
    xv = np.asarray(x, np.float64).astype(LDBL) + LDBL(shift)
    return 1 - (np.sin(LDBL(prefix) * xv) + 1) / 2 * LDBL(0.1)


# ---- PSI -----------------------------------------------------------------------------------------------------------
def psi_ref(frames, s, c):
    """(num, den, sum|s g|, sum|c g|) in long double; frames (N, n)"""
    g = np.asarray(frames).reshape(len(frames), -1).astype(LDBL)
    ws, wc = np.asarray(s, LDBL)[:, None], np.asarray(c, LDBL)[:, None]
    return (ws * g).sum(0), (wc * g).sum(0), np.abs(ws * g).sum(0), np.abs(wc * g).sum(0)


def psi_int_ref(frames, s, c):
    """exact int64 sums of integer frames with integer weights (the caller keeps them inside int64)"""
    g = np.asarray(frames).reshape(len(frames), -1).astype(np.int64)
    ws = np.asarray(s, np.float64).astype(np.int64)[:, None]
    wc = np.asarray(c, np.float64).astype(np.int64)[:, None]
    return (ws * g).sum(0), (wc * g).sum(0)


def psi_int_model(frames, s, c, defect=None):
    """the device's int64 accumulation, or with 'f64' the same sums accumulated in fp64"""
    if defect != 'f64':
        return psi_int_ref(frames, s, c)
    g = np.asarray(frames).reshape(len(frames), -1).astype(np.float64)
    ns = np.zeros(g.shape[1])
    nc = np.zeros(g.shape[1])
    for k in range(len(g)):
        ns += s[k] * g[k]
        nc += c[k] * g[k]
    return ns.astype(np.int64), nc.astype(np.int64)


def fringes(N, n, phase, dtype, amp=1.0, bias=2.0):
    """N phase-shifted frames bias + amp cos(phase - 2 pi k / N) of (n,) samples and their (s, c) weights, whose
    num / den recover phase: sum sin(d_k) g_k / sum cos(d_k) g_k"""
    d = 2 * np.pi * np.arange(N) / N
    g = bias + amp * np.cos(np.asarray(phase)[None, :] - d[:, None])
    return g.astype(dtype), np.sin(d), np.cos(d)


# ---- LP mode fields ------------------------------------------------------------------------------------------------
def bessel_j_model(l, x, defect=None):
    """the device's J_l(x) (csrc/wfs.cu bessel_j) in numpy fp64 with scipy's j0 / j1, or with 'forward_below' the
    forward recurrence used below x = l as well"""
    if l == 0:
        return float(sps.j0(x))
    if l == 1:
        return float(sps.j1(x))
    if x < 1e-20:
        t = 1.0
        for k in range(1, l + 1):
            t *= 0.5 * x / k
        return t
    tox = 2.0 / x
    if x > l or defect == 'forward_below':
        bjm, bj = float(sps.j0(x)), float(sps.j1(x))
        for j in range(1, l):
            bjm, bj = bj, j * tox * bj - bjm
        return bj
    m = 2 * ((l + 24 + int(math.sqrt(400.0 * l))) // 2)
    bjp, bj, s, ans, even = 0.0, 1.0, 0.0, 0.0, False
    for j in range(m, 0, -1):
        bjp, bj = bj, j * tox * bj - bjp
        if abs(bj) > 1e100:
            bj, bjp, ans, s = bj * 1e-100, bjp * 1e-100, ans * 1e-100, s * 1e-100
        if even:
            s += bj
        even = not even
        if j == l:
            ans = bjp
    return ans / (2.0 * s - bj)


def lp_model(cases, defect=None):
    """the J ratios of `cases` ((l, U, rho) rows) from bessel_j_model, with one plan per row: 'offset0' writes the
    modes past the first launch over the first launch's (the second launch at out + 0 instead of out + p0 n),
    'forward_below' uses the forward recurrence below x = l"""
    jdef = defect if defect == 'forward_below' else None
    vals = np.array([bessel_j_model(int(l), U * r, jdef) / bessel_j_model(int(l), U, jdef) for l, U, r in cases])
    if defect == 'offset0' and len(vals) > LP_MAX:
        out = vals.copy()
        for p0 in range(LP_MAX, len(vals), LP_MAX):
            k = min(LP_MAX, len(vals) - p0)
            out[:k] = vals[p0:p0 + k]
        return out
    return vals


BESSEL_FIXTURE = 'wfs_bessel.npz'


def bessel_cases():
    """the (kind, l, U or W, rho) rows of the Bessel fixture: kind 0 is the core ratio J_l(U rho) / J_l(U), kind 1 the
    cladding ratio K_l(W rho) / K_l(W).  a = 1 on the device, so rho is the radius itself."""
    rows = []
    for l in BESSEL_ORDERS:
        for U in (0.7, 2.4, 5.1, 11.3, 37.9, 100.0):
            if abs(sps.jv(l, U)) < 1e-3 * max(1e-300, np.abs(sps.jv(l, np.linspace(0, U, 200))).max()):
                continue                                   # a zero of J_l near U: the ratio is ill-posed
            for rho in np.concatenate((np.linspace(0, 1, 33), [1e-90 / U, 1e-40 / U, 1e-8 / U])):
                rows.append((0, l, U, rho))
            if l >= 2 and U > l + 1:                       # dense within +-1 of x = l, where the J route switches
                for x in np.concatenate((np.linspace(l - 1, l + 1, 41), l * (1 + np.array([-4, -1, 1, 4]) * 2.0 ** -52))):
                    rows.append((0, l, U, x / U))
        for Wv in (1e-3, 0.05, 1.0, 2.0, 7.5, 60.0):
            for rho in (1.0, 1.0 + 2.0 ** -40, 1.001, 1.1, 1.5, 2.0, 3.0, 5.0, 10.0):
                rows.append((1, l, Wv, rho))
    r = np.array(rows, dtype=np.float64)
    return r[:, 0].astype(np.int32), r[:, 1].astype(np.int32), r[:, 2], r[:, 3]


def write_bessel_fixture(golden_dir, digits=40):
    """compute the fixture with mpmath and write it as wfs_bessel.npz (+ .partN.npz, each below 1 MB)"""
    import mpmath
    mpmath.mp.dps = digits
    kind, l, arg, rho = bessel_cases()
    val = np.empty(len(kind))
    for i in range(len(kind)):
        a, r, n = mpmath.mpf(float(arg[i])), mpmath.mpf(float(rho[i])), int(l[i])
        if kind[i] == 0:
            val[i] = float(mpmath.besselj(n, a * r) / mpmath.besselj(n, a))
        else:
            val[i] = float(mpmath.besselk(n, a * r) / mpmath.besselk(n, a))
    arrays = {'kind': kind, 'l': l, 'arg': arg, 'rho': rho, 'val': val}
    parts, cur, size = [], {}, 0
    for k, v in arrays.items():
        if cur and size + v.nbytes > 900_000:
            parts.append(cur)
            cur, size = {}, 0
        cur[k] = v
        size += v.nbytes
    parts.append(cur)
    for i, p in enumerate(parts):
        name = BESSEL_FIXTURE if i == 0 else BESSEL_FIXTURE.replace('.npz', f'.part{i + 1}.npz')
        np.savez_compressed(os.path.join(golden_dir, name), **p)


def mp_ratio(kind, l, arg, rho, digits=40):
    import mpmath
    mpmath.mp.dps = digits
    a, r = mpmath.mpf(float(arg)), mpmath.mpf(float(rho))
    f = mpmath.besselj if kind == 0 else mpmath.besselk
    return float(f(int(l), a * r) / f(int(l), a))


# ---- centroids -----------------------------------------------------------------------------------------------------
def centres(pitch, n):
    """lenslet centres along one axis, as shack_hartmann places them (no shift)"""
    return np.arange(-(n // 2), -(n // 2) + n, dtype=np.float64) * pitch


def owners(coords, c, pitch):
    """owner lenslet of each coordinate under half-open [c - pitch/2, c + pitch/2) in fp64, lowest index first, -1 for
    none"""
    own = np.full(len(coords), -1)
    for i in range(len(c) - 1, -1, -1):
        lo, hi = c[i] - pitch / 2, c[i] + pitch / 2
        own[(lo <= coords) & (coords < hi)] = i
    return own


def centroid_ref(frames, xv, yv, xc, yc, pitch, threshold=0.0):
    """(disp (F, 2, ny, nx), flux (F, ny, nx), scale (2, ny, nx)) in long double by the spot_centroids definition:
    w = max(I - t max I, 0) over each subaperture's owned samples, disp = (sum w x / sum w - xc, sum w y / sum w - yc),
    NaN where sum w = 0 (or for no owned sample), NaN propagating; scale is max|x - xc| (max|y - yc|) over the
    subaperture, the unit of the displacement figure"""
    F = frames.shape[0]
    ox, oy = owners(xv, xc, pitch), owners(yv, yc, pitch)
    nx, ny = len(xc), len(yc)
    disp = np.full((F, 2, ny, nx), np.nan, LDBL)
    flux = np.zeros((F, ny, nx), LDBL)
    scale = np.ones((2, ny, nx))
    for j in range(ny):
        rows = np.flatnonzero(oy == j)
        for i in range(nx):
            cols = np.flatnonzero(ox == i)
            if rows.size == 0 or cols.size == 0:
                continue
            xs, ys = xv[cols].astype(LDBL), yv[rows].astype(LDBL)
            scale[0, j, i] = float(np.max(np.abs(xv[cols] - xc[i]))) or 1.0
            scale[1, j, i] = float(np.max(np.abs(yv[rows] - yc[j]))) or 1.0
            for f in range(F):
                I = frames[f][np.ix_(rows, cols)].astype(LDBL)
                flux[f, j, i] = I.sum()
                t = LDBL(threshold) * I.max() if threshold != 0.0 else LDBL(0)
                w = np.maximum(I - t, 0)
                sw = w.sum()
                if sw != 0 or np.isnan(sw):
                    disp[f, 0, j, i] = (w * xs[None, :]).sum() / sw - LDBL(xc[i])
                    disp[f, 1, j, i] = (w * ys[:, None]).sum() / sw - LDBL(yc[j])
    return disp, flux, scale


def centroid_model(frames, xv, yv, xc, yc, pitch, V, defect=None):
    """the device's chunked column reduction in numpy fp64 for threshold 0: column sums, then each lenslet summed in
    column order across chunks of 256 V columns; 'straddle' counts a lenslet that straddles a chunk boundary only in
    the chunk where it starts"""
    F = frames.shape[0]
    ox, oy = owners(xv, xc, pitch), owners(yv, yc, pitch)
    CC = THREADS * V
    disp = np.full((F, 2, len(yc), len(xc)), np.nan)
    for j in range(len(yc)):
        rows = np.flatnonzero(oy == j)
        for i in range(len(xc)):
            cols = np.flatnonzero(ox == i)
            if rows.size == 0 or cols.size == 0:
                continue
            if defect == 'straddle':
                cols = cols[cols // CC == cols[0] // CC]
            for f in range(F):
                I = frames[f][np.ix_(rows, cols)].astype(np.float64)
                cw = I.sum(0)
                cwy = (I * yv[rows][:, None]).sum(0)
                sw = swx = swy = 0.0
                for k in range(len(cols)):
                    sw += cw[k]
                    swx += cw[k] * xv[cols[k]]
                    swy += cwy[k]
                if sw != 0:
                    disp[f, 0, j, i] = swx / sw - xc[i]
                    disp[f, 1, j, i] = swy / sw - yc[j]
    return disp


def centroid_fig(got, disp, scale):
    """max |got - ref| / scale over the subapertures where the reference is finite"""
    ok = np.isfinite(disp)
    d = np.abs(np.asarray(got, LDBL) - disp) / scale[None]
    return float(np.max(d[ok])) if ok.any() else 0.0


# ---- reconstruction ------------------------------------------------------------------------------------------------
def reconstruct_ref(slopes, idx, ref, R):
    """out[f, k] = sum_m R[k, m] (slopes[f].flat[idx[m]] - ref[m]) and sum_m |R[k, m] (s - ref)| in long double"""
    s = np.asarray(slopes).reshape(len(slopes), -1)[:, idx].astype(LDBL)
    if ref is not None:
        s = s - np.asarray(ref, LDBL)[None]
    RL = np.asarray(R, LDBL)
    return s @ RL.T, np.abs(s) @ np.abs(RL).T


def reconstruct_model(slopes, idx, ref, R, defect=None):
    """fp64 GEMV, or with 'gather_m' the slope read at m instead of idx[m]"""
    s = np.asarray(slopes, np.float64).reshape(len(slopes), -1)
    g = s[:, np.arange(len(idx))] if defect == 'gather_m' else s[:, idx]
    if ref is not None:
        g = g - ref[None]
    return g @ np.asarray(R, np.float64).T


# ---- lenslet screen ------------------------------------------------------------------------------------------------
def lenslet_phase(x, y, pitch, n, efl, aperture='rectangle', dtype=np.float64):
    """the reference's loop over lenslets restated in numpy (DESIGN 4.14): lenslet (j, i) takes the window
    [c + int(centre / dx) - spl, ... + 2 spl) per axis, clamped, with spl = int(pitch / dx + 1) and c = ceil(size / 2),
    masks rsq / (2 efl) with the aperture and adds it into an accumulator of the storage dtype, row j outer and column
    i inner.  The centres and dx have the storage dtype; the arithmetic on a sample is fp64 (as on the device and, at
    fp64, in the reference), rounded to the storage dtype after each addition."""
    H, W = x.shape
    nr, nc = n
    xc = np.arange(-(nc // 2), -(nc // 2) + nc, dtype=dtype) * dtype(pitch)
    yc = np.arange(-(nr // 2), -(nr // 2) + nr, dtype=dtype) * dtype(pitch)
    dx = x[0, 1] - x[0, 0]
    spl = int(dtype(pitch) / dx + 1)
    cx, cy = math.ceil(W / 2), math.ceil(H / 2)
    x64, y64 = x.astype(np.float64), y.astype(np.float64)
    total = np.zeros((H, W), dtype)
    half = np.float64(pitch / 2)
    for j in range(nr):
        y0 = cy + int(yc[j] / dx) - spl
        rs = slice(min(max(y0, 0), H), min(max(y0 + 2 * spl, 0), H))
        for i in range(nc):
            x0 = cx + int(xc[i] / dx) - spl
            cs = slice(min(max(x0, 0), W), min(max(x0 + 2 * spl, 0), W))
            lx = x64[rs, cs] - np.float64(xc[i])
            ly = y64[rs, cs] - np.float64(yc[j])
            rsq = lx * lx + ly * ly
            if aperture == 'rectangle':
                m = (np.abs(lx) <= half) & (np.abs(ly) <= half)
            else:
                m = rsq <= half * half
            t = total[rs, cs]
            total[rs, cs] = np.where(m, (t.astype(np.float64) + rsq / (2 * np.float64(efl))).astype(dtype), t)
    return total


def lenslet_field_ref(total, kphase):
    """exp(i p) in long double of p = kphase * total rounded to fp64, as the device forms the product"""
    p = (np.float64(kphase) * total.astype(np.float64)).astype(LDBL)
    return np.cos(p), np.sin(p)
