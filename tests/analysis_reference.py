"""Plain high-precision references, launch rules and defect models of the PSF / MTF analysis kernels of
csrc/analysis.cu: the linear interpolator (points and polar lattice), the azimuthal statistics, the polar crossings of
estimate_size and the analytic radial functions.

References are written from the documented definitions (the header comment of analysis.cu and include/prysm_b200.h,
scipy's RegularGridInterpolator(method='linear'), numpy's nan* statistics, the estimate_size loop), not from the
engine's host code.  Values are in long double (80-bit on x86-64) and come with a majorant of their error scale.  The
Bessel and Airy values are a committed fixture (tests/golden/analysis_bessel.npz) written at 60 digits with mpmath by
`write_bessel_fixture`; nothing else here imports mpmath.

The `*_model` functions (numpy versions of a kernel, optionally with one deliberate fault) are used by
tests/test_host_analysis_reference.py only, to show that the GPU test's ceilings would catch each fault.
"""
import os

import numpy as np

from accuracy import LDBL, grid_for, sweep  # noqa: F401

EPS = np.finfo(np.float64).eps

# ---- launch rules (mirrors of csrc/analysis.cu and csrc/common.cuh) ------------------------------------------------
AN_THREADS = 256                # AN_THREADS: threads of every analysis block
AZ_MAX_NY = 28672               # PB_AZ_MAX_NY: phi samples of one column held in shared memory
AZ_LAUNCHES = 1                 # pb_azimuthal_stats: one launch whatever the mask
INTERP_LAUNCHES = 1
ANALYTIC_LAUNCHES = 1


def sweep_counts(sm_count):
    c = sweep(sm_count)
    return (1, c - 1, c, c + 1, 3 * c)


def chunk_len(nx):
    """samples each thread of crossing_kernel scans: L = ceil((nx - 1) / 256)"""
    return -(-(nx - 1) // AN_THREADS)


def crossing_launches(relative):
    """pb_polar_crossings: [row maxima,] level, crossings, mean"""
    return 4 if relative else 3


# ---- the interpolator ------------------------------------------------------------------------------------------------
def _axis_weights(ax, p):
    """(i, j, t) of every point: interval i = the largest index with ax[i] <= p clipped to [0, n - 2], j = i + 1 (or i
    for one sample), t = (p - ax[i]) / (ax[j] - ax[i]) in long double (0 for one sample)"""
    ax = np.asarray(ax, np.float64)
    n = ax.size
    if n < 2:
        z = np.zeros(p.shape, np.int64)
        return z, z, np.zeros(p.shape, LDBL)
    i = np.clip(np.searchsorted(ax, p, side='right') - 1, 0, n - 2)
    j = i + 1
    a0, a1 = ax[i].astype(LDBL), ax[j].astype(LDBL)
    return i, j, (p.astype(LDBL) - a0) / (a1 - a0)


def interp_ref(data, xax, yax, px, py, fill=0.0, defect=None):
    """RegularGridInterpolator(method='linear', bounds_error=False, fill_value=fill) of real (ny, nx) data at the fp64
    points (px, py), in long double: (value, majorant); eps times the majorant is the error scale.  The majorant is
    sum |corner weight| plus each corner's magnitude times the rounding of its fp64 weights (so a corner of weight ~0
    still carries a few eps of its value).  A NaN corner gives NaN whatever its weight.  defect: 'lt' (the interval is the largest i with ax[i] < p),
    'skip_zero' (a corner of weight 0 is skipped, so its NaN is lost)."""
    d = np.asarray(data)
    xax, yax = np.asarray(xax, np.float64), np.asarray(yax, np.float64)
    px, py = np.asarray(px, np.float64), np.asarray(py, np.float64)
    shape = np.broadcast(px, py).shape
    px, py = np.broadcast_to(px, shape).reshape(-1), np.broadcast_to(py, shape).reshape(-1)
    if defect == 'lt':
        ix = np.clip(np.searchsorted(xax, px, side='left') - 1, 0, max(xax.size - 2, 0))
        iy = np.clip(np.searchsorted(yax, py, side='left') - 1, 0, max(yax.size - 2, 0))
        jx = ix + (xax.size > 1)
        jy = iy + (yax.size > 1)
        tx = (px.astype(LDBL) - xax[ix]) / (xax[jx].astype(LDBL) - xax[ix]) if xax.size > 1 else np.zeros(px.shape, LDBL)
        ty = (py.astype(LDBL) - yax[iy]) / (yax[jy].astype(LDBL) - yax[iy]) if yax.size > 1 else np.zeros(py.shape, LDBL)
    else:
        ix, jx, tx = _axis_weights(xax, px)
        iy, jy, ty = _axis_weights(yax, py)
    ux, uy = 1 - tx, 1 - ty
    # the device's weights carry (|p| + |ax_i|) / h eps of rounding from p - ax_i, and an eps from each product
    ex = 2 + (np.abs(px) + np.abs(xax[ix])) / (xax[jx] - xax[ix]) if xax.size > 1 else np.zeros(px.shape)
    ey = 2 + (np.abs(py) + np.abs(yax[iy])) / (yax[jy] - yax[iy]) if yax.size > 1 else np.zeros(py.shape)
    wf = (ex + ey + 3).astype(LDBL)
    corners = ((iy, ix, uy * ux), (iy, jx, uy * tx), (jy, ix, ty * ux), (jy, jx, ty * tx))
    val = np.zeros(px.shape, LDBL)
    maj = np.zeros(px.shape, LDBL)
    for r, c, w in corners:
        v = d[r, c].astype(LDBL)
        term = v * w
        if defect == 'skip_zero':
            term = np.where(w == 0, 0, term)
        val = val + term
        maj = maj + np.abs(term) + np.where(np.isfinite(v), np.abs(v), 0) * wf
    maj = maj + LDBL(4 * 5e-324) / LDBL(EPS)      # the rounding unit of subnormal products
    inside = (py >= yax[0]) & (py <= yax[-1]) & (px >= xax[0]) & (px <= xax[-1])
    val = np.where(inside, val, LDBL(fill))
    maj = np.where(inside, maj, 0)
    nan = np.isnan(px) | np.isnan(py)
    val = np.where(nan, LDBL(np.nan), val)
    return val.reshape(shape), maj.reshape(shape)


def interp_model(data, xax, yax, px, py, fill=0.0, defect=None):
    """the reference with one fault, rounded to fp64 (see interp_ref)"""
    return interp_ref(data, xax, yax, px, py, fill, defect)[0].astype(np.float64)


# ---- the polar lattice -----------------------------------------------------------------------------------------------
def lattice_axes(nx, ny, rmax):
    return np.linspace(0, rmax, nx), np.linspace(0, 2 * np.pi, ny)


def lattice_points(nx, ny, rmax, rows=None, cols=None):
    """(px, py, exact) of lattice rows x columns: x = fl64(rho fl64(cos phi)) with cos, sin taken in long double; exact
    where the coordinates do not depend on how sin and cos are rounded (phi = 0 or rho = 0)"""
    rho, phi = lattice_axes(nx, ny, rmax)
    rows = np.arange(ny) if rows is None else np.asarray(rows)
    cols = np.arange(nx) if cols is None else np.asarray(cols)
    p = phi[rows].astype(LDBL)
    c, s = np.cos(p).astype(np.float64), np.sin(p).astype(np.float64)
    r = rho[cols]
    px, py = r[None, :] * c[:, None], r[None, :] * s[:, None]
    exact = (phi[rows] == 0)[:, None] | (r == 0)[None, :]
    return px, py, exact


def _slope_term(data, xax, yax, px, py):
    """|difference of the corners along x| / dx times 2 ulp(px), and the matching y term: what a 1-ulp different
    cos or sin (and the rounding of the product after it) can move the interpolated value"""
    out = np.zeros(px.shape, LDBL)
    for ax, p, axis in ((xax, px, 1), (yax, py, 0)):
        if ax.size < 2:
            continue
        i, j, _ = _axis_weights(ax, p.reshape(-1))
        i, j = i.reshape(p.shape), j.reshape(p.shape)
        ox, oy = _axis_weights(yax if axis == 1 else xax, (py if axis == 1 else px).reshape(-1))[:2]
        ox, oy = ox.reshape(p.shape), oy.reshape(p.shape)
        d = np.asarray(data)
        if axis == 1:
            dd = np.maximum(np.abs(d[ox, j].astype(LDBL) - d[ox, i]), np.abs(d[oy, j].astype(LDBL) - d[oy, i]))
        else:
            dd = np.maximum(np.abs(d[j, ox].astype(LDBL) - d[i, ox]), np.abs(d[j, oy].astype(LDBL) - d[i, oy]))
        h = (ax[j] - ax[i]).astype(LDBL)
        out = out + np.where(np.isfinite(dd), dd, 0) / h * LDBL(2) * np.spacing(np.abs(p)).astype(LDBL)
    return out


def lattice_ref(data, xax, yax, rmax, rows=None, cols=None):
    """the lattice values of rows x columns in long double: (value, majorant, ambiguous); eps times the majorant is
    the error scale.  The majorant adds what a 1-ulp different device sin / cos can move the value; `ambiguous` marks points whose coordinate lies within 4 ulps
    of a node across which the value changes NaN-ness, or of an axis end where the data does not fade to the fill
    value (there the device may decide otherwise)."""
    xax, yax = np.asarray(xax, np.float64), np.asarray(yax, np.float64)
    nx, ny = data.shape[1], data.shape[0]
    px, py, exact = lattice_points(nx, ny, rmax, rows, cols)
    val, maj = interp_ref(data, xax, yax, px, py, 0.0)
    maj = maj + np.where(exact, 0, _slope_term(data, xax, yax, px, py) / LDBL(EPS))
    amb = np.zeros(px.shape, bool)
    for k in (-4, 4):
        for qx, qy in ((px + k * np.spacing(np.abs(px)), py), (px, py + k * np.spacing(np.abs(py)))):
            v2, _ = interp_ref(data, xax, yax, qx, qy, 0.0)
            inside = (qy >= yax[0]) & (qy <= yax[-1]) & (qx >= xax[0]) & (qx <= xax[-1])
            inside0 = (py >= yax[0]) & (py <= yax[-1]) & (px >= xax[0]) & (px <= xax[-1])
            # leaving the axes changes nothing where the data fades to the fill value at the border
            jump = np.abs(np.where(np.isnan(v2) | np.isnan(val), 0, v2 - val)) > 4 * LDBL(EPS) * maj
            amb |= (np.isnan(v2) != np.isnan(val)) | ((inside != inside0) & jump)
    amb &= ~exact
    return val, maj, amb


# ---- azimuthal statistics --------------------------------------------------------------------------------------------
def azstats_ref(col):
    """count, mean, variance (ddof 0, two passes), min, max, median of one column in long double, NaN ignored; the
    median is the mean of the two middle values for an even count.  NaN everywhere for an empty column."""
    v = np.asarray(col, LDBL)
    v = v[~np.isnan(v)]
    n = v.size
    if n == 0:
        return dict(count=0, mean=np.nan, var=np.nan, min=np.nan, max=np.nan, median=np.nan)
    m = v.sum() / n
    s = np.sort(v)
    med = s[n // 2] if n % 2 else (s[n // 2 - 1] + s[n // 2]) / 2
    return dict(count=n, mean=m, var=((v - m) ** 2).sum() / n, min=s[0], max=s[-1], median=med)


def azstats_scales(col, maj):
    """the error scale of each statistic: mean over (n / 256 + 8) sum majorant / count (>= sum |v| / count, times the
    length of the device's summation chains), variance over var +
    2 mean-majorant eps sqrt(var) (+ the square of the mean's own rounding, (n / 256 + 8) eps mean-majorant, over eps: a column of equal values), min, max and median over the column's largest majorant"""
    v = np.asarray(col, LDBL)
    ok = ~np.isnan(v)
    n = int(ok.sum())
    if n == 0:
        return None
    mj = np.asarray(maj, LDBL)[ok]
    r = azstats_ref(col)
    am = mj.sum() / n
    big = mj.max()
    big = big if big > 0 else LDBL(np.finfo(np.float64).tiny)
    K = LDBL(n / AN_THREADS + 8)                  # strided partials, then the warp and block trees
    return dict(mean=(am if am > 0 else big) * K, var=r['var'] + 2 * am * LDBL(EPS) * np.sqrt(r['var']) + am * am * LDBL(EPS) * K ** 2,
                min=big, max=big, median=big)


def azstats_model(col, defect=None):
    """the kernel's column statistics in numpy on fp64 lattice values, or with one fault: 'one_pass' (E[v^2] - mean^2),
    'upper_median' (an even count takes the upper middle value), 'nan_rank' (the median's rank counts NaNs),
    'f32_sums' (the column sums accumulated in float32)"""
    v = np.asarray(col, np.float64)
    ok = ~np.isnan(v)
    x = v[ok]
    n = x.size
    if n == 0:
        return dict(count=0, mean=np.nan, var=np.nan, min=np.nan, max=np.nan, median=np.nan)
    acc = np.float32 if defect == 'f32_sums' else np.float64

    def colsum(vals):                    # per-thread strided partials, then the partials in order
        part = np.zeros(AN_THREADS, acc)
        for i0 in range(0, vals.size, AN_THREADS):
            blk = vals[i0:i0 + AN_THREADS].astype(acc)
            part[:blk.size] = (part[:blk.size] + blk).astype(acc)
        tot = acc(0)
        for p in part:
            tot = acc(tot + p)
        return np.float64(tot)
    m = colsum(x) / n
    if defect == 'one_pass':
        var = np.sum(x * x) / n - m * m
    else:
        var = colsum((x - m) ** 2) / n
    srt = np.sort(v)                     # NaN last, as the order keys put it
    if defect == 'nan_rank':
        nn = v.size
        med = srt[nn // 2] if nn % 2 else (srt[nn // 2 - 1] + srt[nn // 2]) / 2
    elif n % 2:
        med = srt[n // 2]
    else:
        med = srt[n // 2] if defect == 'upper_median' else (srt[n // 2 - 1] + srt[n // 2]) / 2
    return dict(count=n, mean=m, var=var, min=x.min(), max=x.max(), median=med)


# ---- crossings ------------------------------------------------------------------------------------------------------
def crossings_ref(vals, maj, rho, t, last, extra=0, exact=None):
    """estimate_size's loop over the lattice rows (vals (ny, nx) in long double): each row's first or last i with
    (v[i] > t) != (v[i + 1] > t) gives rho_i + frac (rho_{i+1} - rho_i), frac = (t - v_i) / (v_{i+1} - v_i), 0 where
    they are equal.  Returns (count, mean, radii, flagged): the count of rows that cross, the long-double mean (NaN when
    a chosen crossing touches a NaN sample), the radius of every row (+inf for none) and the rows where a lattice value
    lies within 8 eps majorant (plus `extra`, the level's own error) of t, where a device comparison could flip; points
    with `exact` coordinates (an exact tie built on the phi = 0 ray) are not flagged."""
    vals = np.asarray(vals, LDBL)
    rho = np.asarray(rho, np.float64).astype(LDBL)
    t = LDBL(t)
    rad = np.full(vals.shape[0], np.inf, LDBL)
    tol = 8 * LDBL(EPS) * np.asarray(maj, LDBL) + LDBL(extra) + abs(t) * LDBL(EPS)
    near = np.abs(vals - t) <= tol
    if exact is not None:
        near &= ~exact
    flagged = np.any(near, axis=1)
    for r, row in enumerate(vals):
        above = row > t
        idx = np.flatnonzero(above[:-1] != above[1:])
        if idx.size == 0:
            continue
        i = int(idx[-1] if last else idx[0])
        y0, y1 = row[i], row[i + 1]
        frac = LDBL(0) if y1 == y0 else (t - y0) / (y1 - y0)
        rad[r] = rho[i] + frac * (rho[i + 1] - rho[i])
    hit = rad != np.inf
    count = int(hit.sum())
    mean = rad[hit].sum() / count if count else LDBL(np.nan)
    return count, mean, rad, flagged


def crossings_model(vals, rho, t, last, defect=None):
    """the kernel's chunked scan on fp64 lattice values: thread k scans pairs [kL, min((k+1)L, n-1)), the block takes
    the min (first) or max (last) pair index, and the mean counts every row that crossed.  Faults: 'drop_shared' (each
    chunk's scan drops its shared end sample, so its last pair), 'swap' (first takes the max over chunks and last the
    min), 'nan_drop' (NaN radii leave the count and the sum, the parent's rule)."""
    v = np.asarray(vals, np.float64)
    ny, n = v.shape
    L = chunk_len(n)
    rad = np.full(ny, np.inf)
    for r in range(ny):
        found = []
        for k in range(AN_THREADS):
            j0, j1 = k * L, min(k * L + L, n - 1)
            if defect == 'drop_shared':
                j1 -= 1
            hits = [j for j in range(j0, j1) if (v[r, j] > t) != (v[r, j + 1] > t)]
            if hits:
                found.append(hits[-1] if last else hits[0])
        if not found:
            continue
        pick_max = last != (defect == 'swap')
        i = max(found) if pick_max else min(found)
        y0, y1 = v[r, i], v[r, i + 1]
        frac = 0.0 if y1 == y0 else (t - y0) / (y1 - y0)
        rad[r] = rho[i] + frac * (rho[i + 1] - rho[i])
    hit = rad != np.inf
    if defect == 'nan_drop':
        hit &= ~np.isnan(rad)
    count = int(hit.sum())
    return count, (rad[hit].sum() / count if count else np.nan)


def crossing_fig(got_count, got_mean, count, mean, rmax):
    """|mean_got - mean_ref| / rmax, infinite when the counts or the NaN-ness differ"""
    if got_count != count or np.isnan(got_mean) != np.isnan(float(mean)):
        return np.inf
    if np.isnan(got_mean):
        return 0.0
    return float(abs(LDBL(got_mean) - mean) / LDBL(rmax))


# ---- analytic functions ----------------------------------------------------------------------------------------------
BESSEL_FIXTURE = 'analysis_bessel.npz'
JINC_THRESHOLD = 1e-8


def bessel_points():
    """u of the fixture: log-spaced 1e-12 .. 2e4, +-2 ulps around the first 30 zeros of J1, both sides of the jinc
    threshold; s of difflim_core: 1 - 2^-k for k = 1..52, 1, nextafter(1, 2), a uniform grid and small s"""
    import scipy.special as sps
    u = [np.logspace(-12, np.log10(2e4), 4000)]
    for z in sps.jn_zeros(1, 30):
        u.append(np.array([z + k * np.spacing(z) for k in range(-2, 3)]))
    th = JINC_THRESHOLD
    u.append(np.array([np.nextafter(th, 0), th, np.nextafter(th, 1), 0.5 * th, 2 * th, 1e-4, 3e-4, 1e-3]))
    u = np.unique(np.concatenate(u))
    s = np.concatenate((1 - 2.0 ** -np.arange(1, 53), [1.0, np.nextafter(1.0, 2.0)], np.linspace(0, 1, 1001)[1:-1],
                        [0.0, 1e-300, 1e-16, 1e-8, 1e-4]))
    return u, np.unique(s)


def write_bessel_fixture(golden_dir, digits=60):
    """the fixture with mpmath: j0(u), j1(u), 2 j1(u) / u, 1 - j0^2 - j1^2 at each u and difflim_core(s) at each s"""
    import mpmath
    mpmath.mp.dps = digits
    u, s = bessel_points()
    j0, j1, e, ee = (np.empty(u.size) for _ in range(4))
    for i, x in enumerate(u):
        m = mpmath.mpf(float(x))
        a, b = mpmath.besselj(0, m), mpmath.besselj(1, m)
        j0[i], j1[i], e[i], ee[i] = float(a), float(b), float(2 * b / m), float(1 - a * a - b * b)
    core = np.empty(s.size)
    for i, x in enumerate(s):
        m = mpmath.mpf(float(x))
        core[i] = float(2 / mpmath.pi * (mpmath.acos(min(m, 1)) - min(m, 1) * mpmath.sqrt(1 - min(m, 1) ** 2)))
    np.savez_compressed(os.path.join(golden_dir, BESSEL_FIXTURE), u=u, j0=j0, j1=j1, airy_e=e, ee=ee, s=s, core=core)


def analytic_scales(z):
    """the error scale of each function, in units of eps: |f| + |x f'(x)| (argument rounding and the cancellation near
    zeros and near s -> 1); for 1 - J0^2 - J1^2 also its terms' magnitude 2 (the formula itself cancels at small p),
    and for difflim_core also 1 / (2 sqrt(1 - s^2)), what the rounding of s * s moves sqrt(1 - s * s)"""
    u, j0, j1, e = z['u'], z['j0'], z['j1'], z['airy_e']
    ue = np.abs(2 * j0 - 2 * e)                               # u d/du (2 j1(u) / u) = 2 j0 - 4 j1 / u
    s = np.minimum(z['s'], 1.0)
    return dict(efield=np.abs(e) + ue, airy=e * e + 2 * np.abs(e) * ue, ee=np.abs(z['ee']) + 2 * j1 * j1 + 2,
                core=np.abs(z['core']) + 4 / np.pi * s * np.sqrt(1 - s * s) + np.spacing(np.abs(z['core'])) / EPS
                + np.where(s < 1, 0.5 / np.sqrt(np.where(s < 1, 1 - s * s, 1.0)), 0.0))


def jinc_model(u, defect=None):
    """2 jinc(u) as the kernel forms it with scipy's j1, or with one fault: 'threshold' (0.5 below 1e-4 instead of
    1e-8), 'asymptotic' (j1 from its leading large-argument form only)"""
    import scipy.special as sps
    u = np.asarray(u, np.float64)
    th = 1e-4 if defect == 'threshold' else JINC_THRESHOLD
    if defect == 'asymptotic':
        j1 = np.sqrt(2 / (np.pi * u)) * np.cos(u - 3 * np.pi / 4)
    else:
        j1 = sps.j1(u)
    with np.errstate(divide='ignore', invalid='ignore'):
        return 2 * np.where(np.abs(u) < th, 0.5, j1 / u)


def ee_model(p, defect=None):
    import scipy.special as sps
    j1 = np.sqrt(2 / (np.pi * p)) * np.cos(p - 3 * np.pi / 4) if defect == 'asymptotic' else sps.j1(p)
    j0 = sps.j0(p)
    return 1 - j0 * j0 - j1 * j1


def core_model(s):
    s = np.minimum(np.asarray(s, np.float64), 1.0)
    return 2 / np.pi * (np.arccos(s) - s * np.sqrt(1 - s * s))


def analytic_fig(got, ref, scale):
    """max |got - ref| / (eps scale), in units of eps"""
    return float(np.max(np.abs(np.asarray(got, np.float64).astype(LDBL) - ref) / (LDBL(EPS) * scale)))


# ---- the GPU cases (shared with the host test, which checks they stay unambiguous) ----------------------------------
POLAR_N = (1, 2, 255, 256, 257, 4097)
AZ_NY = (1, 255, 256, 257, 511, 512, 513, 4097, 28671, 28672)
CROSS_NX = (2, 3, 257, 258, 513, 4097, 20001)
RADIAL_NX = tuple(n for n in CROSS_NX if n > 3)   # 2 and 3 radii are the ray cases' (a ring needs samples)
METRICS = {'fwhm': (0.5, True), '1/e': (1 / np.e, True), '1/e^2': (1 / np.e ** 2, True), 'abs': (0.2, False)}


def offset_axis(n, frac, step):
    """n ascending samples, the origin at frac of the way along (a single sample is the origin)"""
    return (np.arange(n) - frac * (n - 1)) * step if n > 1 else np.zeros(1)


def zero_border(d):
    """the data fades to the fill value 0 at the axis ends, as a PSF does"""
    if d.shape[0] > 2:
        d[0], d[-1] = 0, 0
    if d.shape[1] > 2:
        d[:, 0], d[:, -1] = 0, 0
    return d


def rmax_of(xax, yax):
    return float(np.max(np.abs([xax[0], xax[-1], yax[0], yax[-1]])))


def polar_case(ny, nx):
    """(data, x, y, rmax, rows, cols) of a pb_interp2d_linear polar case: a smooth field with noise on offset axes, and
    the lattice rows and columns the test compares"""
    x, y = offset_axis(nx, 0.43, 1.0), offset_axis(ny, 0.61, 1.37 * max(nx, 2) / max(ny, 2))
    rng = np.random.default_rng(ny * 7919 + nx)
    r2 = (x[None, :] / max(nx, 2)) ** 2 + (y[:, None] / (1.37 * max(nx, 2))) ** 2
    d = zero_border(np.exp(-8 * r2) + 0.05 * rng.standard_normal((ny, nx)))
    rows = sorted({0, 1, ny // 3, ny // 2, ny - 2, ny - 1} & set(range(ny)))
    cols = sorted({0, 1, nx // 3, nx // 2, nx - 2, nx - 1} & set(range(nx)))
    return d, x, y, rmax_of(x, y), rows, cols


def az_case(ny, kind, nx=None):
    """(data, x, y, rmax, cols): the y axis fine (ny samples), the x axis coarse (nx <= 512).  kinds: 'smooth', 'offset'
    (1e6 + 1e-3 noise), 'nan' (NaN patches: columns of both count parities, an all-NaN column at rho = 0), 'signs'
    (negative values, zeros and subnormal magnitudes)"""
    nx = nx or (512 if ny >= 4097 else 96)
    x = offset_axis(nx, 0.4987, 1.0)
    y = offset_axis(ny, 0.5, (nx - 1) / max(ny - 1, 1) * 0.93)
    rng = np.random.default_rng(ny + 17 * len(kind))
    r2 = (x[None, :] / nx) ** 2 + (y[:, None] / nx) ** 2
    if kind == 'offset':
        d = 1e6 + 1e-3 * rng.standard_normal((ny, nx))
    elif kind == 'signs':
        d = rng.standard_normal((ny, nx)) * 1e-310
        d[:, ::7] = 0.0
        d[::5, 1::7] = -0.0
        d[::3] *= -1e300
    else:
        d = np.exp(-6 * r2) * (1 + 0.1 * rng.standard_normal((ny, nx)))
    if kind == 'nan':
        d[:, nx // 2 - 1:nx // 2 + 1] = np.nan if ny > 1 else d[:, nx // 2 - 1:nx // 2 + 1]
        d[rng.random((ny, nx)) < 0.02] = np.nan
        if ny > 1:
            d[ny // 2 - 1:ny // 2 + 1, nx // 2 - 1:nx // 2 + 1] = np.nan
    zero_border(d)
    cols = sorted({0, 1, 2, 5, nx // 4, nx // 2 - 1, nx // 2, 3 * nx // 4, nx - 2, nx - 1})
    return d, x, y, rmax_of(x, y), cols


def ray_case(nx, variant):
    """(data, x, y, rmax, t): two rows over y = (0, 1), both the profile P along x = linspace(0, R, nx), so the phi = 0
    ray reads P at the lattice radii exactly and the phi = 2 pi ray (y slightly below 0) reads the fill value 0.  P steps across t = 0.5 on a chunk edge of
    crossing_kernel: 'before' between samples kL - 1 | kL, 'after' between kL | kL + 1, 'ring' high over a band whose
    first and last crossings sit in different chunks, 'tie' with P = t exactly at the edge sample, 'never' below t
    throughout, 'nan' a NaN sample beside the crossing."""
    R = 3.7 * (nx - 1)
    x = np.linspace(0, R, nx)
    L = chunk_len(nx)
    k = max(1, min((nx - 1) // L - 1, 3))          # an interior chunk edge at sample kL
    e = k * L
    P = np.zeros(nx)
    if variant == 'before':
        P[:e] = 1.0
    elif variant == 'after':
        P[:e + 1] = 1.0
    elif variant == 'ring':
        a, b = max(1, e - L // 2 - 1), min(nx - 1, e + 2 * L + 1)
        P[a:b] = 1.0
        P[0] = 0.75
    elif variant == 'tie':
        P[:e] = 1.0
        P[e] = 0.5
    elif variant == 'nan':
        P[:e] = 1.0
        P[e] = np.nan
    y = np.array([0.0, 1.0])
    return np.tile(P, (2, 1)), x, y, rmax_of(x, y), 0.5


RAY_VARIANTS = ('before', 'after', 'ring', 'tie', 'never', 'nan')


def radial_case(nx, ny=16, nan=False):
    """(data, x, y, rmax): a ring g(r) = exp(-((r - r0) / w)^2) + 0.45 exp(-(r / w2)^2), so that rows cross each level
    two to four times; nan adds a NaN patch on the ring"""
    x = offset_axis(nx, 0.47, 1.0)
    y = offset_axis(ny, 0.53, 0.97 * (nx - 1) / max(ny - 1, 1))
    r = np.hypot(x[None, :], y[:, None]) / max(nx - 1, 1)
    d = zero_border(np.exp(-((r - 0.22) / 0.07) ** 2) + 0.45 * np.exp(-(r / 0.09) ** 2))
    if nan:
        d[ny // 2 - 1:ny // 2 + 1, int(0.7 * nx):int(0.7 * nx) + 3] = np.nan
    return d, x, y, rmax_of(x, y)


def crossing_level(vals, maj, metric, relative):
    """t as the device forms it (metric, or fl64(metric * max) of the fp64 lattice) and the extra tolerance its
    rounding and the lattice max's own error add"""
    if not relative:
        return np.float64(metric), LDBL(0)
    v = np.asarray(vals, LDBL)
    if np.isnan(v).any():
        return np.float64(np.nan), LDBL(0)
    k = np.unravel_index(np.argmax(v), v.shape)
    m = np.float64(v[k])
    return np.float64(metric) * m, LDBL(metric) * (8 * np.asarray(maj, LDBL)[k] + abs(LDBL(m))) * LDBL(EPS)
