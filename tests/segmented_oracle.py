"""fp64 restatement of the signed-distance geometry (prysm/geometry.py) and of the segmented aperture's composition
(prysm/segmented.py:261-285) in numpy, the cases the engine is checked on, and the writer of
tests/golden/segmented*.npz.

    PYTHONDONTWRITEBYTECODE=1 python tests/segmented_oracle.py   (needs the unmodified reference: PRYSM_REFERENCE or
                                                                   oracle/_ref)

The fixtures are the REFERENCE's own outputs.  At precision 64 the reference runs on float64 grids.  At precision 32
it runs with config.precision = 32 (so its vertex tables and the dtype of its amplitude follow the float32 rules) on
the float32 grid promoted to float64: its arithmetic is then fp64, and what is left between it and the engine's
float32 run is the engine's one rounding per stored value (DESIGN.md section 2).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (ROOT, os.path.join(ROOT, 'oracle')):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import reference  # noqa: E402

SHAPE = (61, 80)           # (rows, cols): non-square, odd rows
DX = 0.0371


def grid(shape, dx, dtype):
    """make_xy_grid(shape, dx=dx) at `dtype` (prysm/coordinates.py:344-378): (i - n//2) * dx per axis."""
    ny, nx = shape
    x = (np.arange(nx) - nx // 2).astype(dtype) * dtype(dx)
    y = (np.arange(ny) - ny // 2).astype(dtype) * dtype(dx)
    return np.broadcast_to(x[None, :], shape).copy(), np.broadcast_to(y[:, None], shape).copy()


# ---- restatement (fp64) -------------------------------------------------------------------------------------------

def polygon_sdf(vertices, x, y):
    """prysm/geometry.py:419-463."""
    v = np.asarray(vertices, dtype=np.float64)
    d2 = np.full(np.broadcast(x, y).shape, np.inf)
    inside = np.zeros(d2.shape, dtype=bool)
    for i in range(len(v)):
        (x0, y0), (x1, y1) = v[i], v[(i + 1) % len(v)]
        ex, ey, wx, wy = x1 - x0, y1 - y0, x - x0, y - y0
        t = np.clip((wx * ex + wy * ey) / (ex * ex + ey * ey), 0, 1)
        px, py = wx - t * ex, wy - t * ey
        d2 = np.minimum(d2, px * px + py * py)
        inside ^= ((y0 > y) != (y1 > y)) & ((wx * ey < ex * wy) == (y1 > y0))
    d = np.sqrt(d2)
    return np.where(inside, -d, d)


def regular_vertices(sides, radius, center, rotation, precision):
    """prysm/geometry.py:521-547 with config.precision = `precision`."""
    k = np.arange(sides, dtype=precision)
    a = k * (2 * np.pi / sides) + np.radians(rotation)
    return np.stack((radius * np.sin(a) + center[0], radius * np.cos(a) + center[1]), axis=1)


def spider_sdf(vanes, width, x, y, rotation=0, center=(0, 0), rotation_is_rad=False):
    """prysm/geometry.py:550-594."""
    x, y = x - center[0], y - center[1]
    rot = rotation if rotation_is_rad else np.radians(rotation)
    d = None
    for k in range(vanes):
        a = 2 * np.pi / vanes * k - rot
        along, across = x * np.cos(a) - y * np.sin(a), x * np.sin(a) + y * np.cos(a)
        v = np.hypot(np.minimum(along, 0), across) - width / 2
        d = v if d is None else np.minimum(d, v)
    return d


def _rotate(x, y, deg):
    r, t = np.hypot(x, y), np.arctan2(y, x) + np.radians(deg)
    return r * np.cos(t), r * np.sin(t)


def _box(qx, qy):
    return np.hypot(np.maximum(qx, 0), np.maximum(qy, 0)) + np.minimum(np.maximum(qx, qy), 0)


def rectangle_sdf(width, x, y, height=None, angle=0):
    """prysm/geometry.py:182-222."""
    height = width if height is None else height
    if angle == 90:
        x, y = y, x
    elif angle != 0:
        x, y = _rotate(x, y, angle)
    return _box(np.abs(x) - width, np.abs(y) - height)


def fillet_sdf(width, height, cradius, x, y, center=(0, 0), rotation=0):
    """prysm/geometry.py:656-696."""
    if rotation != 0:
        x, y = _rotate(x, y, rotation)
    x, y = x - center[0], y - center[1]
    return _box(np.abs(x) - (width - cradius), np.abs(y) - (height - cradius)) - cradius


def annulus_sdf(rin, rout, r):
    """prysm/geometry.py:375-395."""
    return np.abs(r - (rin + rout) / 2) - (rout - rin) / 2


def offset_circle(radius, x, y, center):
    """prysm/geometry.py:627-653."""
    return np.hypot(x - center[0], y - center[1]) - radius <= 0


def compose(windows, masks, bases, coefs, out):
    """prysm/segmented.py:278-285 with the masks and bases of the fixture."""
    out = out.copy()
    for (ys, xs), m, b, c in zip(windows, masks, bases, coefs):
        out[ys, xs] += np.tensordot(c, b, axes=(0, 0)) * m
    return out


# ---- the cases ----------------------------------------------------------------------------------------------------

CONVEX = [(-0.9, -0.7), (1.1, -0.5), (1.3, 0.6), (0.2, 1.05), (-1.05, 0.4)]
CONCAVE = [(-1.0, -0.9), (1.2, -0.9), (1.2, -0.2), (0.1, -0.15), (0.25, 0.95), (-1.1, 0.8)]


def geometry_cases(g, x, y, r):
    """name -> the value of the geometry function under test; `g` is a module with the reference's functions (the
    reference's prysm.geometry, or prysm_b200.geometry)."""
    a = g.regular_polygon_sdf(7, 0.93, x, y, center=(0.13, -0.21), rotation=17)
    b = g.rectangle_sdf(0.83, x, y, height=0.47, angle=23)
    return {
        'poly_ccw': g.polygon_sdf(CONVEX, x, y),
        'poly_cw': g.polygon_sdf(CONVEX[::-1], x, y),
        'poly_concave': g.polygon_sdf(CONCAVE, x, y),
        'poly_empty': g.polygon_sdf(CONVEX, x[0:0], y[0:0]),
        'regpoly': a,
        'regpoly_mask': g.regular_polygon(6, 1.07, x, y, center=(-0.05, 0.11), rotation=90),
        'spider_deg': g.spider_sdf(4, 0.083, x, y, rotation=30, center=(0.1, 0.05)),
        'spider_rad': g.spider_sdf(3, 0.097, x, y, rotation=0.4, rotation_is_rad=True),
        'spider_mask': g.spider(3, 0.097, x, y, rotation=-75),
        'rect': g.rectangle_sdf(0.83, x, y, height=0.47),
        'rect90': g.rectangle_sdf(0.83, x, y, height=0.47, angle=90),
        'rect_rot': b,
        'rect_mask': g.rectangle(0.61, x, y, angle=90),
        'fillet': g.rectangle_with_corner_fillets_sdf(0.9, 0.6, 0.21, x, y, center=(0.1, -0.05)),
        'fillet_rot': g.rectangle_with_corner_fillets_sdf(0.9, 0.6, 0.21, x, y, center=(0.1, -0.05), rotation=12),
        'fillet_mask': g.rectangle_with_corner_fillets(0.9, 0.6, 0.21, x, y, rotation=12),
        'annulus': g.annulus_sdf(0.4, 1.1, r),
        'annulus_mask': g.annulus(0.4, 1.1, r),
        'offset_circle': g.offset_circle(0.7, x, y, center=(0.2, -0.1)),
        'union': g.union(a, b, g.spider_sdf(2, 0.1, x, y)),
        'intersect': g.intersect(a, b),
        'subtract': g.subtract(a, b),
    }


# name -> (shape, dx, rings, segment_diameter, segment_separation, segment_angle, exclude, with bases)
HEX_CASES = {
    'r1_a90': ((64, 72), 0.0271, 1, 0.5, 0.02, 90, (), True),
    'r2_a0_excl': ((80, 96), 0.0213, 2, 0.42, 0.017, 0, (0, 3), True),
    'r3_clamped': ((96, 104), 0.0189, 3, 0.31, 0.011, 90, (5,), True),
    'overlap': ((72, 72), 0.0203, 2, 0.3, 0.004, 90, (), True),
    'offgrid': ((40, 70), 0.0177, 3, 0.33, 0.012, 0, (), False),
}
NMS = [(0, 0), (1, 1), (1, -1), (2, 0), (2, -2), (2, 2)]
MONOMIALS = [(0, 0), (1, 0), (0, 1), (2, 0), (1, 1)]
XY_NORM = (0.23, 0.19)


def xy_monomials(orders, x, y):
    """A Cartesian basis for the x=, y= branch of prepare_opd_bases: plain arithmetic, so numpy arrays and torch
    tensors both work."""
    return [x ** i * y ** j for i, j in orders]


def hex_coefs(name, nseg, nmodes):
    rng = np.random.default_rng(sum(name.encode()) + nmodes)
    return rng.standard_normal((nseg, nmodes)).astype(np.float32).astype(np.float64)


def hex_out0(name, shape):
    return np.random.default_rng(sum(name.encode()) + 99).standard_normal(shape).astype(np.float32).astype(np.float64)


# full-size apertures: (grid n, diameter, rings, segment diameter, gap, exclude), 11 Zernike terms
LARGE_CASES = {
    'jwst512': (512, 6.6, 2, 1.32, 0.007, (0,)),
    'luvoira2048': (2048, 15.0, 6, 1.223, 0.007, (0, 91, 109, 97, 103, 115, 121)),
}
LARGE_NMS = [(0, 0), (1, 1), (1, -1), (2, 0), (2, -2), (2, 2), (3, -1), (3, 1), (3, -3), (3, 3), (4, 0)]
WINDOW = 64
STRIDE = 37


def summarize(prefix, a):
    """A window about the centre, strided samples and sums (accumulated in float64) of a large array."""
    y0, x0 = a.shape[0] // 2 - WINDOW // 2, a.shape[1] // 2 + a.shape[1] // 8
    return {f'{prefix}_window': a[y0:y0 + WINDOW, x0:x0 + WINDOW], f'{prefix}_strided': a[::STRIDE, ::STRIDE],
            f'{prefix}_sum': np.array(a.sum(dtype=np.float64)),
            f'{prefix}_abssum': np.array(np.abs(a).sum(dtype=np.float64))}


def large_grid(n, diameter, dtype):
    dx = diameter / n
    return grid((n, n), dx, dtype)


def run_hex(S, poly, name, x, y, to_numpy=np.asarray):
    """Everything a hex case stores, computed with the segmented module S and polynomial module poly given."""
    shape, dx, rings, diam, sep, angle, exclude, with_bases = HEX_CASES[name]
    cha = S.CompositeHexagonalAperture(x, y, rings, diam, sep, segment_angle=angle, exclude=exclude)
    out = {
        'windows': np.array([[w[0].start, w[0].stop, w[1].start, w[1].stop] for w in cha.windows]).reshape(-1, 4),
        'all_centers': np.array(cha.all_centers, dtype=np.float64).reshape(-1, 2),
        'segment_ids': np.array([int(i) for i in cha.segment_ids]),
        'vtov': np.array(cha.vtov),
        'amp': to_numpy(cha.amp),
        'masks': np.concatenate([to_numpy(m).ravel() for m in cha.local_masks] or [np.zeros(0)]),
        'local_x': np.concatenate([to_numpy(c[0]).ravel() for c in cha.local_coords] or [np.zeros(0)]),
        'local_y': np.concatenate([to_numpy(c[1]).ravel() for c in cha.local_coords] or [np.zeros(0)]),
    }
    if not with_bases:
        return out, cha
    nseg = len(cha.windows)
    for tag, fn, kw in (('zern', poly.zernike_nm_seq, {}), ('xy', xy_monomials, {'normalization_radius': XY_NORM})):
        orders = NMS if tag == 'zern' else MONOMIALS
        grids, bases = cha.prepare_opd_bases(fn, orders, **kw)
        out[f'{tag}_bases'] = np.concatenate([to_numpy(b).ravel() for b in bases])
        out[f'{tag}_grid0'] = np.concatenate([to_numpy(gr[0]).ravel() for gr in grids])
        out[f'{tag}_grid1'] = np.concatenate([to_numpy(gr[1]).ravel() for gr in grids])
        c = hex_coefs(name, nseg, len(orders))
        out[f'{tag}_opd'] = to_numpy(cha.compose_opd(c))
        out0 = hex_out0(name, shape)
        out[f'{tag}_opd_out'] = to_numpy(cha.compose_opd(c, out=_like(out0, x)))
        out[f'{tag}_opd_short'] = to_numpy(cha.compose_opd(c[:nseg - 2]))
    return out, cha


def _like(a, x):
    """`a` as the array type of x (numpy for the reference, a device tensor for the engine)."""
    if isinstance(x, np.ndarray):
        return a.astype(x.dtype)
    import prysm_b200 as pb
    return pb.asdevice(a.astype(np.float32 if str(x.dtype).endswith('32') else np.float64))


def run_large(S, poly, name, x, y, to_numpy=np.asarray):
    n, diameter, rings, diam, sep, exclude = LARGE_CASES[name]
    cha = S.CompositeHexagonalAperture(x, y, rings, diam, sep, exclude=exclude)
    cha.prepare_opd_bases(poly.zernike_nm_seq, LARGE_NMS)
    c = hex_coefs(name, len(cha.windows), len(LARGE_NMS)) * 1e-2
    out = {}
    out.update(summarize(f'{name}_amp', to_numpy(cha.amp)))
    out.update(summarize(f'{name}_opd', to_numpy(cha.compose_opd(c))))
    out[f'{name}_windows'] = np.array([[w[0].start, w[0].stop, w[1].start, w[1].stop] for w in cha.windows])
    return out


def main():
    """Write tests/golden/segmented*.npz from the unmodified reference."""
    with reference.loaded():
        from prysm.conf import config
        from prysm import geometry as G, segmented as S, polynomials as P
        from make_golden import save
        g = {}
        for prec in (64, 32):
            dt = np.float64 if prec == 64 else np.float32
            config.precision = prec
            x, y = (a.astype(np.float64) for a in grid(SHAPE, DX, dt))
            r = np.hypot(x, y)
            for k, v in geometry_cases(G, x, y, r).items():
                g[f'geom{prec}_{k}'] = np.asarray(v)
            for name, case in HEX_CASES.items():
                xx, yy = (a.astype(np.float64) for a in grid(case[0], case[1], dt))
                if prec == 32:       # the windows of the promoted grid must be those of the float32 grid
                    cha32 = S.CompositeHexagonalAperture(*grid(case[0], case[1], dt), case[2], case[3], case[4],
                                                         segment_angle=case[5], exclude=case[6])
                res, cha = run_hex(S, P, name, xx, yy)
                if prec == 32:
                    assert cha32.windows == cha.windows, name
                for k, v in res.items():
                    g[f'hex{prec}_{name}_{k}'] = v
            for name, (n, diameter, *_rest) in LARGE_CASES.items():
                xx, yy = (a.astype(np.float64) for a in large_grid(n, diameter, dt))
                for k, v in run_large(S, P, name, xx, yy).items():
                    g[f'large{prec}_{k}'] = v
    save('segmented.npz', g)


if __name__ == '__main__':
    main()
