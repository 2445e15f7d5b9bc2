"""Pupil geometry on the device (reference prysm/geometry.py): circles, signed-distance shapes and their
combinators.  Every signed distance is computed in fp64 by one kernel (pb_sdf) and rounded once to the coordinates'
dtype; the bool masks are sdf <= 0 of the same fp64 distance.  x and y are either two grids of one shape or the
separable row / column pair that optimize_xy_separable reduces a grid to."""
import numpy as np

from . import _ops
from ._capi import (SDF_ANNULUS, SDF_FILLET_RECTANGLE, SDF_INTERSECT, SDF_OFFSET_CIRCLE, SDF_POLYGON, SDF_RECTANGLE,
                    SDF_SPIDER, SDF_SUBTRACT, SDF_UNION)
from .conf import config


def circle_sdf(radius, r):
    """Signed distance to a circle, negative inside (prysm/geometry.py:337-353)."""
    return _ops.asdevice(r) - radius


def circle(radius, r):
    """Binary mask r - radius <= 0 as a bool tensor (prysm/geometry.py:356-372)."""
    return _ops.circle(_ops.asdevice(r), radius)


def antialias(d, dx):
    """Signed distance -> coverage with a one-sample edge ramp, clip(0.5 - d/dx, 0, 1) (prysm/geometry.py:11-34)."""
    d = _ops.asdevice(d)
    return _ops.circle(d, 0.0, aa_dx=dx)          # the circle kernel with radius 0 ramps any signed distance


def grey_circle(radius, r, dx):
    """antialias(circle_sdf(radius, r), dx) in one pass: the grey-edge aperture coronagraph models need
    (prysm/propagation/coronagraph.py:107-110)."""
    return _ops.circle(_ops.asdevice(r), radius, aa_dx=dx)


def union(*ds):
    """Signed distance of the union of shapes, min over the arrays (prysm/geometry.py:37-54)."""
    out = _ops.asdevice(ds[0])
    for d in ds[1:]:
        out = _ops.sdf_combine(SDF_UNION, out, d)
    return out


def intersect(*ds):
    """Signed distance of the intersection of shapes, max over the arrays (prysm/geometry.py:57-74)."""
    out = _ops.asdevice(ds[0])
    for d in ds[1:]:
        out = _ops.sdf_combine(SDF_INTERSECT, out, d)
    return out


def subtract(d1, d2):
    """Signed distance of shape 1 with shape 2 removed, max(d1, -d2) (prysm/geometry.py:77-93)."""
    return _ops.sdf_combine(SDF_SUBTRACT, d1, d2)


def _rotation(angle_deg):
    a = np.radians(angle_deg)
    return float(np.cos(a)), float(np.sin(a))


def _rect_params(width, height, angle):
    if height is None:
        height = width
    if angle == 0:
        return (width, height, 0, 1.0, 0.0)
    if angle == 90:                     # the reference swaps x and y
        return (width, height, 1, 0.0, 1.0)
    return (width, height, 2, *_rotation(angle))


def rectangle_sdf(width, x, y, height=None, angle=0):
    """Signed distance to a rectangle of half-width `width` and half-height `height` (default: width), rotated by
    `angle` degrees; 90 swaps x and y (prysm/geometry.py:182-222)."""
    return _ops.sdf(SDF_RECTANGLE, x, y, _rect_params(width, height, angle))


def rectangle(width, x, y, height=None, angle=0):
    """rectangle_sdf <= 0 (prysm/geometry.py:225-248)."""
    return _ops.sdf(SDF_RECTANGLE, x, y, _rect_params(width, height, angle), mask=True)


def annulus_sdf(rin, rout, r):
    """Signed distance to an annulus, |r - (rin + rout)/2| - (rout - rin)/2 (prysm/geometry.py:375-395)."""
    return _ops.sdf(SDF_ANNULUS, r, None, (rin, rout))


def annulus(rin, rout, r):
    """annulus_sdf <= 0 (prysm/geometry.py:398-416)."""
    return _ops.sdf(SDF_ANNULUS, r, None, (rin, rout), mask=True)


def _vertex_list(vertices):
    v = np.array([[float(c) for c in vtx] for vtx in vertices], dtype=np.float64).reshape(-1, 2)
    if len(v) == 0:
        raise ValueError('a polygon needs at least one vertex')
    return v


def polygon_sdf(vertices, x, y):
    """Signed distance to the polygon through `vertices` (N x 2, either winding, no repeated closing vertex, need
    not be convex): distance to the nearest edge, negative inside by even-odd crossing parity
    (prysm/geometry.py:419-463).  At most 128 vertices."""
    return _ops.sdf(SDF_POLYGON, x, y, verts=_vertex_list(vertices))


def _generate_vertices(sides, radius=1, center=(0, 0), rotation=0):
    """Vertices of a regular polygon on the host, with the reference's dtype rules: the sample index and its product
    with the step angle are config.precision, the rotation and the sum float64 (prysm/geometry.py:521-547)."""
    step = 2 * np.pi / sides
    rot = np.radians(rotation)
    k = np.arange(sides, dtype=config.precision)
    xs = radius * np.sin(k * step + rot) + center[0]
    ys = radius * np.cos(k * step + rot) + center[1]
    return np.stack((xs, ys), axis=1)


def regular_polygon_sdf(sides, radius, x, y, center=(0, 0), rotation=0):
    """Signed distance to a regular polygon of vertex radius `radius` (prysm/geometry.py:466-491)."""
    return _ops.sdf(SDF_POLYGON, x, y, verts=_generate_vertices(sides, radius, center, rotation))


def regular_polygon(sides, radius, x, y, center=(0, 0), rotation=0):
    """regular_polygon_sdf <= 0 (prysm/geometry.py:494-518)."""
    return _ops.sdf(SDF_POLYGON, x, y, verts=_generate_vertices(sides, radius, center, rotation), mask=True)


def _spider_args(vanes, width, rotation, center, rotation_is_rad):
    rot = rotation if rotation_is_rad else np.radians(rotation)
    step = 2 * np.pi / vanes
    angles = [step * k - rot for k in range(vanes)]
    cs = [(float(np.cos(a)), float(np.sin(a))) for a in angles]
    return (width / 2, center[0], center[1]), cs


def spider_sdf(vanes, width, x, y, rotation=0, center=(0, 0), rotation_is_rad=False):
    """Signed distance to `vanes` semi-infinite capsules of full width `width` leaving `center`, rotated clockwise by
    `rotation` (degrees, or radians with rotation_is_rad) (prysm/geometry.py:550-594)."""
    p, cs = _spider_args(vanes, width, rotation, center, rotation_is_rad)
    return _ops.sdf(SDF_SPIDER, x, y, p, verts=cs)


def spider(vanes, width, x, y, rotation=0, center=(0, 0), rotation_is_rad=False):
    """spider_sdf <= 0 (prysm/geometry.py:597-624)."""
    p, cs = _spider_args(vanes, width, rotation, center, rotation_is_rad)
    return _ops.sdf(SDF_SPIDER, x, y, p, verts=cs, mask=True)


def offset_circle(radius, x, y, center):
    """Mask of a circle of `radius` about `center` = (x, y): hypot(x - cx, y - cy) <= radius (prysm/geometry.py:627-653)."""
    return _ops.sdf(SDF_OFFSET_CIRCLE, x, y, (radius, center[0], center[1]), mask=True)


def _fillet_params(width, height, cradius, center, rotation):
    c, s = _rotation(rotation) if rotation != 0 else (1.0, 0.0)
    return (width, height, cradius, center[0], center[1], 1.0 if rotation != 0 else 0.0, c, s)


def rectangle_with_corner_fillets_sdf(width, height, cradius, x, y, center=(0, 0), rotation=0):
    """Signed distance to a rectangle (half-width, half-height) with corner fillets of radius `cradius`, rotated by
    `rotation` degrees about the coordinate origin, then centred on `center` (prysm/geometry.py:656-696)."""
    return _ops.sdf(SDF_FILLET_RECTANGLE, x, y, _fillet_params(width, height, cradius, center, rotation))


def rectangle_with_corner_fillets(width, height, cradius, x, y, center=(0, 0), rotation=0):
    """rectangle_with_corner_fillets_sdf <= 0 (prysm/geometry.py:699-726)."""
    return _ops.sdf(SDF_FILLET_RECTANGLE, x, y, _fillet_params(width, height, cradius, center, rotation), mask=True)
