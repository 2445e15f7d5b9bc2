"""Segmented apertures on the device (reference prysm/segmented.py:133-368).

The hex ring enumeration, the segment ids, the centres and the windows are host integer and scalar bookkeeping.
Everything on the grid runs in three kernels: one launch rasterises every segment (coverage, local coordinates and
the amplitude), one launch composes the per-segment modal OPD, and two launches give its adjoint with respect to
the coefficients.  The bases are stored once per unique local grid in one packed buffer.
"""
import inspect
import math

import numpy as np
import torch

from . import _ops, coordinates, polynomials
from ._capi import SEGMENT_FIELDS, SEGMENT_TILE_X, SEGMENT_TILE_Y
from .geometry import _generate_vertices

FLAT_TO_FLAT_TO_VERTEX_TO_VERTEX = 1.1547005383792515  # 2/sqrt(3)
VERTEX_TO_VERTEX_TO_FLAT_TO_FLAT = 1 / FLAT_TO_FLAT_TO_VERTEX_TO_VERTEX

# cube-coordinate steps around a hex ring, in the order the reference walks them (prysm/segmented.py:50-53)
_RING_STEPS = ((1, 0, -1), (1, -1, 0), (0, -1, 1), (-1, 0, 1), (-1, 1, 0), (0, 1, -1))


def hex_ring(k):
    """The 6k cells (q, r, s) of ring k, starting at the 'north' cell (prysm/segmented.py:82-99)."""
    q, r, s = -k, k, 0
    cells = []
    for dq, dr, ds in _RING_STEPS:
        for _ in range(k):
            cells.append((q, r, s))
            q, r, s = q + dq, r + dr, s + ds
    return cells[k:] + cells[:k]


def hex_to_xy(cell, radius, rot=90):
    """Centre of a hex cell for cells of `radius` (prysm/segmented.py:66-74)."""
    q, r = cell[0], cell[1]
    if rot == 90:
        x = 3 / 2 * q
        y = VERTEX_TO_VERTEX_TO_FLAT_TO_FLAT * q + math.sqrt(3) * r
    else:
        x = math.sqrt(3) * q + VERTEX_TO_VERTEX_TO_FLAT_TO_FLAT * r
        y = 3 / 2 * r
    return x * radius, y * radius


def local_window(cy, cx, center, dx, samples_per_seg, shape):
    """(row slice, column slice) of the 2*samples_per_seg window about `center`, clamped to the array
    (prysm/segmented.py:102-130)."""
    ny, nx = shape
    ox = cx + int(float(center[0]) / float(dx)) - samples_per_seg      # float64, as the reference's centre array is
    oy = cy + int(float(center[1]) / float(dx)) - samples_per_seg
    ux, uy = ox + 2 * samples_per_seg, oy + 2 * samples_per_seg
    ox, ux = (min(max(v, 0), nx) for v in (ox, ux))
    oy, uy = (min(max(v, 0), ny) for v in (oy, uy))
    return slice(oy, uy), slice(ox, ux)


def hex_layout(shape, dx, rings, segment_diameter, segment_separation, segment_angle=90, exclude=()):
    """Host tables of a composite hexagonal aperture on a grid of `shape` with spacing `dx` (a scalar of the grid's
    dtype, which the window size depends on): (vtov, rseg, all_centers, segment_ids, centres of the included
    segments, windows) (prysm/segmented.py:288-368)."""
    if segment_angle not in {0, 90}:
        raise ValueError('can only synthesize composite apertures with hexagons along a cartesian axis')
    vtov = segment_diameter * FLAT_TO_FLAT_TO_VERTEX_TO_VERTEX
    half_gap = (segment_separation * FLAT_TO_FLAT_TO_VERTEX_TO_VERTEX) / 2
    rseg = vtov / 2
    samples_per_seg = int(rseg / dx + 1)
    cx, cy = int(np.ceil(shape[1] / 2)), int(np.ceil(shape[0] / 2))
    excluded = {int(e) for e in exclude}
    all_centers, ids, centers, windows = [], [], [], []
    if 0 not in excluded:
        all_centers.append((0., 0.))
        ids.append(0)
        centers.append((0., 0.))
        windows.append(local_window(cy, cx, (0, 0), dx, samples_per_seg, shape))
    last = 0
    for ring in range(1, rings + 1):
        for i, cell in enumerate(hex_ring(ring)):
            sid = last + 1 + i
            if sid in excluded:
                continue
            c = hex_to_xy(cell, rseg + half_gap, rot=segment_angle)
            all_centers.append(c)
            ids.append(sid)
            centers.append(c)
            windows.append(local_window(cy, cx, c, dx, samples_per_seg, shape))
        last += 6 * ring
    return vtov, rseg, all_centers, ids, centers, windows


def grid_keys(corner_x, centers, windows):
    """The reference's cache key of each segment's local grid, (local x at the window's first sample, rows, cols)
    (prysm/segmented.py:222-224); corner_x[i] is the global x there.  An empty window has no first sample."""
    keys = []
    for xc, (cxy, (ys, xs)) in zip(corner_x, zip(centers, windows)):
        h, w = ys.stop - ys.start, xs.stop - xs.start
        if h == 0 or w == 0:
            raise IndexError(f'index 0 is out of bounds for axis {0 if h == 0 else 1} with size 0')
        keys.append((float(xc) - float(cxy[0]), h, w))
    return keys


def tile_lists(shape, windows):
    """CSR lists, per output tile of SEGMENT_TILE_Y x SEGMENT_TILE_X samples, of the segments whose windows meet
    the tile, in segment order: (tiles_y, tiles_x, tile_ptr, tile_seg) as int32 host arrays."""
    ny, nx = shape
    ty, tx = -(-ny // SEGMENT_TILE_Y), -(-nx // SEGMENT_TILE_X)
    lists = [[] for _ in range(ty * tx)]
    for s, (ys, xs) in enumerate(windows):
        if ys.stop <= ys.start or xs.stop <= xs.start:
            continue
        for a in range(ys.start // SEGMENT_TILE_Y, (ys.stop - 1) // SEGMENT_TILE_Y + 1):
            for b in range(xs.start // SEGMENT_TILE_X, (xs.stop - 1) // SEGMENT_TILE_X + 1):
                lists[a * tx + b].append(s)
    ptr = np.zeros(ty * tx + 1, dtype=np.int32)
    ptr[1:] = np.cumsum([len(v) for v in lists])
    seg = np.array([s for v in lists for s in v], dtype=np.int32)
    return ty, tx, ptr, seg if seg.size else np.zeros(1, dtype=np.int32)


_ENGINE_BASES = ('zernike_nm_seq', 'zernike_nm')


def _engine_basis(basis_func):
    """The engine's own function in place of the reference's prysm.polynomials Zernike functions."""
    if getattr(basis_func, '__module__', '').startswith('prysm.polynomials') and \
            getattr(basis_func, '__name__', '') in _ENGINE_BASES:
        return getattr(polynomials, basis_func.__name__)
    return basis_func


def _stack_modes(basis, shape, dtype, device):
    """The modes basis_func returned as one contiguous (k, *shape) tensor.  Each mode is broadcast to its window's
    shape, as the reference's product with the mask broadcasts it; a mode that does not broadcast is refused, since
    the kernels read k * rows * cols samples per basis."""
    modes = []
    for i, b in enumerate(basis):
        b = _ops.asdevice(b)
        try:
            modes.append(torch.broadcast_to(b, shape).to(dtype))
        except RuntimeError as e:
            raise ValueError(f'mode {i} of basis_func has shape {tuple(b.shape)}, which does not broadcast to the '
                             f'local grid {shape}') from e
    if not modes:
        return torch.empty((0,) + shape, dtype=dtype, device=device)
    return torch.stack(modes)


class CompositeHexagonalAperture:
    """An aperture composed of several hexagonal segments (prysm/segmented.py:133-285), built on the device."""

    def __init__(self, x, y, rings, segment_diameter, segment_separation, segment_angle=90, exclude=()):
        """Create a new CompositeHexagonalAperture.

        Parameters
        ----------
        x, y : tensor or ndarray
            (m, n) sample positions
        rings : int
            number of rings in the structure
        segment_diameter : float
            flat-to-flat diameter of each segment, same units as x
        segment_separation : float
            edge-to-nearest-edge distance between segments, same units as x
        segment_angle : float, {0, 90}
            rotation angle of each segment
        exclude : sequence of int
            which segment numbers to exclude; 0 is the centre, the others begin 'up' and count clockwise

        """
        x, y = _ops.asdevice(x), _ops.asdevice(y)
        if x.dtype not in (torch.float32, torch.float64):
            x = x.to(torch.float64)
        y = y.to(x.dtype).contiguous()
        if x.ndim != 2 or x.shape != y.shape:
            raise ValueError(f'x {tuple(x.shape)} and y {tuple(y.shape)} must be grids of one shape')
        row = x[0, :2].cpu().numpy()
        dx = row[1] - row[0]                     # in the grid's dtype, like the reference
        self.vtov, rseg, self.all_centers, self.segment_ids, self._centers, self.windows = hex_layout(
            tuple(x.shape), dx, rings, segment_diameter, segment_separation, segment_angle, exclude)
        self.x, self.y = x, y
        self.segment_diameter = segment_diameter
        self.segment_separation = segment_separation
        self.segment_angle = segment_angle
        self.exclude = exclude
        self.opd_bases = None
        self.opd_grids = None

        nseg = len(self.windows)
        self._hw = [(ys.stop - ys.start, xs.stop - xs.start) for ys, xs in self.windows]
        table = np.zeros((nseg, SEGMENT_FIELDS), dtype=np.int64)
        off = 0
        for s, ((ys, xs), (h, w)) in enumerate(zip(self.windows, self._hw)):
            table[s, :5] = ys.start, xs.start, h, w, off
            off += h * w
        self._table = table
        geo = np.zeros((max(nseg, 1), 14))
        for s, c in enumerate(self._centers):
            geo[s, :12] = _generate_vertices(6, rseg, c, rotation=segment_angle).reshape(-1)
            geo[s, 12:] = c
        ty, tx, ptr, lst = tile_lists(tuple(x.shape), self.windows)
        self._tiles = (ty, tx, _ops.asdevice(ptr), _ops.asdevice(lst))
        self._seg = _ops.asdevice(table if nseg else np.zeros((1, SEGMENT_FIELDS), dtype=np.int64))
        cover, lx, ly, self.amp = _ops.hex_segments(x, y, self._tiles, self._seg, _ops.asdevice(geo), 6, float(dx),
                                                    max(off, 1))
        self._cover = cover
        self.local_masks = [cover[o:o + h * w].view(h, w) for o, (h, w) in zip(table[:, 4], self._hw)]
        self.local_coords = [(lx[o:o + h * w].view(h, w), ly[o:o + h * w].view(h, w)) for o, (h, w) in zip(table[:, 4], self._hw)]
        self._bases = None
        self._nmodes = 0

    def prepare_opd_bases(self, basis_func, orders, basis_func_kwargs=None, normalization_radius=None):
        """Prepare the polynomial bases for per-segment phase errors (prysm/segmented.py:178-259).

        basis_func is called with orders and either r=, t= (when its signature has both) or x=, y= keyword grids,
        which are torch tensors on the device: any callable other than the reference's Zernike functions (which
        are replaced by the engine's) must accept torch tensors.  It returns a (k, m, n) tensor or a sequence of
        k tensors that broadcast to the local grid's (m, n).  normalization_radius defaults to half the segment vertex-to-vertex diameter; a 2-tuple
        gives the x and y radii of a Cartesian basis.  Segments whose local grids share a key share one basis.
        """
        if normalization_radius is None:
            normalization_radius = self.vtov / 2
        if not isinstance(normalization_radius, (tuple, list)):
            normalization_radius = (normalization_radius, normalization_radius)
        if basis_func_kwargs is None:
            basis_func_kwargs = {}
        basis_func = _engine_basis(basis_func)
        params = inspect.signature(basis_func).parameters
        radial = 'r' in params and 't' in params
        nseg = len(self.windows)
        corner = np.zeros(nseg)
        if nseg and all(h and w for h, w in self._hw):
            rows, cols = (torch.as_tensor(self._table[:, i], device=self.x.device) for i in (0, 1))
            corner = self.x[rows, cols].cpu().numpy()
        keys = grid_keys(corner, self._centers, self.windows)
        unique = {}
        for s, key in enumerate(keys):
            if key in unique:
                continue
            lx, ly = self.local_coords[s]
            if radial:
                r, th = coordinates.cart_to_polar(lx, ly)
                grid = (r / normalization_radius[0], th)
                basis = basis_func(orders, r=grid[0], t=grid[1], **basis_func_kwargs)
            else:
                grid = (lx / normalization_radius[0], ly / normalization_radius[1])
                basis = basis_func(orders, x=grid[0], y=grid[1], **basis_func_kwargs)
            unique[key] = (grid, _stack_modes(basis, tuple(lx.shape), self.x.dtype, lx.device))
        nmodes = {int(b.shape[0]) for _, b in unique.values()}
        if len(nmodes) > 1:
            raise ValueError(f'basis_func returned different numbers of modes on different local grids: {sorted(nmodes)}')
        self._nmodes = nmodes.pop() if nmodes else 0
        total = sum(b.numel() for _, b in unique.values())
        packed = torch.empty(max(total, 1), dtype=self.x.dtype, device=self.x.device)
        views, off = {}, 0
        for key, (grid, b) in unique.items():
            v = packed[off:off + b.numel()].view(b.shape)
            v.copy_(b)
            views[key] = (grid, v, off)
            off += b.numel()
        for s, key in enumerate(keys):
            self._table[s, 5] = views[key][2]
        self._seg = _ops.asdevice(self._table) if nseg else self._seg
        self._bases = packed
        self.opd_grids = [views[k][0] for k in keys]
        self.opd_bases = [views[k][1] for k in keys]
        return self.opd_grids, self.opd_bases

    def _coefficients(self, coefs):
        if isinstance(coefs, torch.Tensor):
            c = coefs if coefs.is_cuda else coefs.to(self.x.device)
            c = c.to(torch.float64)
        else:
            c = _ops.asdevice(np.asarray(coefs, dtype=np.float64))
        if c.ndim == 1 and c.shape[0] == 0:
            c = c.reshape(0, self._nmodes)
        if c.ndim != 2 or c.shape[1] != self._nmodes:
            raise ValueError(f'coefs of shape {tuple(c.shape)}: one row of {self._nmodes} coefficients per segment is required')
        return c.contiguous()

    def compose_opd(self, coefs, out=None):
        """Compose per-segment optical path error (prysm/segmented.py:261-285): out += mask_s * sum_k c[s, k]
        base_{s,k} over each segment's window, in one launch.  coefs is (n, nmodes), host or device; a float64
        device tensor is read in place, so the call does not synchronise and can be captured in a CUDA graph.  Like
        the reference's zip, fewer rows than segments compose only the leading segments, and overlapping masks add.
        out, allocated as zeros like x if None, is accumulated into and returned."""
        if self._bases is None:
            raise AttributeError('prepare_opd_bases must be called before compose_opd')
        if out is None:
            out = torch.zeros_like(self.x)
        else:
            _ops._check_out(out, self.x.shape, self.x.dtype, self.x.device)
            if not out.is_contiguous():
                raise ValueError('`out` must be contiguous')
        c = self._coefficients(coefs)
        ncoef = min(int(c.shape[0]), len(self.windows))
        return _ops.segment_compose(self._tiles, self._seg, self._cover, self._bases, self._nmodes, c, ncoef, out)

    def compose_opd_adjoint(self, opdbar):
        """Gradient of <compose_opd(c), opdbar> with respect to c: the (nseg, nmodes) device tensor
        sum over segment s's window of opdbar * mask_s * base_{s,k} (a loop of sum_of_2d_modes_adjoint over the
        windows), by a fixed-order two-level reduction: no atomics, no host synchronisation."""
        if self._bases is None:
            raise AttributeError('prepare_opd_bases must be called before compose_opd_adjoint')
        g = _ops.asdevice(opdbar)
        if tuple(g.shape) != tuple(self.x.shape):
            raise ValueError(f'opdbar has shape {tuple(g.shape)}, the aperture is {tuple(self.x.shape)}')
        g = g.to(self.x.dtype).contiguous()
        max_window = max((h * w for h, w in self._hw), default=0)
        return _ops.segment_compose_adjoint(self._seg, len(self.windows), self._cover, self._bases, self._nmodes, g,
                                            max_window)
