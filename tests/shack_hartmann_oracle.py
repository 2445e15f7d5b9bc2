"""The Shack-Hartmann cases the engine is checked on (prysm/x/shack_hartmann.py), the numpy statement of spot_centroids,
and the writer of tests/golden/shack_hartmann*.npz.

    PYTHONDONTWRITEBYTECODE=1 python tests/shack_hartmann_oracle.py   (needs the unmodified reference: PRYSM_REFERENCE
                                                                       or oracle/_ref)

The fixtures are the REFERENCE's own screens at precision 64 on the grids `grid()` builds (make_xy_grid's fftrange * dx
in fp64, so a float32 run starts from the same grid rounded once).  Two derived maps pin behaviours a screen does not
show by itself; both are computed with the reference's own _local_window and geometry functions:
  - `claims_<case>`: how many lenslets claim each sample (the windows' masks summed);
  - `near_<case>` (rotated rectangles only): samples whose reference signed distance to some lenslet's edge is within
    NEAR_ANGLE_ULPS ulp of pi of angle at a radius of one pitch, where a device's atan2 / sincos may round the other way.
"""
import os
import sys
import types
from math import ceil

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (ROOT, os.path.join(ROOT, 'oracle')):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import reference  # noqa: E402

WAVELENGTH = 0.55
NEAR_ANGLE_ULPS = 8
# name -> (grid samples (rows, cols), dx, pitch, n, efl, aperture, aperture_kwargs, shift)
CASES = {
    # dx = 0.01, pitch = 0.32: lenslet edges fall exactly on samples, which two to four lenslets then claim
    'rect_edges': ((256, 256), 0.01, 0.32, 8, 20.0, 'rectangle', None, False),
    'rect_shift_odd': ((255, 255), 0.01, 0.32, 8, 20.0, 'rectangle', None, True),
    'rect_n7_shift': ((250, 250), 0.01, 0.33, 7, 15.0, 'rectangle', None, True),
    'rect_height': ((200, 216), 0.01, 0.3, (6, 7), 20.0, 'rectangle', {'height': 0.1}, False),
    'rect_angle0': ((256, 256), 0.01, 0.32, (5, 8), 20.0, 'rectangle', {'height': 0.12, 'angle': 0}, True),
    'rect_angle90': ((256, 256), 0.01, 0.32, (5, 8), 20.0, 'rectangle', {'height': 0.12, 'angle': 90}, True),
    'rect_angle30': ((257, 257), 0.01, 0.32, (6, 7), 20.0, 'rectangle', {'angle': 30}, True),
    # the polar path with the edges on samples: cos(pi) = -1 and sin(pi) ~ 1.2e-16, so each edge sample's signed distance
    # is a few ulp from 0 and its mask is decided by the rounding of atan2 / cos / sin
    'rect_angle180': ((256, 256), 0.01, 0.32, 8, 20.0, 'rectangle', {'angle': 180}, False),
    'circle_edges': ((256, 256), 0.01, 0.32, 8, 20.0, 'circle', None, False),
    'circle_shift': ((257, 240), 0.01, 0.32, (5, 8), 10.0, 'circle', None, True),
    'circle_n6_shift': ((192, 192), 0.0125, 0.4, (6, 7), 25.0, 'circle', None, True),
}
FREE_SPACE = ((128, 128), 0.01, 0.32, 4, 5.0)          # grid, dx, pitch, n, efl of the one free_space intensity


def grid(shape, dx):
    """make_xy_grid(shape, dx=dx) in fp64: fftrange(n) * dx per axis."""
    ny, nx = shape
    x = np.arange(-(nx // 2), -(nx // 2) + nx, dtype=np.float64) * dx
    y = np.arange(-(ny // 2), -(ny // 2) + ny, dtype=np.float64) * dx
    return np.meshgrid(x, y)


def pupil(shape, dx):
    """A circular pupil with a little coma and astigmatism, complex128."""
    x, y = grid(shape, dx)
    R = min(shape) * dx / 2
    r = np.hypot(x, y) / R
    phase = 0.4 * (3 * r ** 2 - 2) * x / R + 0.3 * (x ** 2 - y ** 2) / R ** 2
    return (r <= 1).astype(np.float64) * np.exp(1j * phase)


def centres(pitch, n, shift):
    """The reference's lenslet centres at precision 64 (shack_hartmann.py:83-89)."""
    if not hasattr(n, '__iter__'):
        n = (n, n)
    yc, xc = (np.arange(-(s // 2), -(s // 2) + s, dtype=np.float64) * pitch for s in n)
    if shift:
        if not n[0] & 1:
            xc += pitch / 2
        if not n[1] & 1:
            yc += pitch / 2
    return xc, yc


# ---- the numpy statement of spot_centroids -------------------------------------------------------------------------
def owners(coords, c, pitch):
    """Owner of each coordinate: the lowest i with c_i - pitch/2 <= v < c_i + pitch/2, else -1."""
    lo, hi = c - pitch / 2, c + pitch / 2
    cov = (lo[None, :] <= coords[:, None]) & (coords[:, None] < hi[None, :])
    return np.where(cov.any(axis=1), cov.argmax(axis=1), -1)


def centroids_numpy(frames, x, y, pitch, n, shift=False, threshold=0.0):
    """spot_centroids as numpy, in fp64: (disp (..., 2, rows, cols), flux (..., rows, cols))."""
    xc, yc = centres(pitch, n, shift)
    xv, yv = np.asarray(x, dtype=np.float64)[0], np.asarray(y, dtype=np.float64)[:, 0]
    xo, yo = owners(xv, xc, pitch), owners(yv, yc, pitch)
    f = np.asarray(frames)
    single = f.ndim == 2
    f = f[None] if single else f
    F = f.shape[0]
    disp = np.full((F, 2, len(yc), len(xc)), np.nan)
    flux = np.zeros((F, len(yc), len(xc)))
    for j in range(len(yc)):
        rows = np.flatnonzero(yo == j)
        for i in range(len(xc)):
            cols = np.flatnonzero(xo == i)
            for k in range(F):
                I = f[k][np.ix_(rows, cols)].astype(np.float64)
                if I.size == 0:
                    continue
                t = threshold * I.max() if threshold != 0 else 0.0
                w = np.maximum(I - t, 0)
                sw = w.sum()
                flux[k, j, i] = I.sum()
                if sw != 0:
                    disp[k, 0, j, i] = (w * xv[cols][None, :]).sum() / sw - xc[i]
                    disp[k, 1, j, i] = (w * yv[rows][:, None]).sum() / sw - yc[j]
    return (disp[0], flux[0]) if single else (disp, flux)


# ---- the reference -------------------------------------------------------------------------------------------------
def reference_modules():
    from prysm.conf import config
    from prysm.x import shack_hartmann as sh
    from prysm import geometry, segmented
    from prysm.propagation import Wavefront
    config.precision = 64
    return types.SimpleNamespace(sh=sh, geometry=geometry, segmented=segmented, Wavefront=Wavefront)


def _claims(m, shape, dx, pitch, n, shift, aperture, kw, near_tol=None):
    """Per sample: the number of lenslets whose window and mask claim it, and (near_tol) whether its signed distance to
    some lenslet's rectangle is within near_tol of 0 -- the reference's loop, counting instead of adding phase."""
    x, y = grid(shape, dx)
    if not hasattr(n, '__iter__'):
        n = (n, n)
    spl = int(pitch / (x[0, 1] - x[0, 0]) + 1)
    xc, yc = centres(pitch, n, shift)
    cx, cy = ceil(x.shape[1] / 2), ceil(y.shape[0] / 2)
    count = np.zeros(x.shape, dtype=np.int64)
    near = np.zeros(x.shape, dtype=bool)
    for yy in yc:
        for xx in xc:
            win = m.segmented._local_window(cy, cx, (xx, yy), x[0, 1] - x[0, 0], spl, x, y)
            lx, ly = x[win] - xx, y[win] - yy
            if aperture == 'circle':
                mask = m.geometry.circle((pitch / 2) ** 2, r=lx * lx + ly * ly)
            else:
                mask = m.geometry.rectangle(pitch / 2, x=lx, y=ly, **(kw or {}))
                if near_tol is not None:
                    d = m.geometry.rectangle_sdf(pitch / 2, x=lx, y=ly, **(kw or {}))
                    near[win] |= np.abs(d) <= near_tol
            count[win] += np.broadcast_to(mask, lx.shape)
    return count, near


def _np(v):
    return np.asarray(getattr(v, 'data', v))


def run(m, to_numpy=_np):
    """Every fixture from the modules m: the reference's, or the reference's under set_backend_to_b200() (then
    to_numpy brings device results to the host)."""
    out = {}
    for name, (shape, dx, pitch, n, efl, ap, kw, shift) in CASES.items():
        x, y = grid(shape, dx)
        aperture = getattr(m.geometry, ap)
        out[f'screen_{name}'] = to_numpy(m.sh.shack_hartmann(pitch, n, efl, WAVELENGTH, x, y, aperture=aperture,
                                                             aperture_kwargs=kw, shift=shift))
        rotated = ap == 'rectangle' and (kw or {}).get('angle', 0) not in (0, 90)
        tol = NEAR_ANGLE_ULPS * np.spacing(np.pi) * pitch if rotated else None
        count, near = _claims(m, shape, dx, pitch, n, shift, ap, kw, tol)
        out[f'claims_{name}'] = count.astype(np.uint8)
        if rotated:
            out[f'near_{name}'] = near
    shape, dx, pitch, n, efl = FREE_SPACE
    x, y = grid(shape, dx)
    screen = m.sh.shack_hartmann(pitch, n, efl, WAVELENGTH, x, y)
    wf = m.Wavefront(pupil(shape, dx), WAVELENGTH, dx)
    out['free_space_intensity'] = to_numpy((wf * screen).free_space(dz=efl).intensity)
    return out


def reference_outputs():
    import warnings
    with reference.loaded(), warnings.catch_warnings():
        m = reference_modules()
        warnings.simplefilter('ignore')
        return run(m)


def main():
    """Write tests/golden/shack_hartmann*.npz from the unmodified reference."""
    with reference.loaded():
        from make_golden import save      # imports the reference
        save('shack_hartmann.npz', reference_outputs())


if __name__ == '__main__':
    main()
