"""fp64 restatement of the deformable mirror (prysm/x/dm.py) and of coordinates.warp (prysm/coordinates.py:644-672) in
numpy / scipy (numpy's FFT, the reference's default), and the writer of tests/golden/dm.npz.

    PYTHONDONTWRITEBYTECODE=1 python tests/dm_oracle.py        (needs the unmodified reference: PRYSM_REFERENCE or
                                                                 oracle/_ref)

The fixtures are the REFERENCE's own fp64 outputs on inputs rounded to float32 once (DESIGN.md section 2); the
restatement below is pinned against them on any machine (tests/test_oracle_dm.py) and bit for bit against the
reference itself where it is installed.  The warp is scipy.ndimage.map_coordinates.
"""
import os
import sys

import numpy as np
from scipy import ndimage

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (ROOT, os.path.join(ROOT, 'oracle')):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import prysm_oracle as O  # noqa: E402
import reference  # noqa: E402


def warp(img, xnew, ynew):
    """map_coordinates(img, (ynew, xnew)): order 3, mode='constant', cval=0, prefilter=True."""
    return ndimage.map_coordinates(img, (ynew, xnew))


def apply_transfer_functions(obj, tf):
    """fftshift(ifft2(fft2(ifftshift(obj)) * tf)).real, with numpy's FFT as the reference's default backend uses
    (prysm/convolution.py:35-114, shift=False)."""
    return np.fft.fftshift(np.fft.ifft2(np.fft.fft2(np.fft.ifftshift(obj)) * tf)).real


def fourier_resample(f, zoom):
    """prysm/fttools.py:538-593 with numpy's FFT; the matrix DFT is the oracle's."""
    m, n = f.shape
    M, N = int(m * zoom), int(n * zoom)
    F = np.fft.fftshift(np.fft.fft2(np.fft.ifftshift(f)))
    fx = O.fftrange(N) * (1.0 / zoom / n)
    fy = O.fftrange(M) * (1.0 / zoom / m)
    out = O.MDFT(O.fftrange(n), O.fftrange(m), fx, fy, sign=+1)(F)
    out *= 1 / (m * n)
    return out.real


def lattice_slices(shape, Nact, sep):
    """(iyy, ixx) slices of prepare_actuator_lattice (prysm/x/dm.py:18-63)."""
    cy, cx = [s // 2 for s in shape]
    (nax, nay), (sx, sy) = Nact, sep
    offx = 0 if nax % 2 else sx // 2
    offy = 0 if nay % 2 else sy // 2
    ix = slice(cx + -nax // 2 * sx + offx, cx + nax // 2 * sx + offx, sx)
    iy = slice(cy + -nay // 2 * sy + offy, cy + nay // 2 * sy + offy, sy)
    return iy, ix


def rotation(rot):
    zyx = np.zeros(3)
    zyx[:len(rot)] = rot
    g, b, a = np.radians(zyx)
    Rx = np.array([[1, 0, 0], [0, np.cos(a), -np.sin(a)], [0, np.sin(a), np.cos(a)]])
    Ry = np.array([[np.cos(b), 0, np.sin(b)], [0, 1, 0], [-np.sin(b), 0, np.cos(b)]])
    Rz = np.array([[np.cos(g), -np.sin(g), 0], [np.sin(g), np.cos(g), 0], [0, 0, 1]])
    return Rx @ Ry @ Rz


def projection(shape, rot):
    """(Mfwd, Mifwd) and the forward / reverse pull coordinates (prysm/x/dm.py:66-83)."""
    oy, ox = [(s - 1) / 2 for s in shape]
    R = np.eye(4)
    R[:3, :3] = rotation(rot)
    Tin, Tout = np.eye(4), np.eye(4)
    Tin[0, 3], Tin[1, 3] = -ox, -oy
    Tout[0, 3], Tout[1, 3] = ox, oy
    M = (Tout @ (R @ Tin))[[0, 1, 3]][:, [0, 1, 3]]
    Mi = np.linalg.inv(M)
    y, x = [np.arange(s, dtype=np.float64) for s in shape]
    x, y = np.meshgrid(x, y)
    pts = np.stack([x.ravel(), y.ravel(), np.ones(x.size)])

    def apply(m):
        xp, yp, w = m @ pts
        return (xp / w).reshape(x.shape), (yp / w).reshape(x.shape)
    return M, Mi, apply(Mi), apply(M)


class DM:
    """prysm/x/dm.py:86-331 at fp64."""

    def __init__(self, ifn, Nout, Nact=50, sep=10, shift=(0, 0), rot=(0, 0, 0), upsample=1):
        Nout = (Nout, Nout) if isinstance(Nout, int) else Nout
        Nact = (Nact, Nact) if isinstance(Nact, int) else Nact
        sep = (sep, sep) if isinstance(sep, int) else sep
        self.ifn = np.asarray(ifn, dtype=np.float64)
        s = self.ifn.shape
        self.Nout, self.Nact, self.upsample = Nout, Nact, upsample
        self.obliquity = float(rotation(rot)[2, 2])
        self.iyy, self.ixx = lattice_slices(s, Nact, sep)
        self.actuators = np.zeros((Nact[1], Nact[0]))
        self.needs_rot = not np.allclose(rot, [0, 0, 0])
        if self.needs_rot:
            _, _, (self.projx, self.projy), (self.invprojx, self.invprojy) = projection(s, rot)
        tf = np.fft.fft2(self.ifn)
        if shift[0] != 0 or shift[1] != 0:
            Y, X = [O.forward_ft_unit(1, n, shift=False) for n in s]
            tf = tf * np.exp(X * (-2j * np.pi * shift[0]))[None, :] * np.exp(Y * (-2j * np.pi * shift[1]))[:, None]
        self.tf = tf

    def update(self, actuators):
        self.actuators[:] = actuators

    def render(self, wfe=True):
        poke = np.zeros(self.ifn.shape)
        poke[self.iyy, self.ixx] = self.actuators
        out = apply_transfer_functions(poke, self.tf)
        if self.needs_rot:
            out = warp(out, self.projx, self.projy)
        if wfe:
            out = out * (2 * self.obliquity)
        if self.upsample != 1:
            out = fourier_resample(out, self.upsample)
        self.Nintermediate = out.shape
        if out.shape[0] < self.Nout[0]:
            out = O.pad2d(out, out_shape=self.Nout)
        elif out.shape[0] > self.Nout[1]:
            out = O.crop_center(out, self.Nout)
        return out

    def render_adjoint(self, g, wfe=True):
        g = np.asarray(g, dtype=np.float64)
        if g.shape[0] > self.Nintermediate[0]:
            g = O.crop_center(g, self.Nintermediate)
        elif g.shape[0] < self.Nintermediate[0]:
            g = O.pad2d(g, out_shape=self.Nintermediate)
        if self.upsample != 1:
            g = fourier_resample(g, self.ifn.shape[0] / g.shape[0])
        if wfe:
            g = g * (2 * self.obliquity)
        if self.needs_rot:
            g = warp(g, self.invprojx, self.invprojy)
        return apply_transfer_functions(g, np.conj(self.tf))[self.iyy, self.ixx]


def influence_function(shape, sep):
    """A Gaussian influence function about sample n//2 per axis, 1/e^2 half width 1.2 actuator pitches, float32."""
    ny, nx = shape
    sx, sy = (sep, sep) if isinstance(sep, int) else sep
    y = np.arange(ny) - ny // 2
    x = np.arange(nx) - nx // 2
    g = np.exp(-2 * ((x[None, :] / (1.2 * sx)) ** 2 + (y[:, None] / (1.2 * sy)) ** 2))
    return g.astype(np.float32)


# name -> (ifn shape, constructor keywords); every case is rendered with wfe True and False
SMALL_CASES = {
    'odd_nact': ((64, 64), dict(Nout=64, Nact=7, sep=6)),
    'even_nact': ((64, 64), dict(Nout=64, Nact=8, sep=6)),
    'rect_nact': ((64, 64), dict(Nout=64, Nact=(9, 6), sep=5)),
    'rect_ifn': ((48, 80), dict(Nout=(48, 80), Nact=(10, 6), sep=6)),
    'odd_ifn': ((63, 63), dict(Nout=63, Nact=8, sep=6)),
    'tuple_sep': ((72, 72), dict(Nout=72, Nact=(8, 9), sep=(7, 6))),
    'shift': ((64, 64), dict(Nout=64, Nact=8, sep=6, shift=(1.37, -0.61))),
    'clocking': ((64, 64), dict(Nout=64, Nact=8, sep=6, rot=(12.5, 0, 0))),
    'xtilt': ((64, 64), dict(Nout=64, Nact=8, sep=6, rot=(0, 0, 17.0))),
    'ytilt': ((64, 64), dict(Nout=64, Nact=8, sep=6, rot=(0, 14.0, 0))),
    'all_rot': ((64, 64), dict(Nout=64, Nact=8, sep=6, rot=(5.0, 7.0, 10.0), shift=(0.4, 0.9))),
    'up075': ((64, 64), dict(Nout=48, Nact=8, sep=6, upsample=0.75)),
    'up15': ((64, 64), dict(Nout=96, Nact=8, sep=6, upsample=1.5, rot=(3.0, 0, 8.0))),
    'pad': ((64, 64), dict(Nout=100, Nact=8, sep=6, rot=(0, 0, 10.0))),
    'crop': ((128, 128), dict(Nout=80, Nact=12, sep=8, upsample=0.75, rot=(5.0, 0, 10.0))),
}
LARGE_CASES = {
    'large512': ((512, 512), dict(Nout=512, Nact=48, sep=8, rot=(5.0, 0, 10.0))),
    'large2048': ((2048, 2048), dict(Nout=1536, Nact=64, sep=24, rot=(5.0, 0, 10.0), upsample=0.75)),
}
WINDOW = 64
STRIDE = 37


def case_inputs(name, shape, kw):
    """Influence function and actuator map (float32 values) of one case, seeded by its name."""
    rng = np.random.default_rng(sum(name.encode()))
    ifn = influence_function(shape, kw.get('sep', 10))
    nact = kw['Nact'] if isinstance(kw['Nact'], tuple) else (kw['Nact'], kw['Nact'])
    act = rng.uniform(-1, 1, (nact[1], nact[0])).astype(np.float32)
    return ifn, act


def protograd_for(name, shape):
    rng = np.random.default_rng(sum(name.encode()) + 1)
    return rng.standard_normal(shape).astype(np.float32)


def summarize(prefix, a):
    """A window, strided samples and sums of a large array (the full_c*.npz style).  The window starts an eighth of
    the way in: the reference's convolution moves the surface by half the array (fft2 of an ifn centred on n//2), so
    the centre of a large render is empty."""
    y0, x0 = a.shape[0] // 8, a.shape[1] // 8
    return {f'{prefix}_window': a[y0:y0 + WINDOW, x0:x0 + WINDOW], f'{prefix}_strided': a[::STRIDE, ::STRIDE],
            f'{prefix}_sum': np.array(a.sum()), f'{prefix}_abssum': np.array(np.abs(a).sum()),
            f'{prefix}_shape': np.array(a.shape)}


def run_case(DMcls, name, shape, kw, to_numpy=np.asarray):
    """render (wfe True / False) and render_adjoint of one case with the DM class given; host fp64 arrays."""
    ifn, act = case_inputs(name, shape, kw)
    dm = DMcls(ifn.astype(np.float64), **kw)
    dm.update(act.astype(np.float64))
    out = {}
    for wfe in (True, False):
        r = to_numpy(dm.render(wfe=wfe))
        g = protograd_for(name, r.shape).astype(np.float64)
        out[f'render_{int(wfe)}'] = r
        out[f'adjoint_{int(wfe)}'] = to_numpy(dm.render_adjoint(g, wfe=wfe))
    return out


def main():
    """Write tests/golden/dm.npz from the unmodified reference at fp64."""
    with reference.loaded():
        from prysm.conf import config
        from prysm.x.dm import DM as RefDM
        config.precision = 64
        from make_golden import save
        g = {}
        for name, (shape, kw) in SMALL_CASES.items():
            for k, v in run_case(RefDM, name, shape, kw).items():
                g[f'{name}_{k}'] = v
        for name, (shape, kw) in LARGE_CASES.items():
            res = run_case(RefDM, name, shape, kw)
            for k, v in res.items():
                g.update(summarize(f'{name}_{k}', v) if v.size > 4096 else {f'{name}_{k}': v})
    save('dm.npz', g)


if __name__ == '__main__':
    main()
