"""Deformable mirrors on the device (reference prysm/x/dm.py).

`DM` keeps the reference's constructor, attributes and methods.  Everything a call does not depend on is built once
in the constructor: the transfer function (influence-function spectrum times the shift ramps, whose phases are
range-reduced in fp64), the actuator lattice, the fp64 projection matrices and the Fourier-resample executors.
`render` is then

    scatter actuators -> FFT (ifftshift fused) -> * tf -> inverse FFT (fftshift fused)
      -> [cubic-spline warp, coordinates from the matrix, 2*obliquity in the same pass] -> [Fourier resample]
      -> pad / crop

and `render_adjoint` runs the reference's chain back to the lattice.  Neither synchronises with the host or builds a
plan, so both can be captured into a CUDA graph.

Kept from the reference (DESIGN.md section 2): `render_adjoint` warps with the forward-projection coordinates, which
is an approximation and not the transpose of the interpolation; the crop test compares shape[0] with Nout[1]; and
`render_adjoint` before any `render` fails, because `Nintermediate` is set by `render`.
Deviations: the projection matrices and the shift-ramp phases are fp64 at either precision, and `render_adjoint`
never scales the caller's array in place.
"""
import copy

import numpy as np
import torch

from . import _ops
from .conf import config
from .fttools import FourierResampler, _expi, crop_center, pad2d


def _axis_lattice(n, nact, sep):
    """Start and stride of the lattice along one axis: the reference's slice(neg, pos, sep) applied to n samples
    (prysm/x/dm.py:18-63; more actuators on the negative side when nact is odd, FFT-centred otherwise)."""
    c = n // 2
    off = 0 if nact % 2 else sep // 2
    neg = c + -nact // 2 * sep + off
    pos = c + nact // 2 * sep + off
    r = range(*slice(neg, pos, sep).indices(n))
    if len(r) != nact:
        raise ValueError(f'{nact} actuators {sep} samples apart do not fit an axis of {n} samples')
    return r.start, r.step


def actuator_lattice(shape, Nact, sep):
    """(y0, sy, x0, sx): the lattice rows are y0 + k*sy, its columns x0 + l*sx (shape is (rows, cols); Nact and sep
    are (X, Y) pairs, as in the reference)."""
    y0, sy = _axis_lattice(shape[0], Nact[1], sep[1])
    x0, sx = _axis_lattice(shape[1], Nact[0], sep[0])
    return y0, sy, x0, sx


def rotation_matrix(rot):
    """3 x 3 rotation for (Z, Y, X) angles in degrees: Rx @ Ry @ Rz (prysm/coordinates.py:381-429), fp64."""
    zyx = np.zeros(3)
    zyx[:len(rot)] = rot
    gz, gy, gx = np.radians(zyx)
    cx, sx, cy, sy, cz, sz = np.cos(gx), np.sin(gx), np.cos(gy), np.sin(gy), np.cos(gz), np.sin(gz)
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    return Rx @ Ry @ Rz


def projection_matrices(shape, rot):
    """(Mfwd, Mifwd), 3 x 3 fp64 homographies on pixel coordinates (x, y, 1): the rotation about the array centre
    ((n-1)/2 per axis) with z dropped, and its inverse.  render pulls through Mifwd and render_adjoint through Mfwd
    (prysm/x/dm.py:66-83)."""
    oy, ox = [(s - 1) / 2 for s in shape]
    R4 = np.eye(4)
    R4[:3, :3] = rotation_matrix(rot)
    Tin, Tout = np.eye(4), np.eye(4)
    Tin[0, 3], Tin[1, 3] = -ox, -oy
    Tout[0, 3], Tout[1, 3] = ox, oy
    keep = [0, 1, 3]
    Mfwd = np.ascontiguousarray((Tout @ (R4 @ Tin))[keep][:, keep])
    return Mfwd, np.linalg.inv(Mfwd)


class DM:
    """A DM whose actuators fill a rectangular region on a perfect grid, and have the same influence function
    (prysm/x/dm.py:86-331).  Inputs may be numpy arrays or CUDA tensors; results are CUDA tensors at
    config.precision."""

    def __init__(self, ifn, Nout, Nact=50, sep=10, shift=(0, 0), rot=(0, 0, 0), upsample=1, project_centering='fft'):
        if isinstance(Nout, int):
            Nout = (Nout, Nout)
        if isinstance(Nact, int):
            Nact = (Nact, Nact)
        if isinstance(sep, int):
            sep = (sep, sep)
        rd = config.real_dtype
        ifn = _ops.asdevice(ifn, rd)
        s = tuple(ifn.shape)
        self.ifn = ifn
        self.Ifn = _ops.fft2(ifn, dir=-1)
        self.Nout = Nout
        self.Nact = Nact
        self.sep = sep
        self.shift = shift
        self.obliquity = float(rotation_matrix(rot)[2, 2])
        self.rot = rot
        self.upsample = upsample

        self._lattice = actuator_lattice(s, Nact, sep)
        self.actuators = torch.zeros((Nact[1], Nact[0]), dtype=rd, device=ifn.device)

        self.needs_rot = not np.allclose(rot, [0, 0, 0])
        self._Mfwd = self._Mifwd = None
        if self.needs_rot:
            self._Mfwd, self._Mifwd = projection_matrices(s, rot)

        if shift[0] != 0 or shift[1] != 0:
            # exp(-2 pi i shift f) per axis with f = fftfreq(n), the phase range-reduced in fp64
            cd = config.complex_dtype
            fy, fx = np.fft.fftfreq(s[0]), np.fft.fftfreq(s[1])
            self.Xramp = _ops.asdevice(_expi(-shift[0] * fx), cd)
            self.Yramp = _ops.asdevice(_expi(-shift[1] * fy), cd)
            self.tf = [_ops.mul_outer(self.Ifn, vy=self.Yramp, vx=self.Xramp)]
        else:
            self.tf = [self.Ifn]

        # the Fourier-resample executors of render (zoom `upsample`) and of render_adjoint (the reference's zoom
        # ifn.shape[0] / intermediate.shape[0]), for the shapes a render produces; others are built on first use
        self._resamplers = {}
        if upsample != 1:
            fwd = self._resampler(s, upsample)
            self._resampler(fwd.out_shape, s[0] / fwd.out_shape[0])

    def _resampler(self, shape, zoom):
        key = (tuple(shape), zoom)
        if key not in self._resamplers:
            self._resamplers[key] = FourierResampler(tuple(shape), zoom)
        return self._resamplers[key]

    def copy(self):
        """Make a (deep) copy of this DM."""
        return copy.deepcopy(self)

    def update(self, actuators):
        """actuators[:] = actuators (a (Nact_y, Nact_x) array or tensor)."""
        self.actuators[:] = _ops.asdevice(actuators, self.actuators.dtype)

    def _convolve(self, a, conj, scale=1.0):
        """fftshift(ifft2(fft2(ifftshift(a)) * tf)) (conj(tf) for the adjoint) as a complex array; `scale` rides in
        the forward transform."""
        ny, nx = a.shape
        O = _ops.fft2(a, dir=-1, shift_in=True, scale=scale)
        O = _ops.mask_multiply(O, self.tf[0], conj=conj)
        return _ops.fft2(O, dir=+1, scale=1.0 / (ny * nx), shift_out=True)

    def render(self, wfe=True):
        """Surface figure error (wfe=False) or reflected wavefront error (2 * obliquity times it), projected into the
        beam normal by `rot`, resampled by `upsample` and padded / cropped to `Nout` (prysm/x/dm.py:219-273)."""
        scale = 2 * self.obliquity if wfe else 1.0
        poke = _ops.dm_scatter(self.actuators, tuple(self.ifn.shape), self._lattice)
        sfe = self._convolve(poke, conj=False)
        if self.needs_rot:       # the real part, the pull through Mifwd and the scale in one pass
            warped = _ops.warp(sfe, matrix=self._Mifwd, scale=scale)
        else:
            warped = _ops.mask_multiply(sfe, real_out=True, scale=scale)
        if self.upsample != 1:
            warped = _ops.component('real', self._resampler(tuple(warped.shape), self.upsample)(warped))
        self.Nintermediate = tuple(warped.shape)
        if warped.shape[0] < self.Nout[0]:
            warped = pad2d(warped, out_shape=self.Nout)
        elif warped.shape[0] > self.Nout[1]:
            warped = crop_center(warped, out_shape=self.Nout)
        return warped

    def render_adjoint(self, protograd, wfe=True):
        """Apply the adjoint of render() to `protograd` (real, the shape render returns); returns the gradient with
        respect to the actuators, shape (Nact_y, Nact_x) (prysm/x/dm.py:275-331).  `protograd` is not modified."""
        g = _ops.asdevice(protograd)
        if g.is_complex():
            raise ValueError('render_adjoint is not compatible with a complex protograd')
        g = g.to(self.actuators.dtype)
        if g.shape[0] > self.Nintermediate[0]:
            g = crop_center(g, out_shape=self.Nintermediate)
        elif g.shape[0] < self.Nintermediate[0]:
            g = pad2d(g, out_shape=self.Nintermediate)
        scale = 2 * self.obliquity if wfe else 1.0
        if self.upsample != 1:
            g = self._resampler(tuple(g.shape), self.ifn.shape[0] / g.shape[0])(g)     # complex; its real part is used
            if not self.needs_rot:
                g, scale = _ops.mask_multiply(g, real_out=True, scale=scale), 1.0
        if self.needs_rot:
            g, scale = _ops.warp(g, matrix=self._Mfwd, scale=scale), 1.0
        in_actuator_space = self._convolve(g, conj=True, scale=scale)
        return _ops.dm_gather(in_actuator_space, self.actuators.shape, self._lattice)
