"""Self-Referenced Interferometer on the device (reference prysm/x/sri.py).

The reference arm focuses the input onto a single-mode fiber, couples into its mode and re-emits that mode with the
coupled power.  Here the coupling and the re-emitted amplitude never leave the device: one pb_overlap writes the
coupling and c = (P_in eta)^1/2 as device scalars, and one pb_wfs_combine forms Efib c e^{i phi} from them.  The
interference of the two arms, |r ref + t test|^2, is one more pb_wfs_combine.

`SelfReferencedInterferometer` builds its pupil <-> fiber executor once, at construction (the reference re-plans the
same transform on every call), so a forward model is one focus_dft, one pb_overlap, one pb_wfs_combine, one
unfocus_dft and one pb_wfs_combine, and can be captured in a CUDA graph.
"""
import warnings

import numpy as np

from . import _ops
from .coordinates import make_xy_grid, cart_to_polar
from .fibers import smf_mode_field, _coupling, _sum_arg
from .propagation import Wavefront, prepare_executor
from ._richdata import RichData

WF = Wavefront


def _wave(w, wavelength, dx):
    """An engine Wavefront of w: one of ours as it is, any object with data / wavelength / dx (the reference's
    Wavefront) around the same data, an array wrapped with the given wavelength and dx."""
    if isinstance(w, Wavefront):
        return w
    if hasattr(w, 'data') and hasattr(w, 'dx') and hasattr(w, 'wavelength'):
        return Wavefront(w.data, w.wavelength, w.dx, getattr(w, 'space', 'pupil'))
    return Wavefront(w, wavelength, dx)


def overlap_integral(E1, E2, sumI1, sumI2):
    """|sum conj(E1) E2|^2 / (sumI1 sumI2) as a 0-d device tensor (sri.py:18-22), one pb_overlap pass."""
    eta, _ = _coupling(E2, [E1], ip=sumI1, ie=sumI2)
    return eta[0]


def _fiber_pass(E, executor, Efib, Efib_c, ifib, phase_shift):
    """focus_dft -> coupling and c on the device -> Efib c e^{i phase_shift} -> unfocus_dft."""
    at_fpm = executor(E)
    eta, c = _coupling(at_fpm, [Efib], ip=ifib, want_c=True)
    alpha = np.exp(1j * phase_shift) if phase_shift != 0 else 1.0
    Eout = _ops.wfs_combine(Efib_c, alpha, alpha_scale=c)
    return executor.adjoint(Eout), at_fpm, Eout, eta[0]


def to_photonic_fiber_and_back(self, efl, Efib, fib_dx, Ifibsum, executor=None, shift=(0, 0), phase_shift=0,
                               return_more=False):
    """Focus the wavefront `self` onto a single-mode fiber of mode field Efib and return the re-emitted mode to the
    pupil (sri.py:25-85).  With return_more: (next pupil, field at the fiber, emitted field, coupling), the coupling a
    0-d device tensor."""
    self = _wave(self, None, None)
    Efib = _ops.asdevice(getattr(Efib, 'data', Efib))
    fib_samples = tuple(Efib.shape)
    input_samples = tuple(self.data.shape)
    if executor is None:
        executor = prepare_executor(pupil_dx=self.dx, pupil_samples=input_samples, focal_dx=fib_dx,
                                    focal_samples=fib_samples, wavelength=self.wavelength, efl=efl, focal_shift=shift)
    Efib_c = _ops.ascomplex(Efib).to(self.data.dtype)
    nxt, at_fpm, Eout, coupling = _fiber_pass(self.data, executor, Efib, Efib_c, Ifibsum, phase_shift)
    if input_samples[0] != input_samples[1]:
        warnings.warn(f'Forward propagation had input shape {input_samples} which was not uniform between axes, scaling is off')
    if fib_samples[0] != fib_samples[1]:
        warnings.warn(f'Forward propagation had fiber shape {fib_samples} which was not uniform between axes, scaling is off')
    out = Wavefront(nxt, self.wavelength, self.dx, self.space)
    if return_more:
        return (out, Wavefront(at_fpm, self.wavelength, executor.focal_dx, 'psf'),
                Wavefront(Eout, self.wavelength, fib_dx, 'psf'), coupling)
    return out


class SelfReferencedInterferometer:
    """Self-Referenced Interferometer (sri.py:88-178)."""

    def __init__(self, x, y, efl, epd, wavelength, fiber_V=2.3, fiber_b=0.5, fiber_a=1.95 / 2, fiber_samples=256,
                 beamsplitter_RT=(0.8, 0.2)):
        """Same parameters as the reference.  The fiber mode, its intensity sum and the pupil <-> fiber executor are
        built here, once."""
        self.x = x
        self.y = y
        self.dx = float(x[0, 1] - x[0, 0])
        self.efl = efl
        self.epd = epd
        self.wavelength = wavelength
        self.fno = efl / epd
        self.flambd = self.fno * self.wavelength

        fiber_fov_radius = 10 * 1.25 * fiber_a
        self.dx_pinhole = (2 * fiber_fov_radius) / fiber_samples
        xfib, yfib = make_xy_grid(fiber_samples, diameter=2 * fiber_fov_radius)
        rfib, _ = cart_to_polar(xfib, yfib)
        Efib = _ops.ascomplex(smf_mode_field(fiber_V, fiber_a, fiber_b, rfib))
        norm = _ops.dot(Efib, Efib).real ** 0.5
        self._Efib_c = _ops.binary('truediv', Efib, norm)        # unitary fiber mode
        self.Efib = _ops.component('real', self._Efib_c)
        self.Ifib = _ops.intensity(self._Efib_c)
        self.Ifibsum = _ops.dot(self._Efib_c, self._Efib_c).real
        self._ifib = _sum_arg(self.Ifibsum)
        self.dxfib = float(xfib[0, 1] - xfib[0, 0])

        self.ref_r = beamsplitter_RT[0] ** 0.5
        self.test_t = beamsplitter_RT[1] ** 0.5
        self.executor = prepare_executor(pupil_dx=self.dx, pupil_samples=tuple(x.shape), focal_dx=self.dxfib,
                                         focal_samples=tuple(self.Efib.shape), wavelength=self.wavelength, efl=efl)

    def forward_model(self, wave_in, phase_shift=0, debug=False):
        """Intensity at the camera as RichData (sri.py:146-178); debug returns {'at_camera': {'ref', 'test'}}."""
        wave_in = _wave(wave_in, self.wavelength, self.dx)
        E = wave_in.data
        ref, _, _, _ = _fiber_pass(E, self.executor, self.Efib, self._Efib_c, self._ifib, phase_shift)
        if debug:
            mk = lambda d, s: Wavefront(_ops.wfs_combine(d, s), wave_in.wavelength, wave_in.dx, wave_in.space)  # noqa: E731
            return {'at_camera': {'ref': mk(ref, self.ref_r), 'test': mk(E, self.test_t)}}
        I = _ops.wfs_combine(ref, self.ref_r, E, self.test_t, real_out=True)
        return RichData(I, wave_in.dx, wave_in.wavelength)
