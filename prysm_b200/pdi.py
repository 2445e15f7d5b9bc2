"""Phase-shifting point diffraction interferometer on the device (reference prysm/x/pdi.py).

The grating is evaluated from the stored x grid inside the pass that multiplies it into the field (pb_grating, fp64
arithmetic), so a phase step costs no grid arithmetic and no temporary grating.  The two arms are the engine's
to_fpm_and_back with executors built at construction, and the interference |ref + t test|^2 is one pb_wfs_combine.
"""
import numpy as np
import torch

from . import _ops
from ._capi import GRATING_SIN_AMP, GRATING_RECTANGLE
from .conf import config
from .coordinates import make_xy_grid
from .geometry import circle
from .propagation import Wavefront as WF, prepare_executor
from ._richdata import RichData
from .sri import _wave


def _rect_params(x_dtype, duty, amplitude, offset, period):
    eps = float(np.finfo(np.float32 if x_dtype == torch.float32 else np.float64).eps)
    return [period, duty * period, offset + amplitude, offset - amplitude, offset, eps]


def _grid(x):
    x = _ops.asdevice(x)
    if x.dtype not in (torch.float32, torch.float64):
        x = x.to(config.real_dtype)
    return x


def rectangle_pulse(x, duty=0.5, amplitude=0.5, offset=0.5, period=2 * np.pi):
    """Rectangular pulse in [offset - amplitude, offset + amplitude] (pdi.py:11-51), one pb_grating pass.

    numpy's mod semantics (the remainder takes the sign of the period); offset + amplitude below duty * period,
    offset - amplitude above, and `offset` where |x mod period| is below the epsilon of x's dtype."""
    x = _grid(x)
    return _ops.grating(GRATING_RECTANGLE, x, _rect_params(x.dtype, duty, amplitude, offset, period))


class PSPDI:
    """Phase Shifting Point Diffraction Interferometer (Medecki interferometer) (pdi.py:54-253)."""

    def __init__(self, x, y, efl, epd, wavelength, test_arm_offset=64, test_arm_fov=64, test_arm_samples=256,
                 test_arm_transmissivity=1, pinhole_diameter=0.25, pinhole_samples=128, grating_rulings=64,
                 grating_type='sin_amp', grating_axis='x'):
        """Same parameters as the reference.  The masks and both arms' executors are built here, once."""
        grating_type = grating_type.lower()
        grating_axis = grating_axis.lower()
        self.x = x
        self.y = y
        self._x = _grid(x)
        self.dx = float(x[0, 1] - x[0, 0])
        self.efl = efl
        self.epd = epd
        self.wavelength = wavelength
        self.fno = efl / epd
        self.flambd = self.fno * self.wavelength

        self.grating_rulings = grating_rulings
        self.grating_period = self.epd / grating_rulings
        self.grating_type = grating_type
        self.grating_axis = grating_axis
        if grating_type == 'ronchi':
            self._grating = (GRATING_RECTANGLE, _rect_params(self._x.dtype, 0.5, 0.5, 0.5, self.grating_period))
        elif grating_type == 'sin_amp':
            self._grating = (GRATING_SIN_AMP, [grating_rulings * np.pi / (epd / 2)])
        else:
            raise ValueError('unsupported grating type')

        self.test_arm_offset = test_arm_offset
        self.test_arm_fov = test_arm_fov
        self.test_arm_samples = test_arm_samples
        self.test_arm_eps = test_arm_fov / test_arm_samples
        self.test_arm_fov_compute = (test_arm_fov + self.test_arm_eps) * self.flambd
        self.test_arm_mask_rsq = (test_arm_fov * self.flambd / 2) ** 2
        self.test_arm_transmissivity = test_arm_transmissivity
        # the grating is always evaluated on x; the axis moves only the test-arm window (pdi.py:159-162)
        if self.grating_axis == 'x':
            self.test_arm_shift = (grating_rulings * self.flambd, 0)
        else:
            self.test_arm_shift = (0, grating_rulings * self.flambd)

        self.pinhole_diameter = pinhole_diameter * self.flambd
        self.pinhole_samples = pinhole_samples
        self.dx_pinhole = pinhole_diameter / (pinhole_samples - 1)
        self.pinhole_fov_radius = pinhole_samples / 2 * self.dx_pinhole
        xph, yph = make_xy_grid(pinhole_samples, diameter=2 * self.pinhole_fov_radius)
        self.pinhole = circle((pinhole_diameter / 2) ** 2, xph * xph + yph * yph)       # grid preparation
        xt, yt = make_xy_grid(test_arm_samples, diameter=self.test_arm_fov_compute)
        self.dx_test_arm = float(xt[0, 1] - xt[0, 0])
        self.test_mask = circle(self.test_arm_mask_rsq, xt * xt + yt * yt)
        # the test arm's amplitude transmissivity, folded into its mask: t * (F^-1 m F E) = F^-1 (t m) F E
        self._test_mask_t = self.test_mask
        if test_arm_transmissivity != 1:
            self._test_mask_t = self.test_mask.to(config.real_dtype) * test_arm_transmissivity

        pupil_samples = tuple(x.shape)
        self.pinhole_executor = prepare_executor(pupil_dx=self.dx, pupil_samples=pupil_samples, focal_dx=self.dx_pinhole,
                                                 focal_samples=tuple(self.pinhole.shape), wavelength=self.wavelength,
                                                 efl=self.efl)
        self.test_executor = prepare_executor(pupil_dx=self.dx, pupil_samples=pupil_samples, focal_dx=self.dx_test_arm,
                                              focal_samples=tuple(self.test_mask.shape), wavelength=self.wavelength,
                                              efl=self.efl, focal_shift=self.test_arm_shift)

    def grating_func(self, x):
        """The grating at x, as the reference's `grating_func` (one pb_grating pass)."""
        kind, params = self._grating
        return _ops.grating(kind, _grid(x), params)

    def forward_model(self, wave_in, phase_shift=0, debug=False):
        """Intensity at the camera as RichData (pdi.py:195-253); sets self.ref_beam / self.test_beam, and with debug
        returns the reference's dict of fields."""
        shift = phase_shift / (2 * np.pi) * self.grating_period if phase_shift != 0 else 0.0
        w = _wave(wave_in, self.wavelength, self.dx)
        kind, params = self._grating
        i = WF(_ops.grating(kind, self._x, params, shift, E=w.data), w.wavelength, w.dx, w.space)
        if debug:
            ref_beam, ref_at_fpm, ref_after_fpm = i.to_fpm_and_back(self.pinhole, self.pinhole_executor,
                                                                    return_more=True)
            test_beam, test_at_fpm, test_after_fpm = i.to_fpm_and_back(self.test_mask, self.test_executor,
                                                                       return_more=True)
            if self.test_arm_transmissivity != 1:
                test_beam = test_beam * self.test_arm_transmissivity
        else:
            ref_beam = i.to_fpm_and_back(self.pinhole, self.pinhole_executor)
            test_beam = i.to_fpm_and_back(self._test_mask_t, self.test_executor)
        self.ref_beam = ref_beam
        self.test_beam = test_beam
        if debug:
            return {
                'total_field': ref_beam + test_beam,
                'at_camera': {'ref': ref_beam, 'test': test_beam},
                'at_fpm': {'ref': (ref_at_fpm, ref_after_fpm), 'test': (test_at_fpm, test_after_fpm)},
            }
        I = _ops.wfs_combine(ref_beam.data, 1.0, test_beam.data, 1.0, real_out=True)
        return RichData(I, ref_beam.dx, ref_beam.wavelength)


def evaluate_test_ref_arm_matching(debug_dict):
    """(mean ref intensity / mean test intensity, ref intensity, test intensity) of a debug dict (pdi.py:256-261); the
    ratio is a host float."""
    pak = debug_dict['at_camera']
    ref, test = pak['ref'], pak['test']
    I1, I2 = ref.intensity, test.intensity
    ratio = _ops.dot(ref.data, ref.data).real / _ops.dot(test.data, test.data).real
    ratio *= test.data.numel() / ref.data.numel()
    return ratio, I1, I2
