"""Backend selection in the style of prysm.mathops (reference prysm/mathops.py:48-116).

`set_backend_to_b200()` is the sibling of `set_backend_to_cupy()`: it plugs this engine into an installed
prysm so that existing user code (`Wavefront.focus`, `free_space`, `prepare_executor`, `mtf_from_psf`, ...)
runs on the H100 kernels unchanged.  The reference's shim forwards *module attributes* (np.exp, fft.fft2);
fusing pad + shifts + FFT into one kernel needs the *function* level, so the hot functions themselves are
re-bound, following the precedent of prysm/x/polarization.py:541-552 (`setattr(propagation, name, wrapper)`).
`Wavefront` methods resolve `focus`, `angular_spectrum`, ... through the names imported into
prysm/propagation/wavefront.py:11-25, so those module globals are re-bound as well.

The reference's `Wavefront` class itself is patched in place as well (its elementwise constructors and
properties are written against the `np` shim -- `np.exp` on the host, three temporaries for `|.|^2`,
prysm/propagation/wavefront.py:59-166): `from_amp_and_phase`, `phase_screen`, `thin_lens`, `intensity`, `phase`,
`real`, `imag`, the `* / + -` operators and the adjoint twins delegate to the kernels and return objects of the
reference's own classes, so user code that imported `Wavefront` before the switch keeps working and never
touches numpy `exp` or eager tensor arithmetic.

The reference's `RichData` class gets `slices`, `exact_polar`, `exact_xy`, `exact_x` and `exact_y` that run on the
device when its `data` is a CUDA tensor (what the re-bound `mtf_from_psf` returns) and call the originals otherwise.

Interferometric metrology follows the same rule, because the reference's host `Interferogram` must behave exactly as
before: the free functions of prysm.interferogram, prysm.util's statistics and prysm.polynomials' lstsq are re-bound to
dispatchers that run the engine when their data argument is a CUDA tensor and call the original otherwise, and the
reference's `Interferogram` class gets its metrology properties and methods patched the same way.

`set_backend_to_defaults()` restores every name it replaced.
"""
import importlib

from . import bayer as _bayer
from . import coatings as _coat
from . import convolution as _conv
from . import coordinates as _coords
from . import detector as _det
from . import dm as _dm
from . import fibers as _fib
from . import fttools as _ft
from . import interferogram as _ifg
from . import otf as _otf
from . import pdi as _pdi
from . import polarization as _pol
from . import polynomials as _poly
from . import propagation as _prop
from . import psf as _psf
from . import psi as _psi
from . import shack_hartmann as _sh
from . import sri as _sri
from . import thinfilm as _tf

# prysm module -> {attribute: replacement}
_PROPAGATION_FUNCS = (
    'focus', 'unfocus', 'focus_adjoint', 'unfocus_adjoint',
    'angular_spectrum', 'angular_spectrum_adjoint', 'angular_spectrum_transfer_function',
    'prepare_executor', 'coordinates_for_focus', 'focus_dft', 'unfocus_dft', 'focus_dft_adjoint', 'unfocus_dft_adjoint',
)
_CORONAGRAPH_FUNCS = (
    'to_fpm_and_back', 'to_fpm_and_back_adjoint', 'to_fpm_and_back_multiresolution',
    'to_fpm_and_back_multiresolution_adjoint', 'babinet', 'babinet_adjoint', 'vortex_phase_mask', 'prepare_measured_fpm',
)
_COATINGS_STACK_FUNCS = ('stack_rt', 'RTA', 'internal_fields', 'field_at_depth')
_COATINGS_DIFF_FUNCS = ('forward_eval', 'ForwardEval', 'thickness_gradient', 'index_gradient')
_COATINGS_MERIT_NAMES = ('Reflectance', 'Transmittance', 'LayerAbsorptance', 'FieldIntensityAtBoundary',
                         'PeakFieldAtInterfaces', 'FieldInLayer', 'MeritFunction', 'as_merit')
_COATINGS_MONITOR_FUNCS = ('monitoring_trace', 'cutoff_levels', 'simulate_run', 'monitoring_error_sensitivity',
                           'choose_monitor_wavelength')
_TARGETS = {
    'prysm.propagation.fft': {n: getattr(_prop, n) for n in ('focus', 'unfocus', 'focus_adjoint', 'unfocus_adjoint')},
    'prysm.propagation.angular_spectrum': {n: getattr(_prop, n) for n in (
        'angular_spectrum', 'angular_spectrum_adjoint', 'angular_spectrum_transfer_function')},
    'prysm.propagation.dft': {**{n: getattr(_prop, n) for n in (
        'prepare_executor', 'coordinates_for_focus', 'focus_dft', 'unfocus_dft', 'focus_dft_adjoint', 'unfocus_dft_adjoint')},
        'MDFT': _ft.MDFT, 'CZT': _ft.CZT, 'FFTDFT': _ft.FFTDFT,
        'prepare_multiresolution': _prop.prepare_multiresolution, 'MultiResolutionExecutor': _prop.MultiResolutionExecutor},
    'prysm.propagation.coronagraph': {n: getattr(_prop, n) for n in _CORONAGRAPH_FUNCS},
    'prysm.propagation.wavefront': {**{n: getattr(_prop, n) for n in _PROPAGATION_FUNCS + _CORONAGRAPH_FUNCS if n not in (
        'angular_spectrum_transfer_function', 'coordinates_for_focus', 'vortex_phase_mask', 'prepare_measured_fpm')},
        'prepare_multiresolution': _prop.prepare_multiresolution, 'pad2d': _ft.pad2d, 'crop_center': _ft.crop_center},
    'prysm.propagation': {**{n: getattr(_prop, n) for n in _PROPAGATION_FUNCS + _CORONAGRAPH_FUNCS},
                          'prepare_multiresolution': _prop.prepare_multiresolution,
                          'MultiResolutionExecutor': _prop.MultiResolutionExecutor},
    'prysm.fttools': {'MDFT': _ft.MDFT, 'CZT': _ft.CZT, 'FFTDFT': _ft.FFTDFT, 'pad2d': _ft.pad2d,
                      'crop_center': _ft.crop_center, 'fourier_resample': _ft.fourier_resample},
    'prysm.convolution': {'conv': _conv.conv, 'apply_transfer_functions': _conv.apply_transfer_functions},
    'prysm.otf': {n: getattr(_otf, n) for n in (
        'transform_psf', 'transform_psf_adjoint', 'mtf_from_psf', 'ptf_from_psf', 'otf_from_psf', 'mtf_ptf_otf_from_psf',
        'mtf_from_psf_adjoint', 'ptf_from_psf_adjoint', 'otf_from_psf_adjoint', 'encircled_energy',
        'encircled_energy_adjoint', 'diffraction_limited_mtf', 'analytical_encircled_energy_circular_aperture')},
    'prysm.psf': {n: getattr(_psf, n) for n in (
        'centroid', 'estimate_size', 'fwhm', 'one_over_e', 'one_over_e_sq', 'airydisk', 'airydisk_efield', 'airydisk_ft')},
    'prysm.polynomials': {'sum_of_2d_modes': _poly.sum_of_2d_modes, 'sum_of_2d_modes_adjoint': _poly.sum_of_2d_modes_adjoint},
    'prysm.polynomials.fitting': {'sum_of_2d_modes': _poly.sum_of_2d_modes,
                                  'sum_of_2d_modes_adjoint': _poly.sum_of_2d_modes_adjoint},
    'prysm.coordinates': {'warp': _coords.warp},
    'prysm.x.dm': {'DM': _dm.DM},
    # the reference's own add_jones_propagation() then wraps the engine's functions with the engine's adapter; the
    # small 2x2 constructors stay the reference's
    'prysm.x.polarization': {n: getattr(_pol, n) for n in (
        'jones_adapter', 'apply_polarization_optic', 'vector_vortex_retarder', 'jones_to_mueller', 'broadcast_kron',
        'pauli_coefficients')},
    # wavefront sensing: prysm.x.sri binds smf_mode_field, prepare_executor and unfocus_dft at import time, so its
    # classes and functions themselves are re-bound (as prysm.x.dm's DM is)
    'prysm.x.fibers': {n: getattr(_fib, n) for n in (
        'compute_LP_modes', 'smf_mode_field', 'mode_overlap_integral', 'multimode_coupling')},
    'prysm.x.sri': {n: getattr(_sri, n) for n in (
        'overlap_integral', 'to_photonic_fiber_and_back', 'SelfReferencedInterferometer')},
    'prysm.x.pdi': {n: getattr(_pdi, n) for n in ('rectangle_pulse', 'PSPDI', 'evaluate_test_ref_arm_matching')},
    'prysm.x.psi': {n: getattr(_psi, n) for n in ('psi_accumulate', 'degroot_formalism_psi')},
    'prysm.x.shack_hartmann': {'shack_hartmann': _sh.shack_hartmann},
    # image sensors: the Detector class itself is re-bound (as prysm.x.dm's DM is)
    'prysm.detector': {'Detector': _det.Detector, 'apply_lut': _det.apply_lut, 'pixel': _det.pixel},
    'prysm.bayer': {n: getattr(_bayer, n) for n in (
        'wb_prescale', 'wb_postscale', 'composite_bayer', 'decomposite_bayer', 'recomposite_bayer',
        'demosaic_deinterlace', 'assemble_superresolved', 'demosaic_malvar')},
    # thin films.  The merit terms and the needle function run on the device.  The reference's refine, CoatingProblem
    # and synthesize bind as_merit, the gradients and needle_function at import time and feed the results to host
    # optimizer loops, so in those modules the names are re-bound to variants that hand back numpy (the evaluation is
    # still on the device); insert_needle, cleanup and the optimizers stay the reference's.  Optical monitoring runs on
    # the device: its five run-level functions are re-bound outright, and turning_points / level_cut are dispatched on
    # their signal (below).
    'prysm.thinfilm': {'multilayer_stack_rt': _tf.multilayer_stack_rt},
    'prysm.x.coatings': {n: getattr(_coat, n) for n in
                         _COATINGS_STACK_FUNCS + _COATINGS_DIFF_FUNCS + _COATINGS_MERIT_NAMES + ('needle_function',)
                         + _COATINGS_MONITOR_FUNCS},
    'prysm.x.coatings.monitoring': {n: getattr(_coat, n) for n in _COATINGS_MONITOR_FUNCS},
    'prysm.x.coatings.stack': {n: getattr(_coat, n) for n in _COATINGS_STACK_FUNCS},
    'prysm.x.coatings.diff': {n: getattr(_coat, n) for n in _COATINGS_DIFF_FUNCS},
    'prysm.x.coatings.merit': {n: getattr(_coat, n) for n in _COATINGS_MERIT_NAMES},
    'prysm.x.coatings.problem': {'as_merit': _coat._host_as_merit, 'thickness_gradient': _coat.thickness_gradient,
                                 'index_gradient': _coat.index_gradient},
    'prysm.x.coatings.refine': {'as_merit': _coat._host_as_merit},
    'prysm.x.coatings.needle': {'as_merit': _coat._host_as_merit, 'needle_function': _coat._host_needle_function},
}

# names that run the engine only when their data argument (name, position) is a CUDA tensor: module -> {attribute:
# (engine function, argument name, position)}
_STATS = {n: (getattr(_ifg, n), 'array', 0) for n in ('mean', 'pv', 'rms', 'Sa', 'std')}
_LSTSQ = {'lstsq': (_poly.lstsq, 'data', 1)}
_MONITOR_CUTS = {n: (getattr(_coat, n), 'signal', 1) for n in ('turning_points', 'level_cut')}
_DISPATCHED = {
    'prysm.interferogram': {**_STATS, **_LSTSQ, 'fit_plane': (_ifg.fit_plane, 'z', 2),
                            'fit_sphere': (_ifg.fit_sphere, 'z', 0), 'make_window': (_ifg.make_window, 'signal', 0),
                            'psd': (_ifg.psd, 'height', 0), 'bandlimited_rms': (_ifg.bandlimited_rms, 'psd', 1),
                            'window_2d_welch': (_ifg.window_2d_welch, 'r', 0),
                            'ideal_lpf_iir2d': (_ifg.ideal_lpf_iir2d, 'r', 0),
                            'designfilt2d': (_ifg.designfilt2d, 'r', 0)},
    'prysm.util': _STATS,
    'prysm.polynomials': _LSTSQ,
    'prysm.polynomials.fitting': _LSTSQ,
    'prysm.x.coatings': _MONITOR_CUTS,
    'prysm.x.coatings.monitoring': _MONITOR_CUTS,
}
_IFG_PROPERTIES = ('dropout_percentage', 'pv', 'rms', 'Sa', 'std', 'strehl')
_IFG_METHODS = ('pvr', 'fill', 'crop', 'recenter', 'remove_piston', 'remove_tiptilt', 'remove_power', 'mask',
                'strip_latcal', 'latcal', 'pad', 'spike_clip', 'psd', 'filter', 'bandlimited_rms',
                'total_integrated_scatter', 'slope')

_saved = {}  # (module name, attribute) -> original
_saved_cls = {}  # (class, attribute) -> original descriptor (or _MISSING)
_MISSING = object()


def _wavefront_patches(ref_cls, ref_richdata):
    """Descriptors that replace the elementwise members of the reference's Wavefront class.  Each one builds the
    engine's Wavefront around the same device array, calls the engine, and hands the result back as an object of
    the REFERENCE's classes (so isinstance checks and attribute access in user code are unchanged)."""
    from . import _ops
    from ._richdata import RichData as _OurRich
    Ours = _prop.Wavefront

    def to_ours(w):
        return Ours(w.data, w.wavelength, w.dx, w.space)

    def unwrap(v):
        if isinstance(v, ref_cls):
            return to_ours(v)
        if isinstance(v, ref_richdata):
            return _OurRich(v.data, v.dx, v.wavelength)
        return v

    def rewrap(v):
        if isinstance(v, Ours):
            return ref_cls(v.data, v.wavelength, v.dx, v.space)
        if isinstance(v, _OurRich):
            return ref_richdata(v.data, v.dx, v.wavelength)
        if isinstance(v, tuple):
            return tuple(rewrap(e) for e in v)
        return v

    def method(name):
        def f(self, *args, **kwargs):
            r = getattr(to_ours(self), name)(*[unwrap(a) for a in args], **{k: unwrap(v) for k, v in kwargs.items()})
            return rewrap(r)
        f.__name__ = name
        f.__doc__ = getattr(Ours, name).__doc__
        return f

    def classm(name):
        def f(cls, *args, **kwargs):
            r = getattr(Ours, name)(*[unwrap(a) for a in args], **{k: unwrap(v) for k, v in kwargs.items()})
            if isinstance(r, Ours):
                return cls(r.data, r.wavelength, r.dx, r.space)
            return rewrap(r)
        f.__name__ = name
        f.__doc__ = getattr(Ours, name).__doc__
        return classmethod(f)

    def prop(name):
        return property(lambda self: rewrap(getattr(to_ours(self), name)), doc=getattr(Ours, name).__doc__)

    out = {n: classm(n) for n in ('from_amp_and_phase', 'phase_screen', 'thin_lens', 'thin_lens_adjoint')}
    out.update({n: prop(n) for n in ('intensity', 'phase', 'real', 'imag')})
    out.update({n: method(n) for n in ('__numerical_operation__', 'intensity_adjoint', 'from_amp_and_phase_adjoint_phase',
                                       'from_amp_and_phase_adjoint_amp', 'phase_screen_adjoint_phase')})
    return out


def _returning_reference_richdata(fn):
    """Wrap an engine function so that every engine RichData in its result becomes a prysm._richdata.RichData."""
    import functools
    from ._richdata import RichData as _OurRich
    ref = importlib.import_module('prysm._richdata').RichData

    def conv(v):
        if isinstance(v, _OurRich):
            return ref(v.data, v.dx, v.wavelength)
        if isinstance(v, tuple):
            return tuple(conv(e) for e in v)
        return v

    @functools.wraps(fn)
    def wrapped(*args, **kwargs):
        return conv(fn(*args, **kwargs))
    wrapped.__wrapped_engine__ = fn
    return wrapped


def _patch_wavefront_class():
    try:
        pw = importlib.import_module('prysm.propagation.wavefront')
        rd = importlib.import_module('prysm._richdata').RichData
    except ImportError:
        return
    cls = pw.Wavefront
    for name, desc in _wavefront_patches(cls, rd).items():
        if (cls, name) not in _saved_cls:
            _saved_cls[(cls, name)] = cls.__dict__.get(name, _MISSING)
        setattr(cls, name, desc)


def _richdata_patches():
    """Methods that replace the sampling members of the reference's RichData class: with a CUDA tensor as `data` they
    run the engine on the object's own x / y axes; otherwise (a host RichData, an Interferogram, ...) they call the
    reference's original, so host objects behave exactly as before."""
    import torch
    from . import _richdata as ours
    ref = importlib.import_module('prysm._richdata').RichData

    def on_device(self):
        return isinstance(self.data, torch.Tensor) and self.data.is_cuda

    def make(name, engine):
        orig = getattr(ref, name)

        def f(self, *args, **kwargs):
            if on_device(self):
                return engine(self, *args, **kwargs)
            return orig(self, *args, **kwargs)
        f.__name__ = name
        f.__doc__ = orig.__doc__
        return f

    def slices(self, twosided=None):
        if twosided is None:
            twosided = self._default_twosided
        return ours.Slices(data=self.data, x=self.x[0], y=self.y[..., 0], twosided=twosided)

    engines = {
        'slices': slices,
        'exact_polar': lambda self, rho, phi=None: ours.exact_polar(self.data, self.x, self.y, rho, phi),
        'exact_xy': lambda self, x, y=None: ours.exact_xy(self.data, self.x, self.y, x, y),
        'exact_x': lambda self, x: ours.exact_x(self.data, self.x, self.y, x),
        'exact_y': lambda self, y: ours.exact_y(self.data, self.x, self.y, y),
    }
    return ref, {n: make(n, e) for n, e in engines.items()}


def _patch_richdata_class():
    try:
        cls, patches = _richdata_patches()
    except ImportError:
        return
    for name, fn in patches.items():
        if (cls, name) not in _saved_cls:
            _saved_cls[(cls, name)] = cls.__dict__.get(name, _MISSING)
            setattr(cls, name, fn)


def _on_device(v):
    import torch
    return isinstance(v, torch.Tensor) and v.is_cuda


def _dispatch(engine, orig, argname, pos):
    """orig with the engine in its place when the data argument is a CUDA tensor; reference RichData results"""
    import functools
    eng = _returning_reference_richdata(engine)

    @functools.wraps(orig)
    def f(*args, **kwargs):
        v = args[pos] if len(args) > pos else kwargs.get(argname)
        return eng(*args, **kwargs) if _on_device(v) else orig(*args, **kwargs)
    f.__wrapped_engine__ = engine
    return f


def _with_reference_mode_sum(fn):
    """A copy of the reference function fn whose call-time `from prysm.polynomials import ...` sees the reference's own
    sum_of_2d_modes.  The reference's host pvr imports it at call time, and the engine's (numpy in, CUDA out), which
    the backend binds in prysm.polynomials, would put its projection on the device.  The copy has its own globals and
    import, so nothing shared is swapped while it runs."""
    import builtins
    import types
    key = ('prysm.polynomials', 'sum_of_2d_modes')
    if key not in _saved:
        return fn
    view = types.ModuleType(key[0])
    view.__dict__.update(importlib.import_module(key[0]).__dict__)
    view.sum_of_2d_modes = _saved[key]

    def imp(name, globals=None, locals=None, fromlist=(), level=0):
        if name == key[0] and fromlist and level == 0:
            return view
        return builtins.__import__(name, globals, locals, fromlist, level)
    g = dict(fn.__globals__)
    g['__builtins__'] = {**builtins.__dict__, '__import__': imp}
    return types.FunctionType(fn.__code__, g, fn.__name__, fn.__defaults__, fn.__closure__)


def _interferogram_patches():
    """Members that replace the metrology of the reference's Interferogram class: with a CUDA tensor as `data` they run
    the engine's Interferogram on the same data, dx and cached coordinates and write the results back (methods change
    the object and return it, as the reference's do); otherwise they call the reference's original."""
    from ._richdata import RichData as _OurRich
    ref = importlib.import_module('prysm.interferogram').Interferogram
    ref_rich = importlib.import_module('prysm._richdata').RichData
    coords = ('_x', '_y', '_r', '_t')

    def to_ours(self, with_coords=True):
        """the engine's object on the same data; with_coords: the cached coordinates too (host ones are uploaded once:
        back() leaves the device copies in the reference object)"""
        o = _ifg.Interferogram.__new__(_ifg.Interferogram)
        o.dx, o.wavelength, o._data = self.dx, self.wavelength, _ifg._real(self.data)
        for c in coords:
            v = getattr(self, c, None) if with_coords else None
            setattr(o, c, None if v is None else _ifg._ops.asdevice(v))
        o.intensity, o.meta, o._latcaled = self.intensity, self.meta, getattr(self, '_latcaled', False)
        return o

    def back(self, o):
        self._data, self.dx, self._latcaled = o._data, o.dx, o._latcaled
        self.interpf_x = self.interpf_y = self.interpf_2d = None
        for c in coords:
            setattr(self, c, getattr(o, c))

    def conv(v):
        if isinstance(v, _OurRich):
            r = ref_rich(v.data, v.dx, v.wavelength)
            for c in coords:
                setattr(r, c, getattr(v, c))
            r._default_twosided = v._default_twosided
            return r
        if isinstance(v, tuple):
            return tuple(conv(e) for e in v)
        return v

    def method(name):
        orig = getattr(ref, name)
        host = _with_reference_mode_sum(orig) if name == 'pvr' else orig

        def f(self, *args, **kwargs):
            if not _on_device(self.data):
                return host(self, *args, **kwargs)
            o = to_ours(self)
            r = getattr(o, name)(*args, **kwargs)
            back(self, o)
            return self if r is o else conv(r)
        f.__name__ = name
        f.__doc__ = orig.__doc__
        return f

    def prop(name):
        orig = ref.__dict__[name]
        # the statistics read no coordinates
        return property(lambda self: getattr(to_ours(self, False), name) if _on_device(self.data) else orig.fget(self),
                        doc=orig.__doc__)

    out = {n: prop(n) for n in _IFG_PROPERTIES}
    out.update({n: method(n) for n in _IFG_METHODS})
    return ref, out


def _patch_interferogram_class():
    try:
        cls, patches = _interferogram_patches()
    except ImportError:
        return
    for name, fn in patches.items():
        if (cls, name) not in _saved_cls:
            _saved_cls[(cls, name)] = cls.__dict__.get(name, _MISSING)
            setattr(cls, name, fn)


def set_backend_to_b200(device=None):
    """Route prysm's propagation hot path through the H100 engine.  Call after `import prysm`
    (like the reference's own set_backend_to_* helpers).  Arrays handed to the re-bound functions may be
    numpy arrays (uploaded) or CUDA tensors; results are CUDA tensors (`prysm.mathops.array_to_true_numpy`
    already understands them, prysm/mathops.py:150-153)."""
    from . import _ops
    if device is not None:
        _ops.set_device(device)
    try:
        import prysm.conf as pconf
    except ImportError as exc:  # pragma: no cover
        raise ImportError('set_backend_to_b200() plugs into an installed prysm; it is not importable here') from exc
    from .conf import config
    config.precision = pconf.config.precision  # follow prysm's precision setting
    # import every target before re-binding any: a module imported mid-way (prysm.x.dm binds fourier_resample,
    # apply_transfer_functions and warp at import time) would otherwise capture engine functions as its defaults
    mods = {}
    for modname in [*_TARGETS, *_DISPATCHED]:
        try:
            mods[modname] = importlib.import_module(modname)
        except ImportError:
            continue
    for modname, mod in mods.items():
        if modname not in _TARGETS:
            continue
        repl = _TARGETS[modname]
        if modname in ('prysm.otf', 'prysm.x.psi'):   # these return RichData: hand back the reference's own container
            repl = {k: _returning_reference_richdata(v) for k, v in repl.items()}
        for attr, new in repl.items():
            if hasattr(mod, attr) and (modname, attr) not in _saved:
                _saved[(modname, attr)] = getattr(mod, attr)
            if hasattr(mod, attr):
                setattr(mod, attr, new)
    for modname, names in _DISPATCHED.items():
        try:
            mod = importlib.import_module(modname)
        except ImportError:
            continue
        for attr, (engine, argname, pos) in names.items():
            if not hasattr(mod, attr) or (modname, attr) in _saved:
                continue
            _saved[(modname, attr)] = orig = getattr(mod, attr)
            setattr(mod, attr, _dispatch(engine, orig, argname, pos))
    _patch_wavefront_class()
    _patch_richdata_class()
    _patch_interferogram_class()
    return sorted(_saved)


def set_backend_to_defaults():
    """Undo set_backend_to_b200(): every re-bound name gets its original object back."""
    for (modname, attr), orig in list(_saved.items()):
        setattr(importlib.import_module(modname), attr, orig)
        del _saved[(modname, attr)]
    for (cls, name), orig in list(_saved_cls.items()):
        if orig is _MISSING:
            delattr(cls, name)
        else:
            setattr(cls, name, orig)
        del _saved_cls[(cls, name)]
