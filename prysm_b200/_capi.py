"""ctypes binding of libprysm_b200.so (the C ABI declared in include/prysm_b200.h).

The library is dlopen'ed directly -- no pybind / torch-extension layer.  If it is missing the
import fails loudly: there is no CPU or PyTorch fallback anywhere in this package.
"""
import ctypes as C
import os
import re

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, '_lib', 'libprysm_b200.so')
HEADER_PATH = os.path.join(os.path.dirname(_HERE), 'include', 'prysm_b200.h')

# exact scalar widths: an int / long long slip passes garbage in the upper half of a register
_SCALARS = {'int': C.c_int, 'long long': C.c_longlong, 'double': C.c_double}


def read_header(path=HEADER_PATH):
    """(SIGNATURES, enums) of the C header: name -> (restype, argtypes) of every `pb_*` prototype, and name -> value of
    every `PB_*` enumerator.  Every pointer and pb_handle_t binds as c_void_p (the C type cannot tell a host array
    from a device one).  A C type outside the mapping, or an enumerator without a literal integer value, raises
    ImportError: nothing is guessed."""
    def ctype(t, ret=False):
        if ret and t == 'const char*':
            return C.c_char_p
        if '*' in t or t == 'pb_handle_t':
            return C.c_void_p
        if t not in _SCALARS:
            raise ImportError(f'{path}: no ctypes type for the C type {t!r}')
        return _SCALARS[t]

    with open(path) as f:
        code = re.sub(r'/\*.*?\*/', '', f.read(), flags=re.S)
    sigs = {}
    for ret, name, params in re.findall(r'^([A-Za-z_][\w ]*?\**)\s*(pb_\w+)\s*\(([^)]*)\)\s*;', code, flags=re.M):
        params = [] if params.strip() in ('', 'void') else params.split(',')
        # every parameter in the header is named: drop the name, keep the type
        sigs[name] = (ctype(ret.strip(), ret=True),
                      [ctype(re.sub(r'\s*\b\w+$', '', ' '.join(p.split()))) for p in params])
    missed = set(re.findall(r'\b(pb_\w+)\s*\(', code)) - set(sigs)
    if missed:
        raise ImportError(f'{path}: cannot read the prototypes of {sorted(missed)}')
    enums = {}
    for body in re.findall(r'\benum\b[^{;]*\{([^}]*)\}', code):
        for item in filter(None, (e.strip() for e in body.split(','))):
            m = re.fullmatch(r'(PB_\w+)\s*=\s*(-?\d+)', item)
            if m is None:
                raise ImportError(f'{path}: the enumerator {item!r} has no literal integer value')
            enums[m.group(1)] = int(m.group(2))
    return sigs, enums


SIGNATURES, _enums = read_header()
# PB_NAME binds as NAME, except the two dtype codes, whose PB_ names every caller uses
globals().update({k if k in ('PB_C64', 'PB_C128') else k[3:]: v for k, v in _enums.items()})


def route_code(kind, L=0, flags=0):
    """the `route` argument of pb_route_launch_count: the 32-bit int the C side forms (kinds 8 and up are negative)"""
    code = (kind << 28 | L << 8 | flags) & 0xFFFFFFFF
    return code - (1 << 32) if code >> 31 else code


def load_library(path=LIB_PATH):
    if not os.path.exists(path):
        raise ImportError(
            f'{path} is missing: build it with `python prysm_b200/build.py` '
            '(prysm_b200 has no CPU fallback)')
    lib = C.CDLL(path)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the .so and the header diverge
        fn.restype = res
        fn.argtypes = args
    return lib


lib = load_library()


class B200Error(RuntimeError):
    """A libprysm_b200 call failed (CUDA error, unsupported shape, bad argument)."""


class Handle:
    """One engine handle per CUDA device (twiddle tables + scratch live here)."""

    def __init__(self, device):
        self._h = C.c_void_p()
        rc = lib.pb_create(C.byref(self._h), int(device))
        if rc != 0:
            raise B200Error(f'pb_create(device={device}) failed with status {rc}: is a CUDA device visible?')
        self.device = int(device)

    def check(self, rc):
        if rc != OK:
            msg = lib.pb_last_error(self._h).decode()
            if rc == ERR_INVALID:
                raise ValueError(msg)
            raise B200Error(f'status {rc}: {msg}')

    @property
    def ptr(self):
        return self._h

    def launch_count(self):
        return int(lib.pb_launch_count(self._h))

    def route_launch_count(self, route):
        """kernels launched on one route of the transform kernels (pb_route_launch_count)"""
        return int(lib.pb_route_launch_count(self._h, int(route)))

    def close(self):
        if self._h:
            lib.pb_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


_handles = {}          # (device, raw stream pointer) -> Handle, in least-recently-used order
_pinned = set()        # keys whose handle must outlive the cache (a captured CUDA graph replays into its scratch)
MAX_HANDLES_PER_DEVICE = 8


def handle_for(device_index, stream=0):
    """One handle per (device, stream): a handle's scratch arenas are only ordered by the stream its calls run
    on, so work issued on different streams must not share one (include/prysm_b200.h: 'not thread-safe').
    The cache is bounded: beyond MAX_HANDLES_PER_DEVICE the least recently used un-pinned handle of that device is
    destroyed (pb_destroy synchronises the device first), so short-lived side streams do not accumulate twiddle
    tables and scratch arenas that torch's allocator cannot see."""
    key = (device_index, stream)
    h = _handles.pop(key, None)
    if h is None:
        mine = [k for k in _handles if k[0] == device_index and k not in _pinned]
        while len(mine) >= MAX_HANDLES_PER_DEVICE:
            _handles.pop(mine.pop(0)).close()
        h = Handle(device_index)
    _handles[key] = h          # (re)insert as most recently used
    return h


def pin_handle(device_index, stream):
    """Keep the handle of (device, stream) alive for the life of the process (graphs.capture)."""
    _pinned.add((device_index, stream))


def release_handle(device_index, stream):
    """Destroy the handle of (device, stream) now (explicit close of a side stream's engine state)."""
    _pinned.discard((device_index, stream))
    h = _handles.pop((device_index, stream), None)
    if h is not None:
        h.close()


def launch_count(device_index):
    """Kernels launched on `device_index` through any stream's handle."""
    return sum(h.launch_count() for (d, _), h in _handles.items() if d == device_index)


def version():
    return lib.pb_version().decode()
