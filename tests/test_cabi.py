"""CPU: the C-ABI library builds for sm_90a, loads, and exports exactly the symbols
include/prysm_b200.h declares (no compute calls here -- there is no GPU on this box)."""
import ctypes
import os
import re

import pytest

from conftest import ROOT


def _header_code():
    src = open(os.path.join(ROOT, 'include', 'prysm_b200.h')).read()
    return re.sub(r'/\*.*?\*/', '', src, flags=re.S)


def header_symbols():
    return sorted(set(re.findall(r'\b(pb_[a-z0-9_]+)\s*\(', _header_code())))


def header_prototypes():
    """name -> [restype, parameter types...] of every prototype in the header, as C type text"""
    protos = {}
    for ret, name, params in re.findall(r'^([A-Za-z_][\w ]*?\**)\s*(pb_[a-z0-9_]+)\s*\(([^)]*)\)\s*;', _header_code(),
                                        flags=re.M):
        params = [' '.join(p.split()) for p in params.split(',')] if params.strip() not in ('', 'void') else []
        # drop the parameter name, keep its type (every parameter in the header is named)
        protos[name] = [ret.strip()] + [re.sub(r'\b\w+$', '', p).strip() for p in params]
    return protos


def _ctype_of(c_type):
    if '*' in c_type or c_type == 'pb_handle_t':
        return 'pointer'
    return {'int': ctypes.c_int, 'long long': ctypes.c_longlong, 'double': ctypes.c_double}[c_type]


def _ctypes_kind(t):
    if t in (ctypes.c_void_p, ctypes.c_char_p) or issubclass(t, ctypes._Pointer):
        return 'pointer'
    return t


def test_library_exports_every_header_symbol():
    from prysm_b200 import _capi
    lib = ctypes.CDLL(_capi.LIB_PATH)
    names = header_symbols()
    assert len(names) >= 18
    for n in names:
        assert hasattr(lib, n), f'{n} declared in the header but not exported'
    assert sorted(_capi.SIGNATURES) == names, 'ctypes SIGNATURES and the header diverge'
    # an int / long long slip at one position passes garbage in the upper half of a register: compare every position
    protos = header_prototypes()
    assert sorted(protos) == names
    for name, (res, args) in _capi.SIGNATURES.items():
        want = [_ctype_of(t) for t in protos[name]]
        got = [_ctypes_kind(t) for t in [res] + list(args)]
        assert len(got) == len(want), f'{name}: {len(args)} ctypes arguments, the header has {len(want) - 1}'
        for i, (g, w) in enumerate(zip(got, want)):
            assert g == w, f'{name}: ' + ('return type' if i == 0 else f'argument {i - 1}') + f' is {g}, the header says {w}'


def test_version_and_null_handle_are_safe():
    from prysm_b200 import _capi
    assert 'sm_90a' in _capi.version()
    assert _capi.lib.pb_last_error(None) == b'null handle'
    assert _capi.lib.pb_launch_count(None) == 0
    assert _capi.lib.pb_mdft_work_elems(512, 4096, 512, 4096, 0, 1) == 512 * 4096


def test_no_cpu_fallback_without_device():
    """On a box without a GPU the product must fail loudly, not silently compute on the host."""
    import torch
    if torch.cuda.is_available():
        pytest.skip('a GPU is present')
    import numpy as np
    from prysm_b200 import propagation, _capi
    with pytest.raises(_capi.B200Error):
        propagation.focus(np.ones((8, 8), dtype=np.complex64), 2)


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, 'prysm_b200')
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(('.py', '.cu', '.cuh', '.h')):
                txt = open(os.path.join(dirpath, f)).read()
                assert 'prysm_oracle' not in txt and 'import oracle' not in txt, f


def test_python_constants_match_the_header_enums():
    """The integer codes the ctypes layer passes are the enum values the header declares: every PB_NAME is
    _capi.NAME, except PB_C64 and PB_C128, which keep their names."""
    from prysm_b200 import _capi
    src = open(os.path.join(ROOT, 'include', 'prysm_b200.h')).read()
    enums = {k: int(v) for k, v in re.findall(r'\b(PB_[A-Z0-9_]+)\s*=\s*(-?\d+)', src)}
    assert len(enums) >= 152
    for name, val in enums.items():
        assert getattr(_capi, name if name in ('PB_C64', 'PB_C128') else name[3:]) == val, name
    assert enums['PB_OK'] == 0 and enums['PB_ERR_INVALID'] == -1      # Handle.check maps -1 to ValueError


@pytest.mark.parametrize('decl', ['int pb_g(pb_handle_t h, float x);', 'enum { PB_A = 1, PB_B };',
                                  'int pb_g(int n) { return n; }'])
def test_read_header_refuses_what_it_cannot_bind(tmp_path, decl):
    """A C type without a ctypes mapping, an enumerator without a literal value or a declaration the reader cannot
    parse fails the import: the binding never guesses an argument type or a code."""
    from prysm_b200 import _capi
    path = tmp_path / 'api.h'
    path.write_text('enum { PB_K = -2 };\nlong long pb_f(pb_handle_t h, const double* x, int n, double s);\n')
    assert _capi.read_header(str(path)) == (
        {'pb_f': (ctypes.c_longlong, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_double])}, {'PB_K': -2})
    path.write_text(path.read_text() + decl + '\n')
    with pytest.raises(ImportError, match=re.escape(str(path))):
        _capi.read_header(str(path))


def test_only_tests_smoke_and_bench_touch_the_oracle():
    """oracle/ is test infrastructure: nothing outside tests/, bench.py and __graft_entry__.py may import it."""
    allowed = {os.path.join(ROOT, 'bench.py'), os.path.join(ROOT, '__graft_entry__.py')}
    for dirpath, dirs, files in os.walk(ROOT):
        dirs[:] = [d for d in dirs if d not in ('.git', 'tests', 'oracle', '__pycache__', '.pytest_cache')]
        for f in files:
            path = os.path.join(dirpath, f)
            if f.endswith('.py') and path not in allowed:
                assert 'prysm_oracle' not in open(path).read(), path


def test_header_is_valid_c99_and_the_c_example_links():
    """The boundary is a C ABI: the header must compile as plain C (not only as C++), and the example that calls it
    from C must link against the built library."""
    import shutil
    import subprocess
    import tempfile
    from prysm_b200 import _capi
    gcc = shutil.which('gcc')
    if gcc is None:
        pytest.skip('no gcc on this box')
    src = os.path.join(ROOT, 'examples', 'focus_from_c.c')
    inc = os.path.join(ROOT, 'include')
    r = subprocess.run([gcc, '-std=c99', '-Wall', '-Wextra', '-pedantic', '-Werror', '-I', inc, '-fsyntax-only', src],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    cudart = '/usr/local/cuda/lib64'
    if os.path.isdir(cudart):
        with tempfile.TemporaryDirectory() as d:
            r = subprocess.run([gcc, '-std=c99', '-I', inc, src, '-L', os.path.dirname(_capi.LIB_PATH), '-lprysm_b200',
                                '-L', cudart, '-lcudart', '-o', os.path.join(d, 'focus_from_c')], capture_output=True, text=True)
            assert r.returncode == 0, r.stderr


def test_every_entry_point_rejects_a_null_handle():
    """No entry point may dereference a NULL handle: each returns PB_ERR_INVALID (-1) instead (nothing crosses the
    boundary as a crash).  Needs no GPU -- the check is the first thing every call does."""
    from prysm_b200 import _capi
    no_handle = {'pb_create', 'pb_destroy', 'pb_last_error', 'pb_version', 'pb_launch_count', 'pb_mdft_work_elems',
                 'pb_mdft_tc_supported', 'pb_mdft_tc_work_bytes', 'pb_polychromatic_czt_work_bytes'}
    checked = 0
    for name, (_, args) in _capi.SIGNATURES.items():
        if name in no_handle:
            continue
        vals = []
        for a in args:
            if a in (ctypes.c_int, ctypes.c_longlong):
                vals.append(0)
            elif a is ctypes.c_double:
                vals.append(0.0)
            else:
                vals.append(None)       # pointers, including the handle
        assert getattr(_capi.lib, name)(*vals) == -1, name
        checked += 1
    assert checked == len(_capi.SIGNATURES) - len(no_handle)
