"""CPU: the long-double reference of tests/test_gpu_generic_axis_vs_fp64.py, and proof that its ceilings would catch a
subtly wrong Bluestein.  Numpy models of the device's Bluestein (the get_chirp, get_chirp_filter and bluestein_len rules
of csrc/fft2.cu) run faithfully land under the complex128 ceiling of 1e-14 (fp64 arithmetic) or the complex64 ceiling
of 1e-6 (fp32 arithmetic); each modelled defect lands at least 10x above it."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import scipy.fft as sfft

import generic_reference as G
from generic_reference import PB_C64, PB_C128
from gpu_fixtures import crand


# ---- the long-double helpers against closed forms -------------------------------------------------------------------
def test_long_double_is_extended():
    assert np.finfo(np.longdouble).eps < 1.2e-19
    assert sfft.fft(np.ones(8, dtype=G.LD)).dtype == G.LD


@pytest.mark.parametrize('n', (7, 1000, 4096, 8191))
def test_fft_ld_of_impulses_and_ramps(n):
    """an impulse at p transforms to exp(-2 pi i k p / n); a ramp exp(2 pi i q j / n) to n delta[k - q]"""
    k = np.arange(n)
    for p in (0, 1, n // 2, n - 1):
        x = np.zeros(n, dtype=G.LD)
        x[p] = 1
        err = np.abs(G.fft_ld(x) - G.ramp_ld(k, p, n, -1)).max()
        assert err < 1e-17, (p, err)
        err = np.abs(G.fft_ld(x, inverse=True) - G.ramp_ld(k, p, n, +1)).max()
        assert err < 1e-17, (p, err)
    q = n // 3
    X = G.fft_ld(G.ramp_ld(k, q, n, +1))
    want = np.zeros(n, dtype=G.LD)
    want[q] = n
    assert np.abs(X - want).max() / n < 1e-17


@pytest.mark.parametrize('inverse', (False, True))
@pytest.mark.parametrize('n,k,crop', [((5, 4), (9, 12), None), ((64, 63), (96, 95), (95, 94)), ((255, 255), (383, 383), None)])
def test_impulse_closed_form_matches_fft(n, k, crop, inverse):
    """centred_ft2_ld (an FFT) and impulse_centred_ft2 (no FFT) agree, odd and even sizes and crops"""
    px = [(0, 0), (n[0] // 2, n[1] // 2), (n[0] - 1, 1)]
    vals = [1 + 0.5j, -0.25 + 1j, 0.75]
    a = np.zeros(n, dtype=G.LD)
    for p, v in zip(px, vals):
        a[p] += v
    got = G.impulse_centred_ft2(n, k, px, vals, inverse=inverse, crop=crop)
    ref = G.centred_ft2_ld(a, k, inverse=inverse, crop=crop)
    assert np.abs(got - ref).max() / np.abs(ref).max() < 1e-17


def test_phase_field_ld():
    """exp(2 pi i turns) with the turns reduced exactly, against the closed values at quarter turns"""
    kscale = 2 * np.pi / 0.6328 / 1e3
    kturns = kscale / (2 * np.pi)
    opd = np.array([0.0, 0.25, 0.5, -0.75, 1e4 + 0.25], dtype=np.float64) / kturns
    turns = kturns * opd
    e = G.phase_field_ld(opd, kscale)
    ref = np.exp(2j * np.pi * (turns.astype(np.longdouble) - np.round(turns.astype(np.longdouble)))).astype(G.LD)
    assert np.abs(e - ref).max() < 3e-16           # the fp64 exp of the reference check, not of phase_field_ld
    assert np.abs(np.abs(e) - 1).max() < 1e-18
    e = G.phase_field_ld(opd, kscale, amp=np.array([0, 1, 2, 0, 1], dtype=np.uint8))
    assert e[0] == 0 and e[3] == 0 and abs(abs(e[2]) - 1) < 1e-18


# ---- the Bluestein models against the ceilings ------------------------------------------------------------------------
def _fig(dtype, n, defect=None, seed=0, dir=-1):
    x = crand((2, n), seed + n, G.CPLX[dtype])
    y = G.bluestein_model(x, dtype, defect, dir)
    ref = G.fft_ld(x, inverse=dir > 0)
    return G.rel_linf(y, ref)


@pytest.mark.parametrize('dir', (-1, 1))
@pytest.mark.parametrize('n', (97, 1000, 4095))
def test_faithful_fp64_model_under_the_complex128_ceiling(n, dir):
    f = _fig(PB_C128, n, dir=dir)
    assert f < G.CEILING[PB_C128] / 3, f


@pytest.mark.parametrize('n', (97, 1000, 8191))
def test_faithful_fp32_model_under_the_complex64_ceiling(n):
    f = _fig(PB_C64, n)
    assert f < G.CEILING[PB_C64] / 2, f


@pytest.mark.parametrize('defect', ('unreduced', 'angle32', 'twiddle32', 'mirror_off', 'filter_conj', 'window_off'))
@pytest.mark.parametrize('n', (1000, 4095))
def test_fp64_defects_land_10x_over_the_complex128_ceiling(n, defect):
    f = _fig(PB_C128, n, defect)
    assert f > 10 * G.CEILING[PB_C128], (defect, f)


@pytest.mark.parametrize('defect', ('jj32', 'mirror_off', 'filter_conj', 'window_off'))
def test_fp32_defects_land_10x_over_the_complex64_ceiling(defect):
    f = _fig(PB_C64, 8191, defect)
    assert f > 10 * G.CEILING[PB_C64], (defect, f)


def test_jj32_is_exact_below_4097():
    """j*j in float32 is exact for j <= 4096: the fp32 defect only shows on the long lengths the GPU test runs"""
    assert _fig(PB_C64, 4095, 'jj32') == _fig(PB_C64, 4095)


# ---- the launch and length rules --------------------------------------------------------------------------------------
def test_length_limits_for_the_h100_cap():
    cap = G.SMEM_OPTIN_H100
    assert G.max_pow2_len(PB_C64, cap) == 16384 and G.max_pow2_len(PB_C128, cap) == 8192
    assert G.max_len(PB_C64, cap) == 8192 and G.max_len(PB_C128, cap) == 4096
    for dt, lmax in ((PB_C64, 16384), (PB_C128, 8192)):
        assert G.accepts(lmax, dt) and not G.accepts(2 * lmax, dt)
        assert G.accepts(lmax // 2 - 1, dt) and not G.accepts(lmax // 2 + 1, dt)
        # every length up to lmax / 2, then powers of two only
        ok = [n for n in range(1, 2 * lmax + 1) if G.accepts(n, dt)]
        assert ok == list(range(1, lmax // 2 + 1)) + [lmax]
        for n in range(1, lmax // 2 + 1):
            L = n if G.is_pow2(n) else G.bluestein_len(n)
            assert L * G.CSIZE[dt] <= cap


def test_launch_rule():
    assert G.axis_launches(1, PB_C64, 0) == {(1, PB_C64, 0): 1}
    assert G.axis_launches(4096, PB_C128, 1) == {(4096, PB_C128, 1): 1}
    assert G.axis_launches(3, PB_C64, 1) == {(8, PB_C64, 1): 2}
    assert G.axis_launches(1000, PB_C128, 0) == {(2048, PB_C128, 0): 2}
    assert G.axis_launches(1025, PB_C128, 0) == {(4096, PB_C128, 0): 2}
    assert G.axis_launches(8191, PB_C64, 0) == {(16384, PB_C64, 0): 2}
    for n in range(2, 3000):
        M = G.bluestein_len(n)
        assert G.is_pow2(M) and 2 * n - 1 <= M < 2 * (2 * n - 1)
    assert G.merge({(8, 0, 0): 2}, {(8, 0, 0): 1, (4, 0, 1): 1}) == {(8, 0, 0): 3, (4, 0, 1): 1}


# ---- the same rules, compiled from the C++ sources ------------------------------------------------------------------
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'prysm_b200', 'csrc')


def _extract(fname, pattern):
    with open(os.path.join(CSRC, fname)) as fh:
        m = re.search(pattern, fh.read(), re.S)
    assert m, f'{pattern!r} not found in {fname}'
    return m.group(0)


HARNESS = r'''
#include <cstdio>
#include <cstdlib>
#include <cstddef>
#include <string>
enum { PB_C64 = 0, PB_C128 = 1, PB_ERR_UNSUPPORTED = -2 };
struct Handle { int max_smem_optin; };
static std::string last;
static int fail(Handle*, int code, const std::string& m) { last = m; return code; }
%(is_pow2)s
%(csize)s
%(bluestein_len)s
%(generic_max_len)s
struct Pass { int dtype; int Llog; };
static int refuse(Handle* h, Pass p) {
    const int n = p.Llog;
    %(refusal)s
    return 0;
}
int main(int argc, char** argv) {
    Handle h{atoi(argv[1])};
    for (int n = 1; n <= 20000; ++n) printf("%%d ", bluestein_len(n));
    printf("\n");
    for (int dt = 0; dt < 2; ++dt) {
        const int lmax = generic_max_len(&h, dt);
        printf("%%d\n", lmax);
        for (int n = 1; n <= 2 * lmax + 2; ++n) putchar(refuse(&h, Pass{dt, n}) ? '0' : '1');
        printf("\n");
        refuse(&h, Pass{dt, lmax / 2 + 1});
        printf("%%s\n", last.c_str());
    }
    return 0;
}
'''


@pytest.fixture(scope='module')
def cxx_rules(tmp_path_factory):
    """generic_max_len (axis_pass.cu), bluestein_len and axis_dft's refusal (fft2.cu), is_pow2 and csize (common.cuh),
    copied out of the sources and compiled for the host"""
    cxx = shutil.which('g++') or shutil.which('c++')
    if cxx is None:
        pytest.skip('no host C++ compiler')
    src = HARNESS % dict(
        is_pow2=_extract('common.cuh', r'inline bool is_pow2\(int n\) \{[^\n]*\}'),
        csize=_extract('common.cuh', r'inline size_t csize\(int dtype\) \{[^\n]*\}'),
        bluestein_len=_extract('fft2.cu', r'static int bluestein_len\(int n\) \{[^\n]*\}'),
        generic_max_len=_extract('axis_pass.cu', r'int generic_max_len\(const Handle\* h, int dtype\) \{.*?\n\}'),
        refusal=_extract('fft2.cu', r'const int lmax = generic_max_len\(h, p\.dtype\);.*?\n    \}'))
    d = tmp_path_factory.mktemp('cxx_rules')
    with open(d / 'rules.cpp', 'w') as fh:
        fh.write(src)
    subprocess.run([cxx, '-std=c++17', '-O1', '-o', str(d / 'rules'), str(d / 'rules.cpp')], check=True)
    return lambda cap: subprocess.run([str(d / 'rules'), str(cap)], check=True, capture_output=True,
                                      text=True).stdout.splitlines()


@pytest.mark.parametrize('cap', (G.SMEM_OPTIN_H100, 100000, 49152))
def test_helpers_agree_with_the_cxx_rules(cxx_rules, cap):
    out = cxx_rules(cap)
    assert [int(v) for v in out[0].split()] == [G.bluestein_len(n) for n in range(1, 20001)]
    for dt, (lmax, flags, msg) in zip((PB_C64, PB_C128), (out[1:4], out[4:7])):
        lmax = int(lmax)
        assert lmax == G.max_pow2_len(dt, cap)
        assert flags == ''.join('1' if G.accepts(n, dt, cap) else '0' for n in range(1, 2 * lmax + 3))
        n = lmax // 2 + 1
        name = 'complex64' if dt == PB_C64 else 'complex128'
        for word in (f'{name} FFT of length {n} ', f'({cap} B)', f'any length up to {G.max_len(dt, cap)} ',
                     f'powers of two up to {lmax}'):
            assert word in msg, (word, msg)
