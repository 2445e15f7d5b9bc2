"""GPU: the CUDA path against the CPU oracle on RANDOM shapes and parameters (hypothesis; derandomised so every box
runs the same examples) -- ragged / odd / prime sizes, fractional Q, shifted focal grids, both precisions.
Tolerances: complex128 1e-11, complex64 2e-6 (relative L-inf vs the fp64 oracle)."""
import numpy as np
import pytest
from hypothesis import given, settings, strategies as st, HealthCheck

import prysm_oracle as O
from conftest import rel_linf
from gpu_fixtures import pb, host  # noqa: F401

pytestmark = pytest.mark.gpu
HeNe = 0.6328
SETTINGS = dict(max_examples=20, deadline=None, derandomize=True,
                suppress_health_check=[HealthCheck.too_slow, HealthCheck.function_scoped_fixture])
shapes = st.tuples(st.integers(1, 40), st.integers(1, 40))


def crand(rng, shape, cdt):
    return (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype(cdt)


def prec(pb, p64):
    pb.config.precision = 64 if p64 else 32
    return (np.complex128, 1e-11) if p64 else (np.complex64, 2e-6)


@given(shape=shapes, Q=st.sampled_from([1, 1.5, 2, 3]), p64=st.booleans(), seed=st.integers(0, 999))
@settings(**SETTINGS)
def test_focus_family_random_shapes(pb, shape, Q, p64, seed):
    cdt, tol = prec(pb, p64)
    rng = np.random.default_rng(seed)
    P = pb.propagation
    a = crand(rng, shape, cdt)
    a64 = a.astype(np.complex128)
    f = P.focus(a, Q)
    assert rel_linf(host(f), O.focus(a64, Q)) < tol
    assert rel_linf(host(P.unfocus(a, Q)), O.unfocus(a64, Q)) < tol
    g = crand(rng, tuple(f.shape), cdt)
    assert rel_linf(host(P.focus_adjoint(g, Q)), O.focus_adjoint(g.astype(np.complex128), Q)) < tol
    assert rel_linf(host(P.unfocus_adjoint(g, Q)), O.unfocus_adjoint(g.astype(np.complex128), Q)) < tol


@given(n=st.tuples(st.integers(2, 28), st.integers(2, 28)), m=st.tuples(st.integers(2, 28), st.integers(2, 28)),
       kind=st.sampled_from(['mdft', 'czt']), shift=st.tuples(st.floats(-3, 3), st.floats(-3, 3)), p64=st.booleans(),
       seed=st.integers(0, 999))
@settings(**SETTINGS)
def test_executors_random_geometry(pb, n, m, kind, shift, p64, seed):
    cdt, tol = prec(pb, p64)
    tol = tol if p64 else 4e-6          # fp32 Bluestein on random data
    rng = np.random.default_rng(seed)
    a, g = crand(rng, n, cdt), crand(rng, m, cdt)
    args = (0.1, n, 1.7, m, HeNe, 50.0, shift)
    ex = pb.propagation.prepare_executor(*args, kind=kind)
    exo = O.prepare_executor(*args, kind)
    assert rel_linf(host(ex(a)), exo(a.astype(np.complex128))) < tol
    assert rel_linf(host(ex.adjoint(g)), exo.adjoint(g.astype(np.complex128))) < tol


@given(shape=st.tuples(st.integers(2, 40), st.integers(2, 40)), Q=st.sampled_from([1, 2]), z=st.floats(-30, 30),
       p64=st.booleans(), seed=st.integers(0, 999))
@settings(**SETTINGS)
def test_angular_spectrum_random_shapes(pb, shape, Q, z, p64, seed):
    cdt, tol = prec(pb, p64)
    rng = np.random.default_rng(seed)
    a = crand(rng, shape, cdt)
    got = pb.propagation.angular_spectrum(a, HeNe, 0.05, z, Q)
    assert rel_linf(host(got), O.angular_spectrum(a.astype(np.complex128), HeNe, 0.05, z, Q)) < tol
    g = crand(rng, tuple(got.shape), cdt)
    assert rel_linf(host(pb.propagation.angular_spectrum_adjoint(g, HeNe, 0.05, z, Q)),
                    O.angular_spectrum_adjoint(g.astype(np.complex128), HeNe, 0.05, z, Q)) < tol


@given(shape=st.tuples(st.integers(2, 24), st.integers(2, 24)), fshape=st.tuples(st.integers(2, 24), st.integers(2, 24)),
       cplx=st.booleans(), p64=st.booleans(), seed=st.integers(0, 999))
@settings(**SETTINGS)
def test_coronagraph_random_shapes(pb, shape, fshape, cplx, p64, seed):
    cdt, tol = prec(pb, p64)
    tol = tol if p64 else 4e-6
    rng = np.random.default_rng(seed)
    P = pb.propagation
    x = crand(rng, shape, cdt)
    fpm = crand(rng, fshape, cdt) if cplx else rng.standard_normal(fshape).astype(x.real.dtype)
    lyot = rng.standard_normal(shape).astype(x.real.dtype)
    ex = P.prepare_executor(0.25, shape, 0.1, fshape, HeNe, 10.0)
    exo = O.prepare_executor(0.25, shape, 0.1, fshape, HeNe, 10.0)
    x64, f64, l64 = x.astype(np.complex128), fpm.astype(np.complex128 if cplx else np.float64), lyot.astype(np.float64)
    assert rel_linf(host(P.to_fpm_and_back(x, fpm, ex)), O.to_fpm_and_back(x64, f64, exo)) < tol
    assert rel_linf(host(P.babinet(x, lyot, fpm, ex)), O.babinet(x64, l64, f64, exo)) < tol
    assert rel_linf(host(P.babinet_adjoint(x, lyot, fpm, ex)), O.babinet_adjoint(x64, l64, f64, exo)[0]) < tol


@given(shape=st.tuples(st.integers(1, 30), st.integers(1, 30)), p64=st.booleans(), seed=st.integers(0, 999))
@settings(**SETTINGS)
def test_image_chain_random_shapes(pb, shape, p64, seed):
    cdt, tol = prec(pb, p64)
    rdt = np.float64 if p64 else np.float32
    rng = np.random.default_rng(seed)
    o, h = rng.random(shape).astype(rdt), rng.random(shape).astype(rdt)
    assert rel_linf(host(pb.convolution.conv(o, h)), O.conv(o.astype(np.float64), h.astype(np.float64))) < tol
    psf = rng.random(shape).astype(rdt) + 0.1
    mtf = pb.otf.mtf_from_psf(psf, 1.5)
    assert np.abs(host(mtf.data) - O.mtf_from_psf(psf.astype(np.float64), 1.5)[0]).max() < (1e-11 if p64 else 5e-6)
