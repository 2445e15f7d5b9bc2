"""GPU: the register-engine axis passes (L in {1024, 2048, 4096}) behind pb_fft2 / pb_axis_dft /
pb_angular_spectrum, against numpy fp64 and against the generic shared-memory kernel."""
import numpy as np
import pytest

import prysm_oracle as O
from conftest import rel_linf
from gpu_fixtures import pb  # noqa: F401

pytestmark = pytest.mark.gpu
HeNe = 0.6328


def crand(shape, seed):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype(np.complex64)


@pytest.mark.parametrize('shape', [(1024, 1024), (2048, 1024), (1024, 4096), (4096, 2048), (1026, 2048)])
def test_plain_fft2_and_centred(pb, shape):
    from prysm_b200 import _ops
    a = crand(shape, shape[0] + shape[1])
    d = pb.asdevice(a)
    ref = np.fft.fft2(a.astype(np.complex128))
    assert rel_linf(_ops.fft2(d, shape, dir=-1).cpu().numpy(), ref) < 1e-6
    inv = np.fft.ifft2(a.astype(np.complex128))
    assert rel_linf(_ops.fft2(d, shape, dir=+1, scale=1.0 / (shape[0] * shape[1])).cpu().numpy(), inv) < 1e-6
    # centred (Q = 1 focus) and cropped adjoint
    assert rel_linf(pb.propagation.focus(d, 1).cpu().numpy(), O.focus(a.astype(np.complex128), 1)) < 1e-6
    assert rel_linf(pb.propagation.unfocus_adjoint(d, 2).cpu().numpy(), O.unfocus_adjoint(a.astype(np.complex128), 2)) < 1e-6


def test_odd_line_count_and_padding(pb):
    a = crand((1023, 700), 5)                       # 1023 populated rows, padded to 1024 x 1024, odd batch
    out = pb.propagation.focus(a, 1024 / 1023 if False else 1)  # Q=1: Bluestein for 1023/700 (generic) -- sanity
    assert rel_linf(out.cpu().numpy(), O.focus(a.astype(np.complex128), 1)) < 2e-6
    b = crand((512, 400), 6)
    from prysm_b200 import _ops
    out = _ops.fft2(pb.asdevice(b), (1024, 2048), dir=-1, shift_in=True, shift_out=True)   # pad 512x400 -> 1024x2048
    ref = np.fft.fftshift(np.fft.fft2(np.fft.ifftshift(O.pad2d(b.astype(np.complex128), out_shape=(1024, 2048)))))
    assert rel_linf(out.cpu().numpy(), ref) < 1e-6


def test_angular_spectrum_and_czt_large(pb):
    P = pb.propagation
    pb.config.precision = 32
    f = crand((1024, 1024), 9)
    ref = O.angular_spectrum(f.astype(np.complex128), HeNe, 0.01, 25.0, 1)
    assert rel_linf(P.angular_spectrum(f, HeNe, 0.01, 25.0, 1).cpu().numpy(), ref) < 1e-6
    ref2 = O.angular_spectrum(f[:512, :512].astype(np.complex128), HeNe, 0.01, 25.0, 2)
    assert rel_linf(P.angular_spectrum(f[:512, :512].copy(), HeNe, 0.01, 25.0, 2).cpu().numpy(), ref2) < 1e-6
    a = crand((1024, 1024), 10)
    ex = P.prepare_executor(0.01, (1024, 1024), 1.5, (512, 512), HeNe, 100.0, (2.0, -1.0), 'czt')   # K = 2048
    exo = O.prepare_executor(0.01, (1024, 1024), 1.5, (512, 512), HeNe, 100.0, (2.0, -1.0), 'czt')
    assert rel_linf(ex(a).cpu().numpy(), exo(a.astype(np.complex128))) < 3e-6
    g = crand((512, 512), 11)
    assert rel_linf(ex.adjoint(g).cpu().numpy(), exo.adjoint(g.astype(np.complex128))) < 3e-6
    pb.config.precision = 64


def test_psf_to_mtf_4096(pb):
    """psf -> mtf at the headline PSF size: real input (generic first pass) + tuned column pass."""
    rng = np.random.default_rng(3)
    psf = rng.random((2048, 2048)).astype(np.float32)
    got = pb.otf.mtf_from_psf(psf, 1.0).data.cpu().numpy()
    ref, _ = O.mtf_from_psf(psf.astype(np.float64), 1.0)
    assert np.abs(got - ref).max() < 2e-6
