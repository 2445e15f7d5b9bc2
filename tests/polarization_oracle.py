"""The polarization cases the engine is checked on (prysm/x/polarization.py) and the writer of
tests/golden/polarization*.npz.

    PYTHONDONTWRITEBYTECODE=1 python tests/polarization_oracle.py   (needs the unmodified reference: PRYSM_REFERENCE or
                                                                      oracle/_ref)

The fixtures are the REFERENCE's own outputs at precision 64, from the inputs `inputs()` builds.  `run(pol, prop, ...)`
computes every case with a polarization module and a propagation module given: the reference's with numpy arrays, or
the engine's (tests/test_gpu_polarization.py).  The propagation cases go through `pol.jones_adapter` directly, so that
running them patches no module.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (ROOT, os.path.join(ROOT, 'oracle')):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import reference  # noqa: E402

SHAPE = (61, 80)           # (rows, cols): non-square, odd rows
PROP_N = 256               # the reference's test_make_propagation_polarized (tests/x/test_polarization.py:129-183)
VVC_N = 128                # the vector vortex coronagraph
WINDOW = 48                # centred window of the 256^2 propagation outputs that is stored


def grid(n, diameter):
    """make_xy_grid(n, diameter=diameter) and its polar form, in fp64."""
    x = (np.arange(n) - n // 2) * (diameter / n)
    xx, yy = np.meshgrid(x, x)
    return xx, yy, np.hypot(xx, yy), np.arctan2(yy, xx)


def inputs():
    """Every input array of the cases, fp64 / complex128 host arrays."""
    rng = np.random.default_rng(20261015)
    ny, nx = SHAPE
    y, x = np.mgrid[:ny, :nx]
    g = {
        'theta': np.arctan2(y - ny // 2 + 0.5, x - nx // 2 + 0.25),
        'retardance': rng.uniform(0, 2 * np.pi, SHAPE),
        'alpha': rng.uniform(0, 1, SHAPE),
        'angle_deg': rng.uniform(-180, 180, SHAPE),
        'J': rng.standard_normal(SHAPE + (2, 2)) + 1j * rng.standard_normal(SHAPE + (2, 2)),
        'K': rng.standard_normal(SHAPE + (2, 2)) + 1j * rng.standard_normal(SHAPE + (2, 2)),
        'field': rng.standard_normal(SHAPE) + 1j * rng.standard_normal(SHAPE),
    }
    _, _, r, _ = grid(PROP_N, 10)
    g['A'] = (r <= 5).astype(np.float64)
    xx, yy, r, _ = grid(VVC_N, 10)
    g['vvc_amp'] = (r <= 5).astype(np.float64)
    g['vvc_phase'] = 0.3 * (xx * yy) / 25 + 0.1 * (2 * (r / 5) ** 2 - 1)
    g['vvc_lyot'] = (r <= 4.5).astype(np.float64)
    return g


# ---- vector vortex coronagraph geometry (128^2, focal plane 128^2 at 0.25 lambda/D) ------------------------------
VVC = dict(wavelength=0.55, efl=100.0, pupil_dx=10 / VVC_N, focal_samples=VVC_N)
VVC['focal_dx'] = VVC['wavelength'] * VVC['efl'] / 10 / 4


def constructors(pol, g, to_numpy=np.asarray):
    """Every constructor at the fixture shape, scalar and per-pixel parameters."""
    c = {
        'rotation': pol.jones_rotation_matrix(0.37, shape=SHAPE),
        'rotation_plane': pol.jones_rotation_matrix(g['theta'], shape=SHAPE),
        'rotation_2x2': pol.jones_rotation_matrix(-1.1),
        'retarder': pol.linear_retarder(0.9, theta=0.3, shape=SHAPE),
        'retarder_plane': pol.linear_retarder(g['retardance'], theta=0.3, shape=SHAPE),
        'retarder_2x2': pol.linear_retarder(2.1, theta=-0.4),
        'diattenuator': pol.linear_diattenuator(0.4, theta=-0.7, shape=SHAPE),
        'diattenuator_2x2': pol.linear_diattenuator(0.8, theta=0.2),
        'half_wave': pol.half_wave_plate(theta=0.5, shape=SHAPE),
        'quarter_wave': pol.quarter_wave_plate(theta=-0.25, shape=SHAPE),
        'polarizer': pol.linear_polarizer(theta=1.2, shape=SHAPE),
        'vvr': pol.vector_vortex_retarder(2, g['theta'].copy()),
        'vvr_rotated': pol.vector_vortex_retarder(3, g['theta'].copy(), retardance=0.8 * np.pi, rotate=0.3),
        'linear_vector': pol.linear_pol_vector(g['angle_deg']),
        'linear_vector_rad': pol.linear_pol_vector(g['theta'], degrees=False),
        'linear_vector_2': pol.linear_pol_vector(30),
        'circular_left': pol.circular_pol_vector('left'),
        'circular_right': pol.circular_pol_vector('right'),
    }
    for i in range(4):
        c[f'pauli{i}'] = pol.pauli_spin_matrix(i, shape=SHAPE)
        c[f'pauli{i}_2x2'] = pol.pauli_spin_matrix(i)
    return {k: to_numpy(v) for k, v in c.items()}


def diattenuator_plane(pol, alpha):
    """linear_diattenuator(alpha, theta=-0.6) with a per-pixel alpha, built from the reference's own steps
    (polarization.py:224-231): the reference function itself accepts only a scalar (its range assert takes the truth
    value of alpha)."""
    jones = pol._empty_jones(shape=alpha.shape)
    jones[..., 0, 0] = 1
    jones[..., 1, 1] = alpha
    return pol.jones_rotation_matrix(0.6) @ jones @ pol.jones_rotation_matrix(-0.6)


def reductions(pol, g, to_numpy=np.asarray):
    out = {
        'mueller': pol.jones_to_mueller(g['J']),
        'mueller_2x2': pol.jones_to_mueller(g['J'][3, 5]),
        'kron': pol.broadcast_kron(g['J'][:30], g['K'][:30]),       # 16 planes: half the rows keep a part < 1 MB
        'pauli_coefficients': pol.pauli_coefficients(g['J']),
        'optic_scalar_field': pol.apply_polarization_optic(g['field'], g['J']),
        'optic_jones_field': pol.apply_polarization_optic(g['K'], g['J']),
    }
    out['pauli_coefficients'] = np.stack([to_numpy(v) for v in out['pauli_coefficients']])
    return {k: to_numpy(v) for k, v in out.items()}


def window(a, w=WINDOW):
    cy, cx = a.shape[0] // 2, a.shape[1] // 2
    return a[cy - w // 2:cy + w // 2, cx - w // 2:cx + w // 2]


def propagation_case(pol, prop, g, to_numpy=np.asarray, asarray=np.asarray):
    """test_make_propagation_polarized's calls (tests/x/test_polarization.py:139-176) on its J = diag(A), through
    jones_adapter: windows of the outputs and their full sums of |.|."""
    A = g['A']
    J = np.zeros([*A.shape, 2, 2])
    J[..., 0, 0] = A
    J[..., 1, 1] = A
    J = asarray(J)
    wave, samples = 1, A.shape[0]
    dx = 5 / samples
    focus, unfocus = pol.jones_adapter(prop.focus), pol.jones_adapter(prop.unfocus)
    angular_spectrum = pol.jones_adapter(prop.angular_spectrum)
    focus_dft, unfocus_dft = pol.jones_adapter(prop.focus_dft), pol.jones_adapter(prop.unfocus_dft)
    J_psf = focus(J, Q=2)
    J_pupil = unfocus(J_psf, Q=1)
    J_prop = angular_spectrum(J_pupil, wvl=wave, dx=dx, z=5e1, Q=1)
    mdft = prop.prepare_executor(pupil_dx=dx, pupil_samples=samples, focal_dx=1000e-3, focal_samples=256, wavelength=wave,
                                 efl=50)
    J_psf_fixed = focus_dft(J, mdft)
    J_pupil_fixed = unfocus_dft(J_psf_fixed, mdft)
    out = {}
    for k, v in (('psf', J_psf), ('pupil', J_pupil), ('prop', J_prop), ('psf_fixed', J_psf_fixed),
                 ('pupil_fixed', J_pupil_fixed)):
        v = to_numpy(v)
        out[f'prop_{k}'] = window(v)
        out[f'prop_{k}_abssum'] = np.abs(v).sum(axis=(0, 1))
    return out


def vvc_case(pol, prop, g, to_numpy=np.asarray, asarray=np.asarray):
    """A small vector vortex coronagraph, all four elements: Jones pupil -> focus_dft (MDFT) -> VVR (charge 2) @ ->
    unfocus_dft -> Lyot stop -> focus_dft."""
    amp, phase, lyot = g['vvc_amp'], g['vvc_phase'], g['vvc_lyot']
    _, _, r, _ = grid(VVC_N, 10)
    field = amp * np.exp(1j * phase)
    optic = pol.linear_retarder(asarray(0.2 * (r / 5) ** 2), theta=0.3, shape=r.shape)
    J = pol.apply_polarization_optic(asarray(field), optic)
    ex = prop.prepare_executor(pupil_dx=VVC['pupil_dx'], pupil_samples=VVC_N, focal_dx=VVC['focal_dx'],
                               focal_samples=VVC['focal_samples'], wavelength=VVC['wavelength'], efl=VVC['efl'])
    fx = (np.arange(VVC_N) - VVC_N // 2) * VVC['focal_dx']
    fxx, fyy = np.meshgrid(fx, fx)
    vvr = pol.vector_vortex_retarder(2, asarray(np.arctan2(fyy, fxx)))
    focus_dft, unfocus_dft = pol.jones_adapter(prop.focus_dft), pol.jones_adapter(prop.unfocus_dft)
    matmul = getattr(pol, 'jones_matmul', np.matmul)        # the reference's `vvr @ J`
    at_fpm = focus_dft(J, ex)
    at_lyot = unfocus_dft(matmul(vvr, at_fpm), ex)
    after_lyot = pol.apply_polarization_optic(asarray(lyot), at_lyot)
    final = focus_dft(after_lyot, ex)
    at_fpm, final = to_numpy(at_fpm), to_numpy(final)
    return {'vvc_at_fpm': window(at_fpm, 64), 'vvc_final': window(final, 96), 'vvc_final_abssum': np.abs(final).sum(axis=(0, 1))}


def run(pol, prop, g, to_numpy=np.asarray, asarray=np.asarray):
    out = {}
    out.update(constructors(pol, g, to_numpy))
    out.update(reductions(pol, g, to_numpy))
    out.update(propagation_case(pol, prop, g, to_numpy, asarray))
    out.update(vvc_case(pol, prop, g, to_numpy, asarray))
    return out


def reference_modules():
    from prysm.conf import config
    from prysm.x import polarization as pol
    from prysm import propagation as prop
    config.precision = 64
    return pol, prop


def reference_outputs():
    with reference.loaded():
        pol, prop = reference_modules()
        g = inputs()
        out = run(pol, prop, g)
        out['diattenuator_plane'] = diattenuator_plane(pol, g['alpha'])
        return out


def main():
    """Write tests/golden/polarization*.npz from the unmodified reference."""
    with reference.loaded():
        from make_golden import save      # imports the reference
        save('polarization.npz', reference_outputs())


if __name__ == '__main__':
    main()
