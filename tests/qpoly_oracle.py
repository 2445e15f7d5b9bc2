"""The Forbes-polynomial cases the engine is checked on (prysm/polynomials/qpoly.py), and the writer of
tests/golden/qpoly*.npz.

    PYTHONDONTWRITEBYTECODE=1 python tests/qpoly_oracle.py   (needs the unmodified reference: PRYSM_REFERENCE or
                                                              oracle/_ref)

The fixtures are the REFERENCE's own outputs at precision 64:
  - `tab_*`: the scalar recurrence tables for n <= 64 (the engine's order limit) and 1 <= m <= 20 (NaN where the
    reference divides by zero), so the engine's C++ restatement of them is pinned independently of any kernel;
  - on two grids (`odd`: 33 x 33 over [-1, 1]; `even`: 32 x 40 on fftrange / 16, both holding r = 0 and r = 1):
    the inputs `<g>_x, <g>_y, <g>_r, <g>_t` and every *_seq / *_der_seq / *_der_xy_seq and compute_z* output;
  - `psf`: a freeform pupil taken to focus by the reference's host pipeline.
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (ROOT, os.path.join(ROOT, 'oracle')):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import reference  # noqa: E402

NMAX = 64                   # the engine's order limit (PB_QPOLY_NMAX)
TAB_M = 20
NS = [0, 1, 2, 3, 5, 8, 12]  # ascending: the reference's 1-D sequences assume it
# m = 0, m = 1 beyond n = 3, large |m|, sine and cosine terms, a repeated pair, unsorted
NMS = [(3, 0), (0, 0), (1, 0), (0, 1), (5, 1), (4, 1), (2, -1), (6, -1), (3, -1), (2, 2), (0, -2), (7, 3), (3, -3),
       (2, 12), (4, -12), (2, 2), (1, 20), (0, 0)]
# compute_z cases: (cm0, ams, bms)
Q2D_SUMS = {
    'mixed': ([0.3, -0.1, 0.05, 0.0, 0.02], [[0.1, 0.2, -0.05, 0.04, 0.01], [0.0, 0.1]],
              [[-0.2, 0.03, 0.01, 0.0, 0.0], [0.05, -0.02, 0.01]]),
    'sine_only': ([], [[], [], []], [[], [], [0.1, -0.04, 0.02]]),     # an order with only sine terms
    'm1_short': ([0.0, 0.0], [[0.2, -0.1, 0.05]], [[0.1]]),          # m = 1 with N <= 2 (no alphas[3] term)
    'zeros': ([0.0, 0.0], [[0.0], [0.0, 0.0]], [[0.0, 0.0], [0.0]]),
}
RADIAL_SUMS = {'dense': [0.4, -0.2, 0.1, 0.05, -0.02, 0.01], 'trailing': [0.0, 0.3, 0.0, -0.1, 0.0, 0.0],
               'zeros': [0.0, 0.0, 0.0]}
# the end-to-end freeform pupil: nms, coefs in waves-scale microns, samples, diameter (mm), wavelength, efl, Q
PSF_NMS = [(0, 0), (1, 0), (2, 0), (0, 1), (1, 1), (3, 1), (0, -1), (2, 2), (1, -2), (0, 3), (1, -3), (0, 4)]
PSF_COEFS = [0.05, -0.03, 0.02, 0.08, -0.04, 0.03, 0.06, 0.05, -0.04, 0.03, 0.02, -0.02]
PSF_N, PSF_D, PSF_WVL, PSF_EFL, PSF_Q = 128, 10.0, 0.6328, 100.0, 2


def grids():
    """name -> (x, y, r, t) in fp64."""
    out = {}
    v = np.linspace(-1.0, 1.0, 33)
    out['odd'] = np.meshgrid(v, v)
    xv = np.arange(-20, 20, dtype=np.float64) / 16
    yv = np.arange(-16, 16, dtype=np.float64) / 16
    out['even'] = np.meshgrid(xv, yv)
    return {k: (x, y, np.hypot(x, y), np.arctan2(y, x)) for k, (x, y) in out.items()}


def psf_inputs():
    """Pupil amplitude (circle, diameter PSF_D) and the normalised polar grid of the end-to-end case, fp64."""
    n = PSF_N
    dx = PSF_D / n
    v = (np.arange(n, dtype=np.float64) - n // 2) * dx
    x, y = np.meshgrid(v, v)
    r = np.hypot(x, y)
    u, t = r / (PSF_D / 2), np.arctan2(y, x)
    amp = (u <= 1).astype(np.float64)
    return amp, u, t, dx


def reference_modules():
    from prysm.conf import config
    from prysm.polynomials import qpoly
    from prysm.propagation import Wavefront
    config.precision = 64
    return types.SimpleNamespace(q=qpoly, Wavefront=Wavefront)


def _abc(q, n, m):
    try:
        return q.abc_q2d(n, m)
    except ZeroDivisionError:
        return (np.nan, np.nan, np.nan)


def tables(q):
    out = {'tab_qbfs': np.array([[q.f_qbfs(n), q.g_qbfs(n), q.h_qbfs(n)] for n in range(NMAX + 1)]),
           'tab_qcon': np.array([q._qcon_abc(n) for n in range(NMAX + 1)])}
    out['tab_q2d'] = np.array([[[*_abc(q, n, m), q.G_q2d(n, m), q.F_q2d(n, m), q.g_q2d(n, m), q.f_q2d(n, m)]
                                for n in range(NMAX + 1)] for m in range(1, TAB_M + 1)])
    return out


def run(m):
    q = m.q
    out = tables(q)
    for g, (x, y, r, t) in grids().items():
        out.update({f'{g}_x': x, f'{g}_y': y, f'{g}_r': r, f'{g}_t': t})
        out[f'{g}_qbfs'] = q.Qbfs_seq(NS, r)
        out[f'{g}_qbfs_der'] = q.Qbfs_der_seq(NS, r)
        out[f'{g}_qcon'] = q.Qcon_seq(NS, r)
        out[f'{g}_qcon_der'] = q.Qcon_der_seq(NS, r)
        out[f'{g}_q2d'] = q.Q2d_seq(NMS, r, t)
        out[f'{g}_q2d_dr'], out[f'{g}_q2d_dt'] = q.Q2d_der_seq(NMS, r, t)
        out[f'{g}_q2d_dx'], out[f'{g}_q2d_dy'] = q.Q2d_der_xy_seq(NMS, x, y)
        for name, c in RADIAL_SUMS.items():
            out[f'{g}_zbfs_{name}'] = q.compute_z_Qbfs(c, r, r * r)
            out[f'{g}_zbfs_{name}_z'], out[f'{g}_zbfs_{name}_dr'] = q.compute_z_zprime_Qbfs(c, r, r * r)
            out[f'{g}_zcon_{name}_z'], out[f'{g}_zcon_{name}_dr'] = q.compute_z_zprime_Qcon(c, r, r * r)
        for name, (cm0, ams, bms) in Q2D_SUMS.items():
            out[f'{g}_z2d_{name}'] = q.compute_z_Q2d(cm0, ams, bms, r, t)
            z, dr, dt = q.compute_z_zprime_Q2d(cm0, ams, bms, r, t)
            out[f'{g}_z2d_{name}_z'], out[f'{g}_z2d_{name}_dr'], out[f'{g}_z2d_{name}_dt'] = z, dr, dt
    amp, u, t, dx = psf_inputs()
    cm0, ams, bms = q.Q2d_nm_c_to_a_b(PSF_NMS, PSF_COEFS)
    opd = q.compute_z_Q2d(cm0, ams, bms, u, t)
    wf = m.Wavefront.from_amp_and_phase(amp, opd * 1e3, PSF_WVL, dx)      # microns -> nm
    out['psf_opd'] = opd
    out['psf'] = np.asarray(wf.focus(PSF_EFL, Q=PSF_Q).intensity.data)
    return {k: np.asarray(v, dtype=np.float64) for k, v in out.items()}


def reference_outputs():
    import warnings
    with reference.loaded(), warnings.catch_warnings():
        m = reference_modules()
        warnings.simplefilter('ignore')
        return run(m)


def main():
    """Write tests/golden/qpoly*.npz from the unmodified reference."""
    with reference.loaded():
        from make_golden import save      # imports the reference
        save('qpoly.npz', reference_outputs())


if __name__ == '__main__':
    main()
