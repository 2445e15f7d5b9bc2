"""The thin-film cases the engine is checked on (prysm/thinfilm.py multilayer_stack_rt, prysm/x/coatings stack.py and
diff.py), and the writer of tests/golden/thinfilm*.npz.

    PYTHONDONTWRITEBYTECODE=1 python tests/thinfilm_oracle.py   (needs the unmodified reference: PRYSM_REFERENCE or
                                                                 oracle/_ref)

The fixtures are the REFERENCE's own outputs at precision 64:
  - `ml_*`: multilayer_stack_rt for the reference's MONO and MULTI stacks at AOI 0, 15, 45 and 70 degrees, a total
    internal reflection case, per-pixel layers (3 x 4, and 64 x 80 with a per-pixel substrate) and 1-D layers with an
    AOI map;
  - `<stack>_<pol>_*`: stack_rt, internal_fields and RTA of every stack of `stacks()` on a wavelength x angle grid that
    runs past the critical angle, and thickness_gradient / index_gradient for each seed kind (dR, dT, dA, dEsq) and a
    mixed seed;
  - `fad_<stack>_<pol>_*`: field_at_depth at the boundary depths and on 12001 depths, and at one depth over the
    wavelength x angle grid.
A thick evanescent gap under total internal reflection (`gap`, `ml_gap`) reaches |Im beta| of about 77.
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

WVL = 0.587725
N_C7980, N_MGF2, N_CEF3, N_ZRO2 = 1.458461, 1.3698, 1.6290 + 1j * 0.0034836, 2.1588
MONO = ([N_MGF2], [0.150])
MULTI = ([N_MGF2, N_ZRO2, N_CEF3], [WVL / 4, WVL / 2, WVL / 4])
ML_AOI = [0, 15, 45, 70]
POLS = ('s', 'p')
GRID_WVL = np.linspace(0.45, 0.75, 7)[:, None]
GRID_THETA = np.radians([0.0, 15.0, 45.0, 70.0, 80.0, 89.0])[None, :]
FAD_WVL, FAD_THETA = 0.55, 0.3
FAD_STACKS = ('multi', 'metal', 'lossy', 'tir', 'gap')


class NK:
    """A material with an `.nk(wvl)` method, as the reference's materials protocol has."""

    def nk(self, wvl):
        return 1.62 + 0.01 / np.asarray(wvl) ** 2 + 1e-4j


def cauchy(wvl):
    return 1.45 + 0.004 / np.asarray(wvl) ** 2


def stacks():
    """name -> (indices, thicknesses, substrate_index, ambient_index)."""
    rng = np.random.default_rng(20261017)
    l40 = [1.45 if i % 2 else 2.3 for i in range(40)]
    l40[5] = 1.5 + 0.3j
    return {
        'mono': (MONO[0], MONO[1], N_C7980, 1.0),
        'multi': (MULTI[0], MULTI[1], N_C7980, 1.0),
        'lossy': ([1.38, 2.05, 1.5 + 0.3j, 2.05], [0.12, 0.08, 0.05, 0.10], 1.52, 1.0),
        'metal': ([1.38, 0.05 + 3.9j], [0.09, 0.1], 1.52, 1.0),
        # glass ambient onto air: total internal reflection beyond 36 degrees
        'tir': ([1.38, 2.05], [0.1, 0.08], 1.0, 1.7),
        'l40': (l40, rng.uniform(0.05, 0.15, 40), 1.52, 1.0),
        'disp': ([cauchy, NK(), 2.05], [0.1, 0.07, 0.09], 1.52, 1.0),
        'zero': ([], np.zeros(0), 1.52, 1.0),
        # frustrated TIR: a 4 um air gap between 1.7 glass, evanescent beyond 36 degrees (|Im beta| up to about 77)
        'gap': ([1.38, 1.0], [0.1, 4.0], 1.7, 1.7),
    }


def seeds(name, shape, N):
    """The cotangents of a gradient case: fixed pseudo-random values of the right shapes."""
    rng = np.random.default_rng(sum(map(ord, name)))
    dR, dT = rng.standard_normal(shape), rng.standard_normal(shape)
    dA, dEsq = rng.standard_normal((N,) + shape), rng.standard_normal((N + 1,) + shape)
    return {'dR': dict(dR=dR), 'dT': dict(dT=dT), 'dA': dict(dA=dA), 'dEsq': dict(dEsq=dEsq),
            'mixed': dict(dR=dR, dT=dT, dA=dA, dEsq=dEsq)}


def ml_cases():
    """name -> (indices, thicknesses, wavelength, polarization, substrate_index, aoi, ambient_index)."""
    rng = np.random.default_rng(7)
    out = {}
    for lname, (n, d) in (('mono', MONO), ('multi', MULTI)):
        for aoi in ML_AOI:
            for pol in POLS:
                out[f'ml_{lname}_{aoi}_{pol}'] = (n, d, WVL, pol, N_C7980, aoi, 1)
    for pol in POLS:
        out[f'ml_tir_{pol}'] = ([1.38, 2.05], [0.1, 0.08], 0.55, pol, 1.0, np.array([20.0, 50.0, 70.0]), 1.7)
        idx = np.array([1.38, 2.05])[:, None, None] * (1 + 0.01 * rng.standard_normal((2, 3, 4)))
        th = np.array([0.1, 0.07])[:, None, None] * (1 + 0.02 * rng.standard_normal((2, 3, 4)))
        out[f'ml_pix34_{pol}'] = (idx, th, 0.55, pol, 1.52, 10.0, 1)
        idx = (np.array([1.38, 2.05, 1.38, 2.05 + 0.01j])[:, None, None] * np.ones((1, 64, 80)))
        th = np.array([0.1, 0.07, 0.1, 0.07])[:, None, None] * (1 + 0.02 * rng.standard_normal((1, 64, 80)))
        sub = 1.52 + 0.01 * rng.standard_normal((64, 80))
        out[f'ml_pix6480_{pol}'] = (idx, th, 0.6328, pol, sub, 12.0, 1)
        out[f'ml_gap_{pol}'] = ([1.38], [5.0], 0.55, pol, 1.7, np.array([60.0, 70.0, 80.0]), 1.7)
        out[f'ml_aoimap_{pol}'] = ([1.38, 2.05], [0.1, 0.07], 0.55, pol, 1.52, np.linspace(0, 40, 12).reshape(3, 4), 1)
    return out


def reference_modules():
    from prysm.conf import config
    from prysm import thinfilm
    from prysm.x import coatings
    from prysm.x.coatings import diff
    config.precision = 64
    return types.SimpleNamespace(thinfilm=thinfilm, coatings=coatings, diff=diff)


def run(m):
    """Every fixture from the namespace m (thinfilm, coatings: Stack, stack_rt, internal_fields, RTA, field_at_depth;
    diff: forward_eval, thickness_gradient, index_gradient)."""
    out = {}
    for name, args in ml_cases().items():
        out[f'{name}_r'], out[f'{name}_t'] = m.thinfilm.multilayer_stack_rt(*args)
    c, diff = m.coatings, m.diff
    for sname, (n, d, sub, amb) in stacks().items():
        st = c.Stack(n, d, sub, amb)
        for pol in POLS:
            k = f'{sname}_{pol}'
            out[f'{k}_r'], out[f'{k}_t'] = c.stack_rt(st, GRID_WVL, GRID_THETA, pol)
            out[f'{k}_E'], out[f'{k}_H'] = c.internal_fields(st, GRID_WVL, GRID_THETA, pol)
            out[f'{k}_R'], out[f'{k}_T'], out[f'{k}_A'] = c.RTA(st, GRID_WVL, GRID_THETA, pol)
            f = diff.forward_eval(st, GRID_WVL, GRID_THETA, pol)
            for seed, kw in seeds(k, np.shape(f.r), len(st)).items():
                out[f'{k}_gth_{seed}'] = diff.thickness_gradient(f, **kw)
                out[f'{k}_gix_{seed}'] = diff.index_gradient(f, **kw)
            if len(st) and sname in FAD_STACKS:
                Z = np.concatenate([[0.0], np.cumsum(st.thicknesses)])
                for zname, z in (('bound', Z), ('dense', np.linspace(0.0, Z[-1], 12001))):
                    E, H = c.field_at_depth(st, z, FAD_WVL, FAD_THETA, pol)
                    out[f'fad_{k}_{zname}_E'], out[f'fad_{k}_{zname}_H'] = E, H
                # one depth over the whole wavelength x angle grid
                E, H = c.field_at_depth(st, 0.7 * Z[-1], GRID_WVL, GRID_THETA, pol)
                out[f'fad_{k}_grid_E'], out[f'fad_{k}_grid_H'] = E, H
    return {k: np.asarray(v) for k, v in out.items()}


def reference_outputs():
    import warnings
    with reference.loaded(), warnings.catch_warnings():
        m = reference_modules()
        warnings.simplefilter('ignore')
        return run(m)


def main():
    """Write tests/golden/thinfilm*.npz from the unmodified reference."""
    with reference.loaded():
        from make_golden import save      # imports the reference
        save('thinfilm.npz', reference_outputs())


if __name__ == '__main__':
    main()
