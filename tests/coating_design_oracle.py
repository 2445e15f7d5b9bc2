"""The coating-design cases the engine is checked on (prysm/x/coatings merit.py and needle.py), and the writer of
tests/golden/coating_design*.npz.

    PYTHONDONTWRITEBYTECODE=1 python tests/coating_design_oracle.py   (needs the unmodified reference: PRYSM_REFERENCE
                                                                      or oracle/_ref)

The fixtures are the REFERENCE's own outputs at precision 64, on stacks of tests/thinfilm_oracle.py (a lossless
quarter-wave stack, the absorbing metal, the evanescent gap and the dispersive callables):
  - `<stack>_<grid>_<pol>_<term>_*`: value, residuals and value_and_grad (thickness and index) of every term class,
    with negative and repeated layer / boundary indices and a PeakFieldAtInterfaces tie, on a scalar sample, a 1-D
    wavelength grid with an array target, and the meshgridded wavelength x angle grid with a target and a weight that
    broadcast;
  - `needle_<stack>_<pol>_<q>_<needle>`: needle_function of an R or T term for a constant and a dispersive needle at
    z = 0, every boundary, the total thickness and beyond both ends.
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (ROOT, HERE, os.path.join(ROOT, 'oracle')):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import reference  # noqa: E402
import thinfilm_oracle as TF  # noqa: E402

POLS = ('s', 'p', 'avg')
QW = 0.55


def stacks():
    """name -> (indices, thicknesses, substrate_index, ambient_index)."""
    s = TF.stacks()
    hl = [2.35, 1.46, 2.35, 1.46]
    return {'qw': (hl, [QW / 4 / n for n in hl], 1.52, 1.0), 'metal': s['metal'], 'gap': s['gap'], 'disp': s['disp']}


def grids():
    """name -> (wvl, theta, target, weight): a scalar sample, a 1-D wavelength grid with an array target, and the
    meshgridded grid of thinfilm_oracle with a target per wavelength and a weight per angle."""
    w1 = np.linspace(0.45, 0.7, 9)
    return {
        'scalar': (0.55, 0.2, 0.1, 2.0),
        'line': (w1, 0.1, np.linspace(0.0, 0.3, 9), 1.0),
        'mesh': (TF.GRID_WVL, TF.GRID_THETA, np.linspace(0.05, 0.4, 7)[:, None], np.linspace(0.5, 2.0, 6)[None, :]),
    }


def terms(m, wvl, theta, pol, target, weight):
    """name -> term of the namespace m, every class with the index cases of the issue."""
    kw = dict(theta=theta, pol=pol, target=target, weight=weight)
    return {
        'R': m.Reflectance(wvl, **kw),
        'T': m.Transmittance(wvl, **kw),
        'A0': m.LayerAbsorptance(0, wvl, **kw),
        'Am1': m.LayerAbsorptance(-1, wvl, **kw),
        'E1': m.FieldIntensityAtBoundary(1, wvl, **kw),
        'Em1': m.FieldIntensityAtBoundary(-1, wvl, **kw),
        'Pall': m.PeakFieldAtInterfaces(wvl, **kw),
        'Pdup': m.PeakFieldAtInterfaces(wvl, boundaries=[0, -1, 1, 1], **kw),
        'Ptie': m.PeakFieldAtInterfaces(wvl, boundaries=[1, 1], **kw),
        'L0': m.FieldInLayer(0, wvl, **kw),
        'Lm1': m.FieldInLayer(-1, wvl, **kw),
    }


def depths(st):
    Z = np.concatenate([[0.0], np.cumsum(np.asarray(st.thicknesses, dtype=np.float64))])
    return np.concatenate([[-0.02], Z, [0.5 * Z[-1], Z[-1] + 0.05]])


def run(m):
    """Every fixture from the namespace m (Stack, the term classes, needle_function, thickness_gradient,
    index_gradient); `host` turns a result into numpy."""
    out = {}
    for sname, (n, d, sub, amb) in stacks().items():
        st = m.Stack(n, d, sub, amb)
        for gname, (wvl, theta, target, weight) in grids().items():
            if gname != 'mesh' and sname != 'qw':
                continue
            for pol in POLS:
                for tname, t in terms(m, wvl, theta, pol, target, weight).items():
                    k = f'{sname}_{gname}_{pol}_{tname}'
                    out[f'{k}_value'] = t.value(st)
                    out[f'{k}_res'] = m.host(t.residuals(st))
                    for gk, fn in (('gth', m.thickness_gradient), ('gix', m.index_gradient)):
                        v, g = t.value_and_grad(st, grad_fn=fn)
                        out[f'{k}_{gk}_value'], out[f'{k}_{gk}'] = v, m.host(g)
        wvl, theta, target, weight = grids()['mesh']
        for pol in POLS:
            for q, cls in (('R', m.Reflectance), ('T', m.Transmittance)):
                t = cls(wvl, theta=theta, pol=pol, target=target, weight=weight)
                for nname, nm in (('c', 1.38), ('d', TF.cauchy)):
                    out[f'needle_{sname}_{pol}_{q}_{nname}'] = m.host(m.needle_function(st, t, nm, depths(st)))
    return {k: np.asarray(v) for k, v in out.items()}


def reference_namespace():
    from prysm.conf import config
    from prysm.x import coatings
    from prysm.x.coatings import merit, needle, diff
    config.precision = 64
    ns = {n: getattr(merit, n) for n in merit.__all__}
    return types.SimpleNamespace(Stack=coatings.Stack, needle_function=needle.needle_function,
                                 thickness_gradient=diff.thickness_gradient, index_gradient=diff.index_gradient,
                                 host=np.asarray, **ns)


def reference_outputs():
    import warnings
    with reference.loaded(), warnings.catch_warnings():
        m = reference_namespace()
        warnings.simplefilter('ignore')
        return run(m)


def main():
    """Write tests/golden/coating_design*.npz from the unmodified reference."""
    with reference.loaded():
        from make_golden import save      # imports the reference
        save('coating_design.npz', reference_outputs())


if __name__ == '__main__':
    main()
