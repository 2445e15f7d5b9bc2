"""The optical-monitoring cases the engine is checked on (prysm/x/coatings monitoring.py), and the writer of
tests/golden/monitoring*.npz.

    PYTHONDONTWRITEBYTECODE=1 python tests/monitoring_oracle.py   (needs the unmodified reference: PRYSM_REFERENCE or
                                                                   oracle/_ref)

The fixtures are the REFERENCE's own outputs at precision 64:
  - `trace_*`: monitoring_trace (grid and signal) of the first, a middle and the last layer and of layer -1 (every
    layer below the growing one, as Python slices `indices[layer + 1:]`), and turning_points / level_cut of each trace;
  - `levels_*`: cutoff_levels;
  - `run_*`: simulate_run's as-built thicknesses for both strategies, turning index 1 and 2, fewer turning points than
    asked, signal and thickness errors, levels passed in, 1, 2, 57 and 1200 grid points and max_factor;
  - `cut_*` / `tp_*`: level_cut and turning_points on analytic arrays: no crossing, an exact zero at a sample, a tie to
    the target, a plateau;
  - `sens_*`: monitoring_error_sensitivity for both strategies and a p-polarized readout;
  - `choose_*`: choose_monitor_wavelength on five candidates from 0.45 to 0.65 µm for a design at 0.55 µm.
Stacks: jittered quarter-wave HL stacks of 10 and 20 layers, a four-layer design, the absorbing metal and the
dispersive callables of tests/thinfilm_oracle.py; the monitor on and off the design wavelength, s and p, R and T, at
0 and 0.3 rad.  The writer refuses a case the reference computes ill-conditioned: every stack case is run again with
its thicknesses scaled by 1 + 1e-13 and must move by less than 1e-10 of its largest magnitude.
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

W = 0.55
SUB = 1.52
PROBE = 1e-13
PROBE_BOUND = 1e-10
CANDIDATES = [0.45, 0.50, 0.55, 0.60, 0.65]


def hl(n, seed):
    """n alternating 2.35 / 1.46 quarter waves at W with thicknesses jittered by up to 5 %"""
    idx = [2.35 if k % 2 == 0 else 1.46 for k in range(n)]
    rng = np.random.default_rng(seed)
    th = np.array([W / 4 / i for i in idx]) * (1 + 0.05 * rng.uniform(-1, 1, n))
    return idx, th, SUB, 1.0


def stacks():
    """name -> (indices, thicknesses, substrate_index, ambient_index)."""
    s = TF.stacks()
    four = [1.46, 2.05, 1.46, 2.05]
    return {'hl10': hl(10, 3), 'hl20': hl(20, 4), 'four': (four, np.array([0.09, 0.067, 0.10, 0.067]), SUB, 1.0),
            'qw4': (four, np.array([W / (4 * n) for n in four]), SUB, 1.0), 'metal': s['metal'], 'disp': s['disp']}


# (stack, layer, monitor wvl, kwargs of monitoring_trace)
TRACES = [
    ('hl10', 0, 0.6, dict()),
    ('hl10', 4, 0.55, dict(pol='p', theta=0.3, n_points=57)),
    ('hl10', -1, 0.6, dict(mode='T', max_factor=2.5)),
    ('hl20', 19, 0.6, dict(n_points=1200, max_factor=1.8)),
    ('qw4', 1, 0.55, dict(n_points=2000, max_factor=1.7)),
    ('metal', 0, 0.6, dict(mode='T', pol='P', theta=0.3)),
    ('disp', 1, 0.6, dict(pol='p', n_points=300, max_factor=1.8)),
    ('disp', -2, 0.5, dict(mode='T')),
]

# (stack, monitor wvl, kwargs of cutoff_levels)
LEVELS = [('hl10', 0.6, dict()), ('hl20', 0.6, dict(pol='p', theta=0.3)), ('metal', 0.6, dict(mode='T')),
          ('disp', 0.6, dict(mode='T', pol='p')), ('four', 0.55, dict())]

# (name, stack, monitor wvl, kwargs of simulate_run); the errors are drawn per case from a seeded generator
RUNS = [
    ('level', 'hl10', 0.6, dict()),
    ('level_on_design', 'four', 0.5, dict(n_points=1200)),
    ('level_p_theta', 'hl10', 0.6, dict(pol='p', theta=0.3, n_points=57)),
    ('level_T', 'hl20', 0.6, dict(mode='T', max_factor=1.5)),
    ('level_sigerr', 'hl20', 0.6, dict(signal_errors='sig')),
    ('level_levels', 'hl10', 0.6, dict(levels='given', signal_errors='sig')),
    ('level_n1', 'hl10', 0.6, dict(n_points=1)),
    ('level_n2', 'hl10', 0.6, dict(n_points=2)),
    ('level_metal', 'metal', 0.6, dict(mode='T')),
    ('level_disp', 'disp', 0.6, dict(pol='p')),
    ('level_ignores_th_err', 'hl10', 0.6, dict(thickness_errors='th')),
    ('turning', 'qw4', 0.55, dict(strategy='turning', n_points=2000)),
    ('turning_thicker', 'qw4', 0.55, dict(strategy='turning', n_points=2000, thickness_errors='th')),
    ('turning_2', 'hl10', 0.6, dict(strategy='turning', turning_index=2, max_factor=2.5)),
    ('turning_fewer', 'hl10', 0.6, dict(strategy='turning', turning_index=5)),
    ('turning_T_p', 'hl20', 0.6, dict(strategy='turning', mode='T', pol='p', theta=0.3, n_points=1200)),
    ('turning_ignores_sig_err', 'qw4', 0.55, dict(strategy='turning', signal_errors='sig', n_points=57)),
    ('turning_n2', 'qw4', 0.55, dict(strategy='turning', n_points=2)),
]

# (name, stack, monitor wvl, kwargs of monitoring_error_sensitivity)
DESIGN_WVLS = np.linspace(0.45, 0.65, 41)
SENS = [
    ('level', 'hl10', 0.6, dict()),
    ('turning', 'qw4', 0.55, dict(strategy='turning', n_points=2000)),
    ('level_design_p', 'four', 0.6, dict(design_pol='p', theta=0.3, n_points=800)),
    # dispersive and absorbing layers, ambient and substrate: the readout resolves them at each design wavelength
    ('level_disp', 'disp', 0.6, dict(design_pol='P', pol='p')),
    ('turning_disp', 'disp', 0.5, dict(strategy='turning', mode='T', theta=0.3, max_factor=2.5)),
    ('level_metal', 'metal', 0.6, dict(mode='T')),
]


def analytic():
    """name -> (d, signal, level, target) for level_cut (level not None) or turning_points (level None)."""
    d = np.linspace(0.0, 1.0, 101)
    return {
        'cut_line': (d, 0.2 + 0.5 * d, 0.45, None),
        'cut_none': (d, 0.2 + 0.5 * d, 2.0, None),                  # no crossing: the sample nearest the level
        'cut_none_tie': (d, np.abs(d - 0.5), -1.0, None),           # no crossing, two nearest samples: the first
        'cut_zero': (d, d - 0.3, 0.0, 0.9),                         # s = 0 exactly at a sample
        'cut_sine_target': (np.linspace(0, 1, 201), np.sin(2 * np.pi * np.linspace(0, 1, 201)), 0.0, 0.48),
        'cut_tie': (np.linspace(0, 1, 5), np.array([1.0, -1.0, 1.0, -1.0, 1.0]), 0.0, 0.5),   # 0.375 and 0.625
        'cut_plateau': (d, np.minimum(d, 0.4), 0.4, 0.8),           # a plateau at the level
        'cut_one': (np.array([0.25]), np.array([0.7]), 0.5, None),
        'tp_sine': (np.linspace(0, 2, 401), np.cos(3 * np.pi * np.linspace(0, 2, 401)), None, None),
        'tp_plateau': (d, np.minimum(np.maximum(d, 0.3), 0.6), None, None),
        'tp_flat_start': (d, np.where(d < 0.2, 0.0, np.sin(8 * d)), None, None),
        'tp_monotone': (d, d ** 2, None, None),
        'tp_short': (np.array([0.0, 1.0]), np.array([0.0, 1.0]), None, None),
    }


def errors(name, N):
    rng = np.random.default_rng(sum(map(ord, name)))
    return {'sig': 2e-3 * rng.standard_normal(N), 'th': 4e-3 * rng.standard_normal(N)}


def run(m, scale=1.0):
    """Every stack fixture from the namespace m (Stack, the seven monitoring functions, RTA, host) with the stacks'
    thicknesses scaled by `scale`; the analytic cases when scale is 1."""
    st = {k: m.Stack(n, np.asarray(d) * scale, sub, amb) for k, (n, d, sub, amb) in stacks().items()}
    out = {}
    for j, (s, layer, wm, kw) in enumerate(TRACES):
        d, sig = m.monitoring_trace(st[s], layer, wm, **kw)
        d, sig = m.host(d), m.host(sig)
        k = f'trace{j}_{s}'
        out[f'{k}_d'], out[f'{k}_sig'] = d, sig
        out[f'{k}_tp'] = m.host(m.turning_points(d if m.device is None else m.device(d),
                                                 sig if m.device is None else m.device(sig)))
        mid = 0.5 * (float(np.min(sig)) + float(np.max(sig)))
        out[f'{k}_cut'] = m.level_cut(d if m.device is None else m.device(d),
                                      sig if m.device is None else m.device(sig), mid, target=0.5 * float(d[-1]))
    for j, (s, wm, kw) in enumerate(LEVELS):
        out[f'levels{j}_{s}'] = m.host(m.cutoff_levels(st[s], wm, **kw))
    for name, s, wm, kw in RUNS:
        kw = dict(kw)
        e = errors(name, len(st[s]))
        for key, src in (('signal_errors', 'sig'), ('thickness_errors', 'th')):
            if key in kw:
                kw[key] = e[src]
        if kw.get('levels') == 'given':
            kw['levels'] = m.host(m.cutoff_levels(st[s], wm)) + 1e-3
        out[f'run_{name}'] = np.asarray(m.run(st[s], wm, **kw).thicknesses, dtype=np.float64)
    for name, s, wm, kw in SENS:
        out[f'sens_{name}'] = m.host(m.monitoring_error_sensitivity(st[s], wm, DESIGN_WVLS, **kw))
    best, scores = m.choose_monitor_wavelength(st['four'], CANDIDATES, np.array([W]), strategy='level',
                                               design_pol='s')
    out['choose_best'], out['choose_scores'] = best, m.host(scores)
    if scale == 1.0:
        for name, (d, sig, level, target) in analytic().items():
            dd, ss = (d, sig) if m.device is None else (m.device(d), m.device(sig))
            out[name] = m.host(m.turning_points(dd, ss)) if level is None else m.level_cut(dd, ss, level, target)
    return {k: np.asarray(v) for k, v in out.items()}


def reference_namespace():
    from prysm.conf import config
    from prysm.x.coatings import Stack, RTA, monitoring as mon
    config.precision = 64
    return types.SimpleNamespace(Stack=Stack, RTA=RTA, host=np.asarray, device=None, run=mon.simulate_run,
                                 **{n: getattr(mon, n) for n in mon.__all__})


def reference_outputs(scale=1.0):
    import warnings
    with reference.loaded(), warnings.catch_warnings():
        m = reference_namespace()
        warnings.simplefilter('ignore')
        return run(m, scale)


def conditioning(base, probed):
    """key -> relative move of each stack fixture under the thickness probe"""
    moves = {}
    for k, v in probed.items():
        a, b = np.asarray(base[k], dtype=np.float64), np.asarray(v, dtype=np.float64)
        if a.shape != b.shape:
            moves[k] = np.inf
            continue
        den = float(np.abs(a).max()) if a.size else 0.0
        moves[k] = float(np.abs(a - b).max()) / den if den > 0 else float(np.abs(a - b).max()) if a.size else 0.0
    return moves


def main():
    """Write tests/golden/monitoring*.npz from the unmodified reference, after the conditioning probe."""
    base = reference_outputs()
    bad = {k: v for k, v in conditioning(base, reference_outputs(1 + PROBE)).items() if not v < PROBE_BOUND}
    if bad:
        raise SystemExit(f'ill-conditioned cases: {bad}')
    with reference.loaded():
        from make_golden import save      # imports the reference
        save('monitoring.npz', base)


if __name__ == '__main__':
    main()
