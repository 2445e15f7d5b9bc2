"""The interferometric-metrology cases the engine is checked on (prysm/interferogram.py, prysm/util.py statistics and
prysm/polynomials lstsq), and the writer of tests/golden/interferogram*.npz.

    PYTHONDONTWRITEBYTECODE=1 python tests/interferogram_oracle.py   (needs the unmodified reference: PRYSM_REFERENCE
                                                                      or oracle/_ref)

Every fixture is the REFERENCE's own result at precision 64, with its inputs stored beside it (`<map>_data`), so a
float32 run starts from the same data rounded once.  Maps (MAPS): `circ` 255 x 255 with a circular NaN mask, tilt
and power; `spiky` 256 x 256 with scattered NaN and spikes; `rect` 200 x 320 all finite.  Keys are `<map>_<what>`:
every statistic, TIS and bandlimited_rms form of every map; the full-size outputs (removals, fits, slopes, crop,
PSDs, filters) on the maps REMOVES, PSD_WINDOWS and `run` name, so that the fixtures stay small.  `small_*`: the
coordinate methods (crop with recenter, latcal, strip_latcal), mask, pad, designfilt2d, ideal_lpf_iir2d and the named
windows on the 37 x 52 map of small_map; `circ_blr_free_*`: bandlimited_rms as a free function in 2-D and 1-D.
"""
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (ROOT, os.path.join(ROOT, 'oracle'), HERE):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import reference  # noqa: E402

DX = 0.1
MAPS = ('circ', 'spiky', 'rect')
STATS = ('mean', 'pv', 'rms', 'Sa', 'std')
WINDOWS = ('none', 'welch', 'hann', 'array')
PSD_WINDOWS = {'circ': WINDOWS, 'spiky': ('none',), 'rect': ('none', 'hann')}
REMOVES = {'circ': ('remove_piston', 'remove_tiptilt', 'remove_power'), 'spiky': ('remove_piston', 'remove_tiptilt'),
           'rect': ('remove_power',)}
FILTERS = {'lp': 1.5, 'hp': 1.5, 'bp': (0.8, 2.5), 'br': (0.8, 2.5)}
BLR_FORMS = {'flow': dict(flow=0.5), 'fhigh': dict(fhigh=2.0), 'band': dict(flow=0.5, fhigh=2.0),
             'wllow': dict(wllow=0.5), 'wlhigh': dict(wlhigh=2.0), 'wl': dict(wllow=0.5, wlhigh=2.0)}
TIS_ANGLES = np.array([0.0, 10.0, 30.0, 60.0])
TIS_WVL = 10.6
PVR_RADIUS = 9.0
BAND = dict(flow=0.7, fhigh=1.9)    # no sample of the circ PSD grid lies within 3e-4 (relative) of either edge


def maps():
    """name -> data of the three maps"""
    rng = np.random.default_rng(77)
    out = {}
    n = 255
    y, x = (np.mgrid[:n, :n] - n // 2) / (n // 2)
    d = 30 * x - 12 * y + 50 * (x * x + y * y) + rng.standard_normal((n, n))
    d[np.hypot(x, y) > 0.9] = np.nan
    out['circ'] = d
    n = 256
    y, x = (np.mgrid[:n, :n] - n // 2) / (n // 2)
    d = 5 * x + 8 * (x * x + y * y) + 0.5 * rng.standard_normal((n, n))
    d[rng.random((n, n)) < 0.01] = np.nan
    d[rng.random((n, n)) < 0.002] = 40.0
    out['spiky'] = d
    y, x = np.mgrid[:200, :320]
    out['rect'] = np.sin(x / 7.0) + np.cos(y / 11.0) + 0.1 * rng.standard_normal((200, 320))
    return out


def small_map():
    """37 x 52 with tilt, NaN outside an ellipse (so that crop trims it) and the mask the `mask` case applies"""
    rng = np.random.default_rng(12)
    y, x = (np.mgrid[:37, :52] - np.array([18, 26])[:, None, None]) / np.array([18, 26])[:, None, None]
    d = 3 * x + 2 * y + 0.2 * rng.standard_normal((37, 52))
    d[(x / 0.8) ** 2 + (y / 0.7) ** 2 > 1] = np.nan
    return d, x > -0.5


def user_window(shape):
    ny, nx = shape
    return np.outer(np.linspace(0.2, 1, ny), np.linspace(1, 0.3, nx))


def lstsq_inputs():
    """(modes (6, 64, 64) whose last mode duplicates the second, data with NaN)"""
    rng = np.random.default_rng(5)
    modes = rng.standard_normal((6, 64, 64))
    modes[5] = modes[1]
    data = rng.standard_normal((64, 64))
    data[rng.random((64, 64)) < 0.1] = np.nan
    return modes, data


def _copy(a):
    return a.clone() if hasattr(a, 'clone') else a.copy()


def _host(v):
    return v.detach().cpu().numpy() if hasattr(v, 'detach') else np.asarray(v)


def run(ifg, util, lstsq, prep=lambda a: a):
    """Every case, on the modules given (the reference's, or the engine's with `prep` putting each input map on the
    device at its precision); host arrays out."""
    out = {}
    m, d = lstsq_inputs()
    out['lstsq_modes'], out['lstsq_data'], out['lstsq_coefs'] = m, d, lstsq(prep(m), prep(d))
    I = ifg.Interferogram
    for name, d in maps().items():
        out[f'{name}_data'] = d
        d = prep(d)
        for s in STATS:
            out[f'{name}_{s}'] = getattr(util, s)(d)
        i = I(_copy(d), dx=DX)
        out[f'{name}_dropout'] = i.dropout_percentage
        out[f'{name}_strehl'] = i.strehl
        for meth in REMOVES[name]:
            out[f'{name}_{meth}'] = getattr(I(_copy(d), dx=DX), meth)().data
        if name != 'spiky':
            out[f'{name}_fit_plane'] = ifg.fit_plane(i.x, i.y, d)
            out[f'{name}_fit_sphere'] = ifg.fit_sphere(d)[1]
            out[f'{name}_slope_x'], out[f'{name}_slope_y'], out[f'{name}_slope_r'] = \
                (a.data for a in I(_copy(d), dx=DX).slope())
        if name != 'rect':
            out[f'{name}_crop'] = I(_copy(d), dx=DX).crop().data
        out[f'{name}_pvr_radius'] = I(_copy(d), dx=DX).pvr(PVR_RADIUS)
        if d.shape[0] == d.shape[1]:
            out[f'{name}_pvr'] = I(_copy(d), dx=DX).pvr()
        if name == 'spiky':
            out[f'{name}_clip'] = I(_copy(d), dx=DX).spike_clip(3).data
            out[f'{name}_psd_nan'] = ifg.psd(d, DX)[2]
        f = I(_copy(d), dx=DX).fill(0).data
        for w in PSD_WINDOWS[name]:
            win = {'none': None, 'array': prep(user_window(d.shape))}.get(w, w)
            out[f'{name}_psd_{w}'] = ifg.psd(f, DX, win)[2]
        i = I(_copy(f), dx=DX)
        for k, kw in BLR_FORMS.items():
            out[f'{name}_blr_{k}'] = i.bandlimited_rms(**kw)
        out[f'{name}_tis'] = i.total_integrated_scatter(TIS_WVL, TIS_ANGLES)
    f = I(prep(maps()['rect']), dx=DX).fill(0).data
    for typ, fc in FILTERS.items():
        out[f'rect_filter_{typ}'] = I(_copy(f), dx=DX).filter(fc, typ).data
    f = I(prep(maps()['circ']), dx=DX).fill(0).data
    out['circ_filter_lp'] = I(_copy(f), dx=DX).filter(FILTERS['lp'], 'lp').data
    # the automatic window of a circular map with zero corners, and the Welch window itself
    i = I(prep(maps()['circ']), dx=DX).fill(0)
    out['circ_window_auto'] = ifg.make_window(i.data, DX)
    out['circ_window_2d_welch'] = ifg.window_2d_welch(i.r, 8)
    out['rect_hann2d'] = ifg.hann2d(200, 320)
    # bandlimited_rms as a free function, on the PSD's own r: 2-D, and 1-D along the centre row
    p = I(prep(maps()['circ']), dx=DX).fill(0).psd()
    c = p.data.shape[0] // 2
    out['circ_blr_free_2d'] = ifg.bandlimited_rms(p.r, p.data, **BAND)
    out['circ_blr_free_1d'] = ifg.bandlimited_rms(p.r[c], p.data[c], **BAND)
    # the coordinate methods, mask and pad, the filter design functions and the named windows on a small map
    d, keep = small_map()
    out['small_data'], out['small_mask_in'] = d, keep
    d = prep(d)
    out['small_mask'] = I(_copy(d), dx=DX).mask(keep).data
    i = I(_copy(d), dx=DX)
    i.x                                 # cached, so that crop crops it and recenter shifts the cropped grid
    i.crop().recenter()
    out['small_recenter_x'], out['small_recenter_y'] = i.x, i.y
    i = I(_copy(d), dx=0).latcal(0.25)
    out['small_latcal_x'], out['small_latcal_y'], out['small_latcal_dx'] = i.x, i.y, i.dx
    out['small_strip_x'] = I(_copy(d), dx=DX).strip_latcal().x
    i = I(_copy(d), dx=DX).pad(samples=(3, 4))
    out['small_pad'], out['small_pad_x'] = i.data, i.x
    out['small_pad_zero'] = I(_copy(d), dx=DX).pad(0.0, shape=(41, 60)).data
    r = I(_copy(d), dx=DX).r
    for typ in ('lp', 'bp'):
        out[f'small_designfilt_{typ}'] = ifg.designfilt2d(r, DX, FILTERS[typ], typ)
    out['small_lpf'] = ifg.ideal_lpf_iir2d(r, DX, 0.3)
    f = I(_copy(d), dx=DX).fill(0).data
    for w in ('welch', 'hann'):
        out[f'small_window_{w}'] = ifg.make_window(f, DX, w)
    return {k: _host(v) for k, v in out.items()}


def reference_outputs():
    with reference.loaded(), warnings.catch_warnings():
        warnings.simplefilter('ignore')
        from prysm.conf import config
        config.precision = 64
        from prysm import interferogram, util
        from prysm.polynomials import lstsq
        return run(interferogram, util, lstsq)


def main():
    """Write tests/golden/interferogram*.npz from the unmodified reference."""
    with reference.loaded():
        from make_golden import save      # imports the reference
        save('interferogram.npz', reference_outputs())


if __name__ == '__main__':
    main()
