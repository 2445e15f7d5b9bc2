"""GPU timing of the SURVEY.md 8(f) rows: Lyot-coronagraph compositions and the phase-retrieval gradient chain.

    python tools/bench_coronagraph.py

Prints one line per workload: us per call (CUDA events, 20 reps after warm-up) and the kernel launches per call."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import prysm_b200 as pb  # noqa: E402
from benchlib import timed  # noqa: E402
from prysm_b200 import _ops, propagation as P  # noqa: E402

HeNe = 0.6328


gen = torch.Generator(device='cuda').manual_seed(1)


def crand(shape, dt):
    rd = torch.float32 if dt == torch.complex64 else torch.float64
    return torch.complex(torch.randn(shape, generator=gen, device='cuda', dtype=rd),
                         torch.randn(shape, generator=gen, device='cuda', dtype=rd))


for prec in (32, 64):
    pb.config.precision = prec
    cdt = torch.complex64 if prec == 32 else torch.complex128
    # single-executor Lyot coronagraph: 1024^2 pupil <-> 1024^2 focal plane
    n = m = 1024
    w = crand((n, n), cdt)
    fpm = torch.rand((m, m), generator=gen, device='cuda', dtype=w.real.dtype)
    lyot = torch.rand((n, n), generator=gen, device='cuda', dtype=w.real.dtype)
    for kind in ('mdft', 'czt'):
        ex = P.prepare_executor(10.0 / n, n, 1.0, m, HeNe, 100.0, kind=kind)
        tc = kind == 'mdft' and getattr(ex, '_tc', None) is not None and getattr(ex, '_tc_adj', None) is not None
        us, nl = timed(lambda: P.to_fpm_and_back(w, fpm, ex), 20)
        us *= 1e6
        print(f'[p{prec}] to_fpm_and_back {n}^2<->{m}^2 {kind}{" (wgmma both legs)" if tc else ""}: {us:.0f} us, {nl:.0f} launches')
        us, nl = timed(lambda: P.babinet(w, lyot, fpm, ex), 20)
        us *= 1e6
        print(f'[p{prec}] babinet         {n}^2<->{m}^2 {kind}: {us:.0f} us, {nl:.0f} launches')
        step = pb.graphs.capture(lambda w_: P.babinet(w_, lyot, fpm, ex), w)
        us, _ = timed(lambda: step(w), 20)
        us *= 1e6
        print(f'[p{prec}] babinet         {n}^2<->{m}^2 {kind}, CUDA graph replay: {us:.0f} us')
        g = crand((n, n), cdt)
        us, nl = timed(lambda: P.babinet_adjoint(g, lyot, fpm, ex), 20)
        us *= 1e6
        print(f'[p{prec}] babinet_adjoint {n}^2<->{m}^2 {kind}: {us:.0f} us, {nl:.0f} launches')
    # the reference's vortex rig (tests/test_propagation.py:463-541): 384^2 pupil, 640^2 + 5 x 256^2 focal levels
    npup, nd, pdx, efl = 384, 320, 0.05, 100.0
    period = HeNe * efl / pdx
    pupil = crand((npup, npup), cdt)
    vm = P.vortex_phase_mask(2)
    for kind in ('mdft', 'czt'):
        mex = P.prepare_multiresolution(pdx, npup, period / (2 * nd), 2 * nd, HeNe, efl, num_levels=6, fine_samples=256, kind=kind)
        us, nl = timed(lambda: P.to_fpm_and_back_multiresolution(pupil, vm, mex), 20)
        us *= 1e6
        print(f'[p{prec}] vortex 6-level multiresolution 384^2 {kind}: {us:.0f} us, {nl:.0f} launches')
        us, nl = timed(lambda: P.to_fpm_and_back_multiresolution_adjoint(pupil, vm, mex), 20)
        us *= 1e6
        print(f'[p{prec}] vortex 6-level multiresolution adjoint 384^2 {kind}: {us:.0f} us, {nl:.0f} launches')
        step = pb.graphs.capture(lambda w_: P.to_fpm_and_back_multiresolution(w_, vm, mex), pupil)
        ref = P.to_fpm_and_back_multiresolution(pupil, vm, mex)
        err = float((step(pupil) - ref).abs().max() / ref.abs().max())
        us, _ = timed(lambda: step(pupil), 20)
        us *= 1e6
        print(f'[p{prec}] vortex 6-level multiresolution 384^2 {kind}, CUDA graph replay: {us:.0f} us (max diff vs eager {err:.1e})')
    # modal phase-retrieval gradient (docs/source/how-tos/Differentiable Optical Models.ipynb): 512^2 pupil -> 256^2 PSF, 19 modes
    npup, npsf = 512, 256
    amp = torch.ones((npup, npup), device='cuda', dtype=w.real.dtype)
    basis = torch.randn((19, npup, npup), generator=gen, device='cuda', dtype=w.real.dtype)
    coefs = np.random.default_rng(0).random(19) * 25
    target = torch.rand((npsf, npsf), generator=gen, device='cuda', dtype=w.real.dtype)
    ex = None

    def cost_grad():
        global ex
        phs = pb.polynomials.sum_of_2d_modes(basis, coefs)
        wf = P.Wavefront.from_amp_and_phase(amp, phs, HeNe, 10.0 / npup)
        if ex is None:
            ex = wf.prepare_executor(100.0, 2.0, npsf)
        foc = wf.focus_dft(ex)
        diff = _ops.binary('sub', _ops.ascomplex(foc.intensity.data), _ops.ascomplex(target)).real   # dcost/dI up to a scale
        fbar = foc.intensity_adjoint(diff)
        wbar = fbar.focus_dft_adjoint(ex)
        pbar = wf.from_amp_and_phase_adjoint_phase(wbar)
        return pb.polynomials.sum_of_2d_modes_adjoint(basis, pbar)

    us, nl = timed(cost_grad, 20)
    us *= 1e6
    print(f'[p{prec}] modal phase-retrieval cost+gradient 512^2 -> 256^2, 19 modes: {us:.0f} us, {nl:.0f} launches')
    ex = None
