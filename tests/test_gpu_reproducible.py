"""GPU: two processes running the same script give the same bits.

The focus pipeline on stacks at N = 1024 and 2048, both directions, and the matrix DFT at two shapes: 512^2 -> 256^2
(split-K second stage) and 1024^2 -> 512^2 (stream-K first stage on an H100: 64 tiles on 132 SMs; the tile owner adds
its neighbours' partials in a fixed order).  Nothing a process sets up (handles, tables, scratch arenas) may change an
output.

The fp64 reductions, at 512^2 (past the 4-blocks-per-SM cap of the grid fold) in both precisions: each is called twice
in the process and must give the same bits both times, and the two processes must agree."""
import hashlib
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_SCRIPT = r'''
import hashlib, sys
import numpy as np, torch
sys.path.insert(0, %(root)r)
import prysm_b200 as pb
from prysm_b200 import _ops, fttools as F
pb.config.precision = 32
gen = torch.Generator(device='cuda').manual_seed(11)
def rnd(*s): return torch.complex(torch.randn(s, generator=gen, device='cuda'), torch.randn(s, generator=gen, device='cuda'))
h = hashlib.sha1()
for n, b in ((1024, 5), (2048, 3)):
    stack = rnd(b, n, n)
    for d in (-1, 1):
        out = _ops.fft2_batch(stack, (2 * n, 2 * n), dir=d, scale=1.0 / (2 * n), shift_in=True, shift_out=True)
        h.update(out.cpu().numpy().tobytes())
print('focus', h.hexdigest())
h = hashlib.sha1()
for n, m in ((512, 256), (1024, 512)):
    x = (np.arange(n) - n // 2) * 0.1
    f = (np.arange(m) - m // 2) * (0.37 / (n * 0.1))
    ex = F.MDFT(x, x, f, f, -1, 0.5)
    assert ex._tc is not None
    h.update(ex(rnd(n, n)).cpu().numpy().tobytes())
print('mdft', h.hexdigest())

def bits(v):
    if isinstance(v, dict):
        return b''.join(bits(v[k]) for k in sorted(v))
    if isinstance(v, (tuple, list)):
        return b''.join(bits(x) for x in v)
    return (v.detach().cpu().numpy() if torch.is_tensor(v) else np.asarray(v)).tobytes()
h = hashlib.sha1()
def twice(name, f):
    a, b = bits(f()), bits(f())
    assert a == b, name + ' gave different bits on a second call'
    h.update(a)
n = 512
for rd in (torch.float32, torch.float64):
    pb.config.precision = 32 if rd == torch.float32 else 64
    cd = torch.complex64 if rd == torch.float32 else torch.complex128
    def rr(*s): return torch.randn(s, generator=gen, device='cuda', dtype=torch.float64).to(rd)
    a, b, w = rnd(n, n).to(cd), rnd(n, n).to(cd), rr(n, n)
    twice('dot', lambda: _ops.dot(a, b))
    twice('dot_w', lambda: _ops.dot(a, b, w))
    modes, bar = rr(3, n, n), rr(n, n)
    twice('mode_projection', lambda: _ops.mode_projection(modes, bar))
    psf = rr(n, n).abs()
    twice('centroid', lambda: pb.psf.centroid(psf, 1.0))
    twice('encircled_energy', lambda: pb.otf.encircled_energy(psf, 1.0, [5.0, 20.0, 80.0]))
    twice('mtf_adjoint', lambda: pb.otf.mtf_from_psf_adjoint(bar, psf=psf, dx=1.0))
    twice('otf_adjoint', lambda: pb.otf.otf_from_psf_adjoint(a, psf=psf, dx=1.0))
    twice('conv', lambda: pb.convolution.conv(psf * 1e5, bar.abs()))
    def balanced(wb, img, *gains):
        img = img.clone()
        wb(img, *gains, safe=True, saturation=1.0)
        return img
    rgb = rr(n, n, 3).abs()
    twice('wb_prescale', lambda: balanced(pb.bayer.wb_prescale, psf, 1.5, 1.0, 1.0, 2.0))
    twice('wb_postscale', lambda: balanced(pb.bayer.wb_postscale, rgb, 1.5, 1.0, 2.0))
    fields = {0: [rr(n, n) for _ in range(3)], 1: [rr(n, n) for _ in range(2)]}
    E = rnd(n, n).to(cd)
    twice('multimode_coupling', lambda: pb.fibers.multimode_coupling(E, fields))
    x, y = pb.coordinates.make_xy_grid((n, n), diameter=8.0)
    cha = pb.segmented.CompositeHexagonalAperture(x, y, 2, 1.32, 0.007)
    cha.prepare_opd_bases(pb.polynomials.zernike_nm_seq, [(0, 0), (1, 1), (1, -1), (2, 0)])
    g = rr(n, n)
    twice('compose_opd_adjoint', lambda: cha.compose_opd_adjoint(g))
    d = rr(n, n)
    d[::7, ::5] = float('nan')
    twice('nan_stats', lambda: _ops.nan_stats(d))
print('reductions', h.hexdigest())
'''


def _run():
    r = subprocess.run([sys.executable, '-c', _SCRIPT % {'root': ROOT}], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    return dict(line.split() for line in r.stdout.strip().splitlines() if line.split()[0] in ('focus', 'mdft', 'reductions'))


@pytest.mark.gpu
def test_two_processes_give_the_same_bits():
    first = _run()
    second = _run()
    assert second['focus'] == first['focus']
    assert second['mdft'] == first['mdft']
    assert second['reductions'] == first['reductions']
