"""GPU: two processes running the same script give the same bits.

The focus pipeline on stacks at N = 1024 and 2048, both directions, and the matrix DFT at two shapes: 512^2 -> 256^2
(split-K second stage) and 1024^2 -> 512^2 (stream-K first stage on an H100: 64 tiles on 132 SMs; the tile owner adds
its neighbours' partials in a fixed order).  Nothing a process sets up (handles, tables, scratch arenas) may change an
output."""
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
'''


def _run():
    r = subprocess.run([sys.executable, '-c', _SCRIPT % {'root': ROOT}], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    return dict(line.split() for line in r.stdout.strip().splitlines() if line.split()[0] in ('focus', 'mdft'))


@pytest.mark.gpu
def test_two_processes_give_the_same_bits():
    first = _run()
    second = _run()
    assert second['focus'] == first['focus']
    assert second['mdft'] == first['mdft']
