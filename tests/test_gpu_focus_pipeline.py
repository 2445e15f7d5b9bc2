"""GPU: the plane-unit focus kernel (PB_FOCUS_V=4, csrc/focus_fused.cu) gives the same bits as the column + row kernel
pair (PB_FOCUS_V=2).

Both do the same per-column and per-row arithmetic in the same order, so the SHA-1 of every output must agree:
N = 2048 stacks of 2, 3 and 16 fields and one of 66 (two launches: the counter arrays take 64 fields), both directions,
complex, intensity and accumulated-intensity outputs, and an output with padded row and field strides.  In the v4
process two repeated calls and a CUDA-graph replay (prysm_b200.graphs) give the same bits too.  The switches are read
once per process, so each variant runs in a subprocess, under a timeout: the kernel's workers spin on each other's
counters.
"""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_SCRIPT = r'''
import hashlib, sys
import torch
sys.path.insert(0, %(root)r)
import prysm_b200 as pb
from prysm_b200 import _ops, _capi, graphs
pb.config.precision = 32
n = 2048

def digest(t):
    h = hashlib.sha1()
    flat = t.reshape(t.shape[0], -1)
    for i in range(flat.shape[0]):      # field by field: the large case does not need a host copy of the whole stack
        h.update(flat[i].cpu().numpy().tobytes())
    return h.hexdigest()

def stack(b, seed):
    gen = torch.Generator(device='cuda').manual_seed(seed)
    return torch.complex(torch.randn((b, n, n), generator=gen, device='cuda'), torch.randn((b, n, n), generator=gen, device='cuda'))

def run(x, d, kind=_capi.OUT_COMPLEX, out=None):
    return _ops.fft2_batch(x, (2 * n, 2 * n), dir=d, scale=1.0 / (2 * n), shift_in=True, shift_out=True, out_kind=kind, out=out)

for b in (2, 3, 16):
    x = stack(b, 100 + b)
    for d in (-1, 1):
        print('complex', b, d, digest(run(x, d)))
        torch.cuda.empty_cache()
x = stack(3, 7)
print('intensity', digest(run(x, -1, _capi.OUT_INTENSITY)))
gen = torch.Generator(device='cuda').manual_seed(8)
acc = torch.rand((3, 2 * n, 2 * n), generator=gen, device='cuda')
print('accumulate', digest(run(x, 1, _capi.OUT_ACCUMULATE, out=acc)))
big = torch.zeros((3, 2 * n + 3, 2 * n + 6), dtype=torch.complex64, device='cuda')   # padded field and row strides
view = big[:, 1:2 * n + 1, 2:2 * n + 2]
run(x, -1, out=view)
print('padded', digest(big))
del big, view, acc
first = digest(run(x, -1))
print('repeat', first == digest(run(x, -1)))
step = graphs.capture(lambda w: run(w, -1), x)
print('graph', digest(step(x)) == first)
step.close()
del x, step
torch.cuda.empty_cache()
x = stack(66, 9)
print('two_launches', digest(run(x, -1, _capi.OUT_INTENSITY)))
'''


def _run(version):
    e = {k: v for k, v in os.environ.items() if not k.startswith('PB_')}
    e['PB_FOCUS_V'] = version
    r = subprocess.run([sys.executable, '-c', _SCRIPT % {'root': ROOT}], env=e, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return [line for line in r.stdout.strip().splitlines() if line.split()[0] in
            ('complex', 'intensity', 'accumulate', 'padded', 'repeat', 'graph', 'two_launches')]


@pytest.mark.gpu
def test_plane_kernel_is_bit_identical_to_the_kernel_pair():
    base = _run('2')
    plane = _run('4')
    assert 'repeat True' in plane and 'graph True' in plane
    assert [ln for ln in plane if ln.split()[0] not in ('repeat', 'graph')] == \
           [ln for ln in base if ln.split()[0] not in ('repeat', 'graph')]
