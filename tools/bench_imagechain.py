"""GPU timing of the SURVEY.md 8(f) rank-4 row: conv / apply_transfer_functions / fourier_resample (fp32).

    python tools/bench_imagechain.py
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import prysm_b200 as pb  # noqa: E402
from benchlib import timed  # noqa: E402
from prysm_b200 import _ops, convolution as CV, fttools as FT  # noqa: E402


pb.config.precision = 32
gen = torch.Generator(device='cuda').manual_seed(3)
for n in (2048, 4096):
    o = torch.rand((n, n), generator=gen, device='cuda')
    h = torch.rand((n, n), generator=gen, device='cuda')
    us, nl = timed(lambda: CV.conv(o, h), 20)
    us *= 1e6
    print(f'conv real x real {n}^2 (packed: 1 forward + 1 inverse FFT): {us:.0f} us, {nl:.0f} launches')

    def three_fft():
        O = _ops.fft2(o, (n, n), dir=-1, shift_in=True)
        H = _ops.fft2(h, (n, n), dir=-1, shift_in=True)
        return _ops.fft2(_ops.binary('mul', O, H), (n, n), dir=+1, scale=1.0 / (n * n), shift_out=True)
    us, nl = timed(three_fft, 20)
    us *= 1e6
    print(f'conv real x real {n}^2 the reference way (3 FFTs + product): {us:.0f} us, {nl:.0f} launches')
    tf = torch.rand((n, n), generator=gen, device='cuda')
    us, nl = timed(lambda: CV.apply_transfer_functions(o, 1.0, [tf, tf]), 20)
    us *= 1e6
    print(f'apply_transfer_functions {n}^2, 2 array TFs: {us:.0f} us, {nl:.0f} launches')
f = torch.rand((1024, 1024), generator=gen, device='cuda')
us, nl = timed(lambda: FT.fourier_resample(f, 2), 20)
us *= 1e6
print(f'fourier_resample 1024^2 -> 2048^2 (plan rebuilt per call, like the reference): {us:.0f} us, {nl:.0f} launches')
