"""CPU: the references of tests/test_gpu_tuned_vs_fp64.py are right before they meet a GPU -- the closed form of a focused
sum of impulses against the oracle's FFT, and the output-row classes of the focus pair against a restatement of the
intermediate's layout (DESIGN §3, §4.1)."""
import numpy as np
import pytest

import prysm_oracle as O
from test_gpu_tuned_vs_fp64 import CLASSES, IMPULSE_SUMS, impulse_focus, impulse_pixels, plane1_keep, row_classes


@pytest.mark.parametrize('inverse', [False, True])
@pytest.mark.parametrize('N', [16, 32, 64])
@pytest.mark.parametrize('name', sorted(IMPULSE_SUMS))
def test_impulse_closed_form_matches_the_oracle(N, inverse, name):
    px = impulse_pixels(N)
    terms = IMPULSE_SUMS[name]
    a = np.zeros((N, N), dtype=np.complex128)
    for p, v in terms:
        a[px[p]] += v
    want = (O.unfocus if inverse else O.focus)(a, 2)
    got = impulse_focus(N, 2, [px[p] for p, _ in terms], [v for _, v in terms], inverse)
    assert np.abs(got - want).max() < 1e-13 * np.abs(want).max()


def test_impulse_closed_form_sees_a_wrong_pixel():
    """the comparison the GPU test makes can tell neighbouring pixels and the two directions apart"""
    N = 16
    a = np.zeros((N, N), dtype=np.complex128)
    a[3, 5] = 1.0
    want = O.focus(a, 2)
    for pix, inv in (((3, 6), False), ((4, 5), False), ((3, 5), True)):
        assert np.abs(impulse_focus(N, 2, [pix], [1.0], inv) - want).max() > 0.1 * np.abs(want).max()


def kept_bytes_from_source():
    """kPlane1KeepBytes as csrc/fft_tuned.cu states it"""
    import os
    import re
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'prysm_b200', 'csrc',
                            'fft_tuned.cu')).read()
    m = re.search(r'constexpr long long kPlane1KeepBytes = (\d+)LL << (\d+);', src)
    assert m, 'kPlane1KeepBytes not found in csrc/fft_tuned.cu'
    return int(m.group(1)) << int(m.group(2))


def test_plane1_keep_is_two_mib_of_whole_thread_ranges():
    from test_gpu_tuned_vs_fp64 import PLANE1_KEEP_BYTES
    assert PLANE1_KEEP_BYTES == kept_bytes_from_source()
    # line groups of L/4 lines x 128 bytes, in whole ranges of L/64 groups: all of plane 1 at L = 512, none at 4096
    assert [plane1_keep(L) for L in (256, 512, 1024, 2048, 4096)] == [64, 128, 64, 32, 0]


@pytest.mark.parametrize('L', [256, 512, 1024, 2048, 4096])
def test_row_classes_against_the_layout(L):
    """Brute force: walk the intermediate as the kernels do.  The row kernel stores row j of plane p at output row
    (2j + p + L) mod 2L.  A row of plane 1 takes 8L bytes, and the column kernel picks the L2 policy per thread range of
    L/16 rows (rows g L/16 .. (g + 1) L/16 - 1), so a row is kept when its whole range lies within the first
    kPlane1KeepBytes of plane 1.  Plane 0 is always kept."""
    keep, row_bytes, rng = kept_bytes_from_source(), 8 * L, L // 16
    want = np.full(2 * L, -1)
    for p in range(2):
        for j in range(L):
            orow = (2 * j + p + L) % (2 * L)
            assert want[orow] == -1           # a permutation of the output rows
            if p == 0:
                want[orow] = 0
            else:
                want[orow] = 1 if (j // rng + 1) * rng * row_bytes <= keep else 2
    got = row_classes(L)
    assert (got == want).all()
    counts = [int((got == c).sum()) for c in range(len(CLASSES))]
    assert counts[0] == L and sum(counts) == 2 * L
