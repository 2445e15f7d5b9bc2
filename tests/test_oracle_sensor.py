"""CPU: the reference, where it is installed (oracle/_ref), re-derives every image-sensor fixture (tests/golden/sensor*.npz)
from the inputs tests/sensor_oracle.py builds; the Malvar filters the engine uses are the reference's and are symmetric
under a 180-degree rotation, so the engine's correlation equals scipy's convolution."""
import os

import numpy as np
import pytest

from conftest import load_golden
import sensor_oracle as O
import reference


@pytest.fixture(scope='module')
def golden():
    return load_golden('sensor.npz')


def test_fixture_inputs_are_deterministic():
    a, b = O.inputs(), O.inputs()
    assert sorted(a) == sorted(b)
    for k in a:
        assert np.array_equal(a[k], b[k]), k


def test_reference_rederives_the_fixtures(golden):
    if not reference.installed():
        pytest.skip('reference prysm not installed')
    mine = O.reference_outputs()
    assert sorted(mine) == sorted(golden)
    for k, v in golden.items():
        got = np.asarray(mine[k])
        assert got.dtype == v.dtype, k
        np.testing.assert_array_equal(got, v, err_msg=k)


def test_fixtures_cover_every_bayer_function_and_the_error_cases(golden):
    for prefix in ('malvar_', 'deint_', 'comp_', 'recomp_', 'decomp_', 'wbpre_0', 'wbpre_1', 'wbpost_0', 'wbpost_1',
                   'superres_', 'pixel_', 'lut_', 'expose_'):
        assert any(k.startswith(prefix) for k in golden), prefix
    for shape in O.SHAPES:
        assert any(k.endswith(f'{shape[0]}x{shape[1]}') and k.startswith('malvar_u16') for k in golden), shape
    for k in ('bad_malvar_grbg', 'bad_deint_GRBG', 'bad_comp_grbg', 'bad_recomp_GRBG', 'bad_decomp_grbg',
              'bad_wbpre_GRBG', 'bad_superres_bggr', 'bad_superres_RGGB'):
        assert str(golden[k]) == 'NotImplementedError', k
    assert str(golden['lut_short_overflow']) == 'IndexError'
    assert str(golden['expose_bits33']) == 'ValueError'
    assert str(golden['deint_f64_rggb_3x5']) == 'ValueError'      # odd sides: the planes' shapes differ


def test_malvar_filters_are_the_references_and_point_symmetric():
    from prysm_b200 import bayer as ours
    if not reference.installed():
        pytest.skip('reference prysm not installed')
    with reference.loaded():
        from prysm import bayer
        ref = {'G_at_R_or_B': bayer.kernel_G_at_R_or_B, 'R_at_G_in_RB': bayer.kernel_R_at_G_in_RB,
               'R_at_G_in_BR': bayer.kernel_R_at_G_in_BR, 'R_at_B_in_BB': bayer.kernel_R_at_B_in_BB}
    assert sorted(ref) == sorted(ours.MALVAR_KERNELS)
    for name, k in ours.MALVAR_KERNELS.items():
        np.testing.assert_array_equal(k, np.asarray(ref[name], dtype=np.float64), err_msg=name)
        assert np.array_equal(k, k[::-1, ::-1]), name
        assert k.sum() == 8.0, name


def test_malvar_taps_in_the_kernel_source_match_the_python_table():
    """csrc/sensor.cu carries the taps as a literal table: it must be the one the Python module documents."""
    import re
    from prysm_b200 import bayer as ours
    src = open(os.path.join(O.ROOT, 'prysm_b200', 'csrc', 'sensor.cu')).read()
    body = src[src.index('kMalvarTaps[4][5][5] = {'):]
    body = body[:body.index('};')]
    nums = [float(v.rstrip('f')) for v in re.findall(r'-?\d+(?:\.\d+)?f?', body.split('=', 1)[1])]
    table = np.array(nums).reshape(4, 5, 5)
    order = ('G_at_R_or_B', 'R_at_G_in_RB', 'R_at_G_in_BR', 'R_at_B_in_BB')
    for i, name in enumerate(order):
        np.testing.assert_array_equal(table[i], ours.MALVAR_KERNELS[name], err_msg=name)
