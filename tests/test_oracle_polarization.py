"""CPU: the reference, where it is installed (oracle/_ref), re-derives every polarization fixture
(tests/golden/polarization*.npz) from the inputs tests/polarization_oracle.py builds."""
import numpy as np
import pytest

from conftest import load_golden
import polarization_oracle as O
import reference


@pytest.fixture(scope='module')
def golden():
    return load_golden('polarization.npz')


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
        np.testing.assert_array_equal(np.asarray(mine[k]), v, err_msg=k)
