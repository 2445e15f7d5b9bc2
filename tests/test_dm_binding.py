"""CPU: set_backend_to_b200() re-binds prysm.x.dm.DM and prysm.coordinates.warp, and set_backend_to_defaults()
restores them.  Runs where the unmodified reference is installed in oracle/_ref or PRYSM_REFERENCE names one."""
import pytest

import reference


@pytest.fixture()
def prysm_pkg():
    if not reference.installed():
        pytest.skip('reference prysm not installed')
    with reference.loaded():
        import prysm
        import prysm.x.dm  # noqa: F401
        yield prysm


def test_dm_and_warp_rebinding_round_trip(prysm_pkg):
    import prysm.coordinates as pco
    import prysm.x.dm as pdm
    from prysm_b200 import mathops, coordinates as bco, dm as bdm
    orig = (pdm.DM, pco.warp)
    names = mathops.set_backend_to_b200()
    try:
        assert ('prysm.x.dm', 'DM') in names and ('prysm.coordinates', 'warp') in names
        assert pdm.DM is bdm.DM and pco.warp is bco.warp
        from prysm.x.dm import DM
        assert DM is bdm.DM                      # a DM constructed after the switch is an engine DM
    finally:
        mathops.set_backend_to_defaults()
    assert (pdm.DM, pco.warp) == orig
    assert mathops._saved == {}
