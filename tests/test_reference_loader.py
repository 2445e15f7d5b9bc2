"""CPU: reference.loaded() (oracle/reference.py) leaves no module of the reference imported and REF off sys.path, also
when its body raises.  The check is on the whole of sys.modules, so it also fails when a test that ran earlier in the
session left the reference imported."""
import sys

import pytest

import reference

pytestmark = pytest.mark.skipif(not reference.installed(), reason='reference prysm not installed')


def reference_modules():
    return sorted(name for name in sys.modules if name.split('.')[0] == 'prysm')


def test_loaded_forgets_the_reference_on_exit():
    with reference.loaded():
        import prysm.propagation  # noqa: F401
        assert 'prysm.propagation' in sys.modules and sys.path[0] == reference.REF
    assert reference_modules() == []
    assert reference.REF not in sys.path


def test_loaded_forgets_the_reference_when_the_body_raises():
    with pytest.raises(RuntimeError, match='body'):
        with reference.loaded():
            import prysm.propagation  # noqa: F401
            raise RuntimeError('body')
    assert reference_modules() == []
    assert reference.REF not in sys.path
