"""Where the unmodified reference package (prysm) is, and how tests and tools import it for a while.

REF is $PRYSM_REFERENCE, or else oracle/_ref, where oracle/install_reference.py copies it.  Inside `loaded()`,
`import prysm` finds the reference; on leaving it every module imported meanwhile is forgotten, so what a later test
imports as `prysm` does not depend on which tests ran before it."""
import contextlib
import os
import sys

REF = os.environ.get('PRYSM_REFERENCE', os.path.join(os.path.dirname(os.path.abspath(__file__)), '_ref'))


def installed():
    """Whether REF holds a prysm package."""
    return os.path.isdir(os.path.join(REF, 'prysm'))


@contextlib.contextmanager
def loaded(also=()):
    """Put REF first on sys.path (writing no bytecode into it) for the block.  On exit, also when the block raises,
    every module imported inside whose top-level name is `prysm` or one of `also` leaves sys.modules and REF leaves
    sys.path."""
    names = {'prysm', *also}
    before = set(sys.modules)
    write_bytecode = sys.dont_write_bytecode
    sys.dont_write_bytecode = True
    sys.path.insert(0, REF)
    try:
        yield
    finally:
        for name in set(sys.modules) - before:
            if name.split('.')[0] in names:
                del sys.modules[name]
        sys.path.remove(REF)
        sys.dont_write_bytecode = write_bytecode
