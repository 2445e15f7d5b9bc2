"""Copy the unmodified reference package (prysm v0.22, pure Python) into oracle/_ref/prysm.

    python oracle/install_reference.py [SRC]        (SRC: a prysm source checkout; default $PRYSM_REFERENCE)

oracle/_ref is git-ignored.  The tests and tools/bench_*.py import the reference from there through
oracle/reference.py (which a PRYSM_REFERENCE checkout overrides), and `bench.py --impl reference` imports it directly;
they skip or fail loudly where it was not installed.
The package is copied file for file and checked to be identical to its source: nothing in it is changed."""
import filecmp
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
DST = os.path.join(HERE, '_ref')


def install(src):
    """Returns the installed package directory, or None when `src` holds no prysm package."""
    pkg = os.path.join(src, 'prysm')
    if not os.path.isfile(os.path.join(pkg, '__init__.py')):
        return None
    dst = os.path.join(DST, 'prysm')
    tmp = dst + '.tmp'
    shutil.rmtree(tmp, ignore_errors=True)
    shutil.copytree(pkg, tmp, ignore=shutil.ignore_patterns('__pycache__', '*.pyc'))
    _check_identical(pkg, tmp)
    shutil.rmtree(dst, ignore_errors=True)
    os.replace(tmp, dst)
    return dst


def _check_identical(a, b):
    """Same file names in every directory and the same bytes in every file (compared by content, not by stat)."""
    cmp = filecmp.dircmp(a, b, ignore=['__pycache__'])
    bad = cmp.left_only + cmp.right_only + cmp.funny_files
    bad += [f for f in cmp.common_files if not filecmp.cmp(os.path.join(a, f), os.path.join(b, f), shallow=False)]
    if bad:
        raise RuntimeError(f'reference copy differs from {a}: {bad}')
    for sub in cmp.common_dirs:
        _check_identical(os.path.join(a, sub), os.path.join(b, sub))


if __name__ == '__main__':
    src = sys.argv[1] if len(sys.argv) > 1 else os.environ.get('PRYSM_REFERENCE', '')
    out = install(src)
    print(out if out else f'no prysm package under {src!r}')
    sys.exit(0 if out else 1)
