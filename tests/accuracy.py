"""The accuracy ledger of the extended-precision GPU suites, and the reference helpers their *_reference.py modules
share.

Every suite holds each figure to 1.5x the figure measured on an H100 (its `MEASURED` table, recorded with
PB_TEST_MEASUREMENTS), capped at a ceiling the suite's host test shows every modelled defect exceeds; a figure measured
as 0 stays 0.  `Ledger` is that rule, the worst figure of each name and the audit of figures with no measurement.
"""
import math
import os

import numpy as np

LDBL = np.longdouble
assert np.finfo(LDBL).nmant >= 63, (
    'the references need an 80-bit long double (x86-64); this host has '
    f'{np.finfo(LDBL).nmant + 1} mantissa bits')

# ---- launch geometry (csrc/common.cuh grid_for) --------------------------------------------------------------------
THREADS = 256
BLOCKS_PER_SM = 16              # grid_for's cap


def grid_for(n, sm_count, threads=THREADS):
    """csrc/common.cuh grid_for: ceil(n / threads) blocks, at least 1, at most sm_count * 16"""
    return max(1, min((n + threads - 1) // threads, sm_count * BLOCKS_PER_SM))


def sweep(sm_count, threads=THREADS):
    """items one sweep of a capped grid-stride launch covers"""
    return sm_count * BLOCKS_PER_SM * threads


# ---- figures --------------------------------------------------------------------------------------------------------
def ld(a):
    """the exact values the device got, as long double"""
    a = np.asarray(a)
    return a.astype(np.clongdouble if np.iscomplexobj(a) else LDBL)


def rel_l2(a, b):
    """||a - b|| / ||b|| in fp64"""
    return float(np.linalg.norm((a - b).ravel()) / np.linalg.norm(b.ravel()))


def _current_test():
    return os.environ.get('PYTEST_CURRENT_TEST', '').split(' ')[0]


class Ledger:
    """The bounds of a suite's figures and the worst figure of each name.

    `measured` maps a figure name to its measured value, or a case to {metric: value} (the name is 'case/metric').
    `ceiling` and `factor` are numbers or functions of the name; `key(name)` is the name's entry in `measured`.  The
    worst figure of a name is kept over the whole module, or over one test with `per_test`; `one_test_per_name` fails
    a name that a second test records, so that the measured table keeps every figure rather than the last of several.
    """

    def __init__(self, measured, ceiling, factor=1.5, key=None, per_test=False, one_test_per_name=False):
        self.measured = {}
        for k, v in measured.items():
            if isinstance(v, dict):
                self.measured.update({f'{k}/{metric}': m for metric, m in v.items()})
            else:
                self.measured[k] = v
        self.ceiling, self.factor = ceiling, factor
        self.key = key or (lambda name: name)
        self.per_test, self.one_test_per_name = per_test, one_test_per_name
        self.worst = {}         # name -> (figure, note)
        self.open = {}          # names recorded since the last done(), in order
        self.routes = []        # route failures since the last done()
        self.tests = {}         # name -> the test that recorded it
        self.test = None

    def bound(self, name):
        """factor x the measured figure, at most the ceiling; the smallest subnormal for a figure measured as 0; the
        ceiling for a figure with no entry"""
        cap = self.ceiling(name) if callable(self.ceiling) else self.ceiling
        m = self.measured.get(self.key(name))
        if m is None:
            return cap
        factor = self.factor(name) if callable(self.factor) else self.factor
        return min(factor * m, cap) if m > 0 else float(np.nextafter(0.0, 1.0))

    def _enter(self):
        """a new test starts with nothing open (what a failed test left is dropped)"""
        test = _current_test()
        if test != self.test:
            self.open.clear()
            self.routes.clear()
            self.test = test

    def record(self, name, value, note=None):
        """keep the worst figure of `name` and its note (NaN is the worst of all)"""
        self._enter()
        if self.one_test_per_name:
            assert self.tests.setdefault(name, self.test) == self.test, \
                f'{name} is recorded by {self.tests[name]} and {self.test}'
        value = float(value)
        old = self.worst.get(name) if not self.per_test or name in self.open else None
        if old is None or not (math.isnan(old[0]) or value <= old[0]):
            self.worst[name] = (value, note)
        self.open[name] = None

    def route(self, ok, msg):
        """a check of which kernels ran; done() fails with every one that did not hold"""
        self._enter()
        if not ok:
            self.routes.append(msg)

    def done(self):
        """every figure recorded since the last done() through conftest.within (PB_TEST_MEASUREMENTS keeps them), then
        one failure naming every figure over its bound, with its note, and every route that did not hold"""
        from conftest import within     # here, so that the reference modules importing this file need numpy only
        bad = []
        for name in self.open:
            value, note = self.worst[name]
            try:
                within(name, value, self.bound(name))
            except AssertionError as e:
                bad.append(f'{e} ({note})' if note else str(e))
        bad += self.routes
        self.open.clear()
        self.routes = []
        assert not bad, '\n'.join(bad)

    def check(self, name, value):
        """record one figure and hold it to its bound now"""
        self.record(name, value)
        self.done()

    def missing(self):
        """the figures recorded so far that have no measured entry"""
        return sorted(name for name in self.worst if self.key(name) not in self.measured)
