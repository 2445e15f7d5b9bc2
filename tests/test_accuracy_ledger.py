"""CPU: the bound rule of tests/accuracy.py's Ledger, which every extended-precision GPU suite holds its figures to."""
import numpy as np
import pytest

import conftest
from accuracy import Ledger

TINY = float(np.nextafter(0.0, 1.0))


def test_bound_rule():
    led = Ledger({'a': 2e-7, 'zero': 0.0, 'big': 1e-3}, 1e-6)
    assert led.bound('a') == 1.5 * 2e-7
    assert led.bound('big') == 1e-6                 # capped at the ceiling
    assert led.bound('zero') == TINY                # measured as exact: stays exact
    assert led.bound('none') == 1e-6                # no entry: the ceiling


def test_table_flattening():
    led = Ledger({'c128/fft/64': dict(linf=2e-16, l2=1e-16), 'c64/x': 3e-7}, 1.0)
    assert led.measured == {'c128/fft/64/linf': 2e-16, 'c128/fft/64/l2': 1e-16, 'c64/x': 3e-7}
    assert led.bound('c128/fft/64/l2') == 1.5 * 1e-16
    assert led.bound('c128/fft/64/other') == 1.0


def test_callable_ceiling_factor_and_key():
    ceil = {'c64': 1e-6, 'c128': 1e-14}
    led = Ledger({'c64/a': 1e-6, 'c128/a': 1e-15, 'c128/atomic': 1e-15}, lambda n: ceil[n.split('/')[0]],
                 factor=lambda n: 3.0 if n.endswith('atomic') else 1.5)
    assert led.bound('c64/a') == 1e-6 and led.bound('c128/a') == 1.5 * 1e-15
    assert led.bound('c128/atomic') == 3 * 1e-15
    assert led.bound('c128/none') == 1e-14
    led = Ledger({'legendre/value': 2.0}, 1e4, key=lambda n: n.split('/', 1)[1])
    assert led.bound('32/legendre/value') == led.bound('64/legendre/value') == 3.0
    assert led.missing() == []
    led.record('32/legendre/value', 1.0)
    led.record('32/cheby1/value', 1.0)
    assert led.missing() == ['32/cheby1/value']


def test_worst_figure_notes_and_one_failure(monkeypatch):
    seen = {}
    monkeypatch.setattr(conftest, '_MEASURED', seen)
    led = Ledger({'a': 1.0, 'b': 1.0, 'c': 0.0}, 10.0)
    led.record('a', 1.2, 'first')
    led.record('a', 1.4, 'second')
    led.record('a', 1.3, 'third')
    led.done()
    assert seen['a'] == {'measured': 1.4, 'bound': 1.5}
    led.record('a', 1.6, 'over')
    led.record('b', float('nan'), 'nan')
    led.record('b', 0.5)                             # NaN stays the worst
    led.record('c', 0.0)
    led.route(False, 'route: the wrong kernel ran')
    with pytest.raises(AssertionError) as e:
        led.done()
    msg = str(e.value)
    assert 'a: 1.600e+00 is not below 1.500e+00' in msg and '(over)' in msg
    assert 'b: nan is not below' in msg and '(nan)' in msg
    assert 'route: the wrong kernel ran' in msg and 'c:' not in msg
    led.done()                                       # done() starts over: nothing open
    led.record('a', 1.0)
    with pytest.raises(AssertionError):
        led.done()                                   # the worst over the module is still 1.6


def test_per_test_and_one_test_per_name(monkeypatch):
    monkeypatch.setattr(conftest, '_MEASURED', {})
    led = Ledger({'a': 1.0}, 10.0, per_test=True, one_test_per_name=True)
    monkeypatch.setenv('PYTEST_CURRENT_TEST', 'x.py::one (call)')
    led.record('a', 1.6)
    led.route(False, 'left behind by a failed test')
    monkeypatch.setenv('PYTEST_CURRENT_TEST', 'x.py::two (call)')
    with pytest.raises(AssertionError, match='a is recorded by x.py::one and x.py::two'):
        led.record('a', 1.0)
    led = Ledger({'a': 1.0}, 10.0, per_test=True)
    led.record('a', 1.6)
    monkeypatch.setenv('PYTEST_CURRENT_TEST', 'x.py::three (call)')
    led.record('a', 1.0)                             # a new test: its own worst, and nothing left open
    led.done()
    assert conftest._MEASURED['a']['measured'] == 1.0
