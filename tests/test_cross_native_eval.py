"""The cross's per-distinct-value function evaluated by the library (lowering.numeric_program ->
dampr_host_eval_f64) against CPython itself, bit for bit, on a million random ints; expressions outside the
lowered set, and values for which CPython raises, must come back as None (the caller then runs Python)."""
import math

import numpy as np
import pytest

from dampr_b200 import lowering, plan


def _comp(fn, pick=None):
    """the expression of one output of a cross function fn(inner, outer), as _lower_cross sees it"""
    e = lowering.analyze(fn)
    assert e is not None
    return e.a[pick] if pick is not None else e


def _python(fn, vals, total, pick=None):
    out = []
    for v in vals.tolist():
        r = fn(total, (None, v))
        out.append(r[pick] if pick is not None else r)
    return np.array(out, dtype=np.float64)


def _same_bits(a, b):
    return a.dtype == b.dtype == np.float64 and np.array_equal(a.view(np.uint64), b.view(np.uint64))


@pytest.fixture(scope="module")
def counts():
    rng = np.random.default_rng(7)
    # document frequencies of a Zipf corpus (tens to ~10^8) plus the small and huge ends of int64
    v = np.concatenate((rng.integers(1, 200_000_000, 900_000), rng.integers(1, 100, 90_000),
                        rng.integers(1 << 40, 1 << 52, 10_000)))
    return rng.permutation(v).astype(np.int64)


FNS = [
    ("bench idf", lambda total, df: (df[0], df[1], math.log(1 + (float(total) / df[1]))), 2),
    ("log(total/df)", lambda total, df: math.log(total / df[1]), None),
    ("log(float(total)/df)", lambda total, df: math.log(float(total) / df[1]), None),
    ("float arithmetic", lambda total, df: (df[1] * 0.5 - total) / 3.0 + 1e-9, None),
    ("int then float", lambda total, df: float(total - df[1] * 3) * 0.1, None),
    ("negation", lambda total, df: -math.log(float(df[1])) + -1.5, None),
    ("const first", lambda total, df: 2.0 / (df[1] + total), None),
]


@pytest.mark.parametrize("name,fn,pick", FNS, ids=[f[0] for f in FNS])
@pytest.mark.parametrize("total", [123_456_789, 1, 99_999_999_999])
def test_native_equals_python(counts, name, fn, pick, total):
    prog = lowering.numeric_program(_comp(fn, pick), 1, total)
    assert prog is not None, name
    got = plan._native_eval(_comp(fn, pick), 1, total, counts)
    assert got is not None
    assert _same_bits(got, _python(fn, counts, total, pick)), name


def test_float_broadcast_value(counts):
    fn = lambda total, df: math.log(1 + (total / df[1]))
    got = plan._native_eval(_comp(fn), 1, 1.25e8, counts)
    assert _same_bits(got, _python(fn, counts, 1.25e8))


@pytest.mark.parametrize("vals,fn", [
    ([3, 0, 5], lambda total, df: math.log(1 + (float(total) / df[1]))),        # ZeroDivisionError
    ([3, 0, 5], lambda total, df: math.log(total / df[1])),                      # ZeroDivisionError (int / int)
    ([3, -4, 5], lambda total, df: math.log(float(total) / df[1])),              # negative log argument
    ([3, 1000, 5], lambda total, df: math.log(float(df[1]) - 100.0)),            # negative log argument
    ([3, 100, 5], lambda total, df: math.log(float(df[1] - 100))),               # log(0)
    ([3, 1 << 62, 5], lambda total, df: float(df[1] * 4 + total)),               # int64 overflow (Python ints grow)
    ([3, (1 << 53) + 1, 5], lambda total, df: total / df[1]),                    # int / int beyond 2^53
])
def test_fallback_where_python_would_not_take_the_ieee_path(vals, fn):
    col = np.array(vals, dtype=np.int64)
    assert lowering.numeric_program(_comp(fn), 1, 10) is not None
    assert plan._native_eval(_comp(fn), 1, 10, col) is None


@pytest.mark.parametrize("fn", [
    lambda total, df: math.sqrt(df[1]),
    lambda total, df: math.log(df[1], 2),
    lambda total, df: df[1] ** 2 * 1.0,
    lambda total, df: df[1] // 3 * 1.0,
    lambda total, df: df[1] + total,              # an int result: Python's ints, not float64
    lambda total, df: float(df[0]),               # another field
    lambda total, df: math.log(len(df)),
    lambda total, df: abs(df[1]) * 1.0,
])
def test_outside_the_lowered_set(fn):
    assert lowering.numeric_program(_comp(fn), 1, 10) is None
    assert plan._native_eval(_comp(fn), 1, 10, np.arange(1, 5, dtype=np.int64)) is None


def test_non_number_broadcast_value():
    fn = lambda total, df: math.log(1 + (float(total) / df[1]))
    assert lowering.numeric_program(_comp(fn), 1, "10") is None
    assert lowering.numeric_program(_comp(fn), 1, True) is None
