"""The dynamic-filter oracle (oracle/dynamic_filter.py) against the reference's own cases: T/sql/gen/TestDynamicPageFilter.java."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
import dynamic_filter as df  # noqa: E402


def _cols(*columns):
    out = []
    for c in columns:
        vals = np.array([0 if v is None else v for v in c], dtype=np.int64)
        nulls = np.array([v is None for v in c])
        out.append((vals, nulls if nulls.any() else None))
    return out


def golden_cases():
    """(name, domains, threshold, pages, expected selected positions or counts per page) restated from TestDynamicPageFilter.java"""
    page_ab = _cols([1, 2, None, 5, None], [None, 102, 135, None, 3])
    seq = lambda lo, hi: (np.arange(lo, hi, dtype=np.int64), None)
    cases = [
        ("testLongBlockFilter onlyNull :137-140", [df.Domain(0, df.NONE, True)], 1.0, [page_ab], [[2, 4]]),
        ("testLongBlockFilter multipleValues :142-147", [df.Domain(0, df.DISCRETE, False, values=[2, 3, 4, 5])], 1.0, [page_ab], [[1, 3]]),
        ("testLongBlockFilter value + null :149-154", [df.Domain(0, df.DISCRETE, True, values=[1])], 1.0, [page_ab], [[0, 2, 4]]),
        ("testSelectivePageFilter :179-197", [df.Domain(1, df.DISCRETE, False, values=[-10, 5, 15, 135, 185, 250])], 1.0,
         [[seq(0, 101), seq(100, 201)], page_ab], [[35, 85], [2]]),
        ("testNonSelectivePageFilter :199-220", [df.Domain(1, df.DISCRETE, False, values=list(range(-5, 205)))], 1.0,
         [[seq(0, 101), seq(100, 201)], page_ab], [101, [1, 2, 4]]),
        ("testIneffectiveFilter :351-366", [df.Domain(0, df.RANGE, False, lo=100, hi=4999)], 0.9, [[seq(0, 1024)]] * 3, [924, 924, 1024]),
        ("testEffectiveFilter :368-381", [df.Domain(0, df.DISCRETE, False, values=[13])], 0.1, [[seq(0, 1024)]] * 5, [1] * 5),
        ("testIneffectiveFilterFirst :383-401", [df.Domain(0, df.RANGE, False, lo=100, hi=1023), df.Domain(1, df.DISCRETE, False, values=[13])], 0.9,
         [[seq(0, 1024)] * 2] * 3, [0, 0, 1]),
        ("testIneffectiveFilterLast :403-422", [df.Domain(0, df.RANGE, False, lo=50, hi=949), df.Domain(1, df.RANGE, False, lo=100, hi=1023)], 0.9,
         [[seq(0, 1024)] * 2] * 4, [850, 850, 850, 900]),
        ("testMultipleColumnsShortCircuit :424-443", [df.Domain(0, df.DISCRETE, False, values=[-10, 5, 15, 35, 50, 85, 95, 105]), df.Domain(1, df.DISCRETE, False, values=[0]),
                                                       df.Domain(2, df.RANGE, False, lo=150, hi=249)], 1.0, [[seq(0, 100)] * 3] * 5, [0] * 5),
        ("testDynamicFilterOnSubsetOfColumns :445-463", [df.Domain(1, df.DISCRETE, False, values=[-10, 5, 15, 35, 50, 85, 95, 105]), df.Domain(3, df.RANGE, False, lo=-50, hi=89)], 1.0,
         [[seq(0, 1024)] * 5] * 5, [5] * 5),
    ]
    return cases


def double_bits(values):
    """raw IEEE bits of DOUBLE values (None = NULL) as a column (values, nulls) of the oracle"""
    vals = np.array([0.0 if v is None else v for v in values], dtype=np.float64).view(np.int64)
    nulls = np.array([v is None for v in values])
    return vals, nulls if nulls.any() else None


def double_range(channel, lo, hi, null_allowed=False):
    return df.Domain(channel, df.RANGE, null_allowed, *np.array([lo, hi], dtype=np.float64).view(np.int64).tolist(), double=True)


def double_range_cases():
    """DOUBLE ranges by value (DoubleType.compare): -0.0 == 0.0, NaN lies in no range, negative bounds order by value, not by bits"""
    inf, nan = float("inf"), float("nan")
    neg_nan = -np.float64(nan)
    return [
        ("double range: -0.0 == 0.0", [double_range(0, 0.0, 1.0)], 1.0,
         [[double_bits([-0.0, 0.0, 1.0, -5e-324, 0.5, 1.0000000000000002, None])], [double_bits([0.0, -0.0, 5e-324, -5e-324])]],
         [[0, 1, 2, 4], [0, 1, 2]]),
        ("double range: [-0.0, -0.0]", [double_range(0, -0.0, -0.0, True)], 1.0, [[double_bits([0.0, -0.0, 5e-324, None])]], [[0, 1, 3]]),
        ("double range: NaN lies in no range", [double_range(0, -inf, inf)], 1.0, [[double_bits([nan, inf, -inf, 0.0, neg_nan, 1e308])]], [[1, 2, 3, 5]]),
        ("double range: negative bounds", [double_range(0, -2.5, -1.0)], 1.0, [[double_bits([-3.0, -2.5, -1.5, -1.0, -0.5, 1.0, -inf])]], [[1, 2, 3]]),
    ]


def test_oracle_reproduces_the_reference_cases():
    for name, domains, threshold, pages, expected in golden_cases() + double_range_cases():
        ev = df.DynamicFilterEvaluator(domains, threshold)
        for page, want in zip(pages, expected):
            got = ev.evaluate(page)
            if isinstance(want, int):
                assert len(got) == want, name
            else:
                assert got.tolist() == want, name
