"""The exact aggregation reference (agg_reference.py) pinned to known answers and to the CPU oracle, without a GPU."""
import math
import struct
from fractions import Fraction

import numpy as np
import pytest

from agg_reference import INT64_MAX, INT64_MIN, AggregateOverflow, aggregate
from helpers import aggregation_known_answer_cases, hash_aggregation_operator_case, oracle_agg_rows
from trino_b200 import abi
from trino_b200.page import Block, Page

FNS = (abi.AGG_COUNT_STAR, abi.AGG_COUNT, abi.AGG_SUM, abi.AGG_AVG, abi.AGG_MIN, abi.AGG_MAX)


def _bits(x):
    return struct.unpack("<q", struct.pack("<d", x))[0]


def test_known_answer_sequences():
    # AbstractTestAggregationFunction's sequences over DOUBLE and BIGINT (see helpers.aggregation_known_answer_cases)
    aggs = [(abi.AGG_COUNT_STAR, -1, -1), (abi.AGG_COUNT, 1, -1), (abi.AGG_SUM, 1, -1), (abi.AGG_AVG, 1, -1), (abi.AGG_MIN, 1, -1), (abi.AGG_MAX, 1, -1),
            (abi.AGG_SUM, 2, -1), (abi.AGG_COUNT, 2, -1)]
    for case in aggregation_known_answer_cases():
        n = len(case["values"])
        page = Page(Block.bigint(np.zeros(n, dtype=np.int64)), Block.double(case["values"].astype(np.float64), case["nulls"]), Block.bigint(case["values"], case["nulls"]))
        [row] = aggregate([page], [0], aggs)
        conv = [None if v is None else float(v) if isinstance(v, Fraction) else v for v in row]
        assert conv == [0, case["count_star"], case["count"], case["sum_double"], case["avg_double"], case["min"], case["max"], case["sum_bigint"], case["count"]], case["name"]


def test_hash_aggregation_operator_case():
    pages, keys, aggs, expected = hash_aggregation_operator_case(5000)
    got = aggregate(pages, keys, aggs)
    assert [tuple(float(v) if isinstance(v, Fraction) else v for v in r) for r in got] == expected


def _random_pages(rng, key_types, value_type, sizes, null_frac):
    pages = []
    for n in sizes:
        keys = []
        for t in key_types:
            if t == abi.FLOAT64:
                k = rng.choice(np.array([0.0, -0.0, 1.5, -2.0, np.nan, 3.0]), n)
                keys.append(Block.double(k, rng.random(n) < 0.05))
            else:
                mk = {abi.INT64: Block.bigint, abi.INT32: Block.integer, abi.INT16: Block.smallint, abi.INT8: Block.tinyint}[t]
                keys.append(mk(rng.integers(-6, 6, n), rng.random(n) < 0.05))
        if value_type == abi.FLOAT64:
            v = Block.double(rng.integers(-(1 << 30), 1 << 30, n) / 1024.0, rng.random(n) < null_frac)
        else:
            info = np.iinfo({abi.INT64: np.int32, abi.INT32: np.int32, abi.INT16: np.int16, abi.INT8: np.int8}[value_type])
            mk = {abi.INT64: Block.bigint, abi.INT32: Block.integer, abi.INT16: Block.smallint, abi.INT8: Block.tinyint}[value_type]
            v = mk(rng.integers(info.min, info.max, n, endpoint=True), rng.random(n) < null_frac)
        mask = Block.boolean(rng.random(n) < 0.6, rng.random(n) < 0.1)
        pages.append(Page(*keys, v, mask))
    return pages


@pytest.mark.parametrize("value_type", [abi.INT64, abi.INT32, abi.INT16, abi.INT8, abi.FLOAT64])
@pytest.mark.parametrize("key_types", [(abi.INT64,), (abi.INT32, abi.INT8), (abi.FLOAT64,), (abi.INT16, abi.FLOAT64)], ids=lambda k: "-".join(map(str, k)))
def test_reference_equals_the_oracle(value_type, key_types):
    # where the oracle is defined: no mask on min / max; values k / 1024 (DOUBLE) so that the oracle's left fold is exact as well
    rng = np.random.default_rng(value_type * 31 + len(key_types) * 7 + key_types[0])
    pages = _random_pages(rng, key_types, value_type, (1, 700, 0, 333, 2000), 0.2)
    nk = len(key_types)
    v, m = nk, nk + 1
    aggs = [(f, -1 if f == abi.AGG_COUNT_STAR else v, -1) for f in FNS]
    aggs += [(f, -1 if f == abi.AGG_COUNT_STAR else v, m) for f in (abi.AGG_COUNT_STAR, abi.AGG_COUNT, abi.AGG_SUM, abi.AGG_AVG)]
    got = aggregate(pages, list(range(nk)), aggs)
    want = oracle_agg_rows(pages, list(range(nk)), aggs)
    assert len(got) == len(want)
    for g, w in zip(got, want):
        for x, y in zip(g, w):
            x = float(x) if isinstance(x, Fraction) else x
            if isinstance(x, float) or isinstance(y, float):
                assert isinstance(x, float) and isinstance(y, float), (g, w)
                assert (x != x and y != y) or _bits(x) == _bits(y), (g, w)
            else:
                assert x == y, (g, w)


def test_double_orderings_and_specials():
    nan, inf = math.nan, math.inf
    neg_nan = struct.unpack("<d", struct.pack("<Q", 0xFFF8000000000001))[0]
    groups = {1: [1.0, nan], 2: [nan], 3: [0.0, -0.0], 4: [-0.0], 5: [inf, -inf, 2.0], 6: [neg_nan, inf], 7: [-inf, 5e-324], 8: [5e-324, 5e-324]}
    keys, vals = [], []
    for k, xs in groups.items():
        keys += [k] * len(xs)
        vals += xs
    page = Page(Block.bigint(keys), Block.double(vals))
    rows = aggregate([page], [0], [(abi.AGG_SUM, 1, -1), (abi.AGG_MIN, 1, -1), (abi.AGG_MAX, 1, -1)])
    by = {r[0]: r[1:] for r in rows}
    assert math.isnan(by[1][0]) and by[1][1] == 1.0 and by[1][2] == 1.0
    assert all(math.isnan(x) for x in by[2])
    assert by[3][0] == 0 and _bits(by[3][1]) == _bits(-0.0) and _bits(by[3][2]) == _bits(0.0)
    assert by[4][0] == 0 and _bits(float(by[4][0])) == 0 and _bits(by[4][1]) == _bits(-0.0)          # sum({-0.0}) = +0.0
    assert math.isnan(by[5][0]) and by[5][1:] == (-inf, inf)
    assert by[6][1] == inf and by[6][2] == inf                       # NaN is the largest for min, the smallest for max
    assert by[7] == (-inf, -inf, 5e-324)
    assert by[8][0] == Fraction(5e-324) * 2


def test_keys_group_by_identical_and_keep_the_first_raw_value():
    nan_a = struct.unpack("<d", struct.pack("<Q", 0x7FF8000000000123))[0]
    nan_b = struct.unpack("<d", struct.pack("<Q", 0xFFF0000000000001))[0]
    page = Page(Block.double([-0.0, 0.0, nan_a, nan_b, None, 1.0]), Block.bigint([1, 2, 3, 4, 5, 6]))
    rows = aggregate([page], [0], [(abi.AGG_SUM, 1, -1)])
    assert [_bits(r[0]) if r[0] is not None else None for r in rows] == [_bits(-0.0), 0x7FF8000000000123, None, _bits(1.0)]
    assert [r[1] for r in rows] == [3, 7, 5, 6]
    # multi-column keys: equal only when every field is, NULL included
    page = Page(Block.integer([1, 1, None, None, 1]), Block.tinyint([None, None, 1, None, -1]), Block.bigint([1, 2, 4, 8, 16]))
    assert aggregate([page], [0, 1], [(abi.AGG_SUM, 2, -1)]) == [(1, None, 3), (None, 1, 4), (None, None, 8), (1, -1, 16)]


def test_bigint_sum_overflow_is_decided_by_the_final_total():
    page = Page(Block.bigint([0, 0, 1, 1]), Block.bigint([1 << 62, (1 << 62) - 1, -(1 << 62), -(1 << 62)]))
    assert aggregate([page], [0], [(abi.AGG_SUM, 1, -1)]) == [(0, INT64_MAX), (1, INT64_MIN)]
    with pytest.raises(AggregateOverflow):
        aggregate([Page(Block.bigint([0, 0]), Block.bigint([1 << 62, 1 << 62]))], [0], [(abi.AGG_SUM, 1, -1)])
    # masks: a zero or NULL mask drops the row, for min / max as well
    page = Page(Block.bigint([0, 0, 0]), Block.bigint([5, -7, 9]), Block.boolean([1, 0, None]))
    assert aggregate([page], [0], [(abi.AGG_MIN, 1, 2), (abi.AGG_MAX, 1, 2), (abi.AGG_COUNT_STAR, -1, 2)]) == [(0, 5, 5, 1)]
