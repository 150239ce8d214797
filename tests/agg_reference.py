"""An exact host reference of grouped aggregation (HashAggregationOperator, SINGLE step), written from Trino's rules rather than from the
device algorithm.  Plain Python over the pages: no oracle, no floating-point accumulation.

aggregate(pages, key_channels, aggs) -> rows in group-id order: the key values, then one value per (function, input channel, mask
channel) triple (channel -1: none).

Group ids follow first appearance over the whole stream (GroupByHash.java:118-125).  A NULL key is an ordinary group.  DOUBLE keys
group by IDENTICAL (DoubleType.java:218-229: NaN = NaN, -0.0 = +0.0) and the output key is the first raw value seen for the group, bit
for bit (NaN payload and zero sign included).  A multi-column key is equal only when every field is, NULL included.
VARCHAR keys are bytes, INT128 (long DECIMAL) keys Python ints, REAL keys their float value (no rule is stated here for a REAL NaN or
-0.0 key).

A row counts for an aggregate only if its mask is non-NULL and non-zero; NULL inputs are skipped (count(*) counts the row).

  count(*), count      Python int.
  sum (integers)       Python int.  AggregateOverflow is raised when a group's final total leaves the BIGINT range: the device
                       accumulates in 128 bits and checks at output.  Known deviation, not tested: Trino's LongSumAggregation uses
                       Math.addExact and also fails on a transient overflow whose final total is in range; which partial sums occur
                       depends on the order the rows are folded in.
  sum (DOUBLE)         the exact value as a Fraction, +0.0 (Fraction(0)) when it is zero: Trino's state and the device accumulator both
                       start at +0.0, so sum({-0.0}) = +0.0.  With a non-finite input the IEEE result as a float: NaN if any input is
                       NaN or +Inf and -Inf both occur, otherwise that infinity.
  avg (DOUBLE)         the exact quotient (Fraction), or the non-finite sum as above (divided by the count: still that value).
  avg (integers)       the exact quotient (Fraction).  Trino's LongAverageAggregation sums in a double; that sum equals the exact one
                       while every partial sum stays below 2^53, and inputs for which this matters must be generated that way.
  min, max (integers)  Python int.
  min (DOUBLE)         Double.compare order (COMPARISON_UNORDERED_LAST, DoubleType.java:231-235): NaN is the largest value and
                       -0.0 < +0.0, so min({0.0, -0.0}) = -0.0 and min({1.0, NaN}) = 1.0.
  max (DOUBLE)         COMPARISON_UNORDERED_FIRST (:237-252): NaN is the smallest value, so max({1.0, NaN}) = 1.0, max({NaN}) = NaN.
  empty groups         count 0, every other function NULL (None).
"""
import math
import struct
from fractions import Fraction

import numpy as np

from trino_b200 import abi

INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1


class AggregateOverflow(ArithmeticError):
    """A BIGINT-valued sum whose final total does not fit 64 bits (NUMERIC_VALUE_OUT_OF_RANGE)"""


def _bits(x):
    return struct.unpack("<q", struct.pack("<d", x))[0]


def _float_of_bits(b):
    return struct.unpack("<d", struct.pack("<q", int(b)))[0]


def _column(page, channel):
    """(type, python values with None for NULL) of one channel; DOUBLE values are rebuilt from their bits so that payloads survive"""
    blk = page.get_block(channel).flatten()
    n = page.position_count
    nulls = blk.nulls if blk.nulls is not None else np.zeros(n, dtype=bool)
    if blk.type == abi.FLOAT64:
        vals = [_float_of_bits(b) for b in blk.values.view(np.int64).tolist()]
    elif blk.type == abi.FLOAT32:
        vals = [float(x) for x in blk.values.tolist()]
    elif blk.type in (abi.UTF8, abi.INT128):
        vals = [blk.get(i) if not nulls[i] else None for i in range(n)]
    else:
        vals = blk.values.astype(np.int64).tolist()
    return blk.type, [None if z else v for v, z in zip(vals, nulls.tolist())]


def _identical_key(t, v):
    if v is None:
        return None
    if t == abi.FLOAT64:
        if v != v:
            return "NaN"
        return 0.0 if v == 0 else v
    return v


def _min_order(x):
    """sort key of Double.compare: NaN last, -0.0 before +0.0"""
    if x != x:
        return (1, 0.0, 0)
    return (0, x, 0 if math.copysign(1.0, x) < 0 else 1)


def _max_order(x):
    """sort key of COMPARISON_UNORDERED_FIRST: NaN first, otherwise Double.compare"""
    if x != x:
        return (0, 0.0, 0)
    return (1, x, 0 if math.copysign(1.0, x) < 0 else 1)


class _DoubleSum:
    def __init__(self):
        self.finite = Fraction(0)
        self.nan = self.pos_inf = self.neg_inf = False

    def add(self, x):
        if x != x:
            self.nan = True
        elif x == math.inf:
            self.pos_inf = True
        elif x == -math.inf:
            self.neg_inf = True
        else:
            self.finite += Fraction(x)

    def value(self):
        if self.nan or (self.pos_inf and self.neg_inf):
            return math.nan
        if self.pos_inf:
            return math.inf
        if self.neg_inf:
            return -math.inf
        return self.finite


class _State:
    def __init__(self, fn, is_double):
        self.fn, self.is_double = fn, is_double
        self.count = 0
        self.total = _DoubleSum() if is_double else 0
        self.best = None

    def add(self, x):
        self.count += 1
        fn = self.fn
        if fn in (abi.AGG_SUM, abi.AGG_AVG):
            if self.is_double:
                self.total.add(x)
            else:
                self.total += x
        elif fn == abi.AGG_MIN:
            if self.best is None or (_min_order(x) < _min_order(self.best) if self.is_double else x < self.best):
                self.best = x
        elif fn == abi.AGG_MAX:
            if self.best is None or (_max_order(x) > _max_order(self.best) if self.is_double else x > self.best):
                self.best = x

    def result(self):
        fn = self.fn
        if fn in (abi.AGG_COUNT_STAR, abi.AGG_COUNT):
            return self.count
        if self.count == 0:
            return None
        if fn == abi.AGG_SUM:
            if self.is_double:
                return self.total.value()
            if not INT64_MIN <= self.total <= INT64_MAX:
                raise AggregateOverflow(self.total)
            return self.total
        if fn == abi.AGG_AVG:
            s = self.total.value() if self.is_double else Fraction(self.total)
            return s / self.count if isinstance(s, Fraction) else s
        return self.best


def aggregate(pages, key_channels, aggs):
    """rows (keys..., aggregates...) in group-id order; raises AggregateOverflow (see the module docstring)"""
    ids = {}
    keys = []
    states = []
    for page in pages:
        n = page.position_count
        if n == 0:
            continue
        kcols = [_column(page, c) for c in key_channels]
        acols = [_column(page, ch) if ch >= 0 else (None, None) for _, ch, _ in aggs]
        mcols = [_column(page, m)[1] if m >= 0 else None for _, _, m in aggs]
        for i in range(n):
            ident = tuple(_identical_key(t, vals[i]) for t, vals in kcols)
            gid = ids.get(ident)
            if gid is None:
                gid = ids[ident] = len(keys)
                keys.append(tuple(vals[i] for _, vals in kcols))
                states.append([_State(fn, acols[a][0] == abi.FLOAT64) for a, (fn, _, _) in enumerate(aggs)])
            for a, (fn, ch, _) in enumerate(aggs):
                m = mcols[a]
                if m is not None and not m[i]:          # NULL or zero mask
                    continue
                if fn == abi.AGG_COUNT_STAR:
                    states[gid][a].add(None)
                    continue
                x = acols[a][1][i]
                if x is not None:
                    states[gid][a].add(x)
    return [keys[g] + tuple(s.result() for s in states[g]) for g in range(len(keys))]
