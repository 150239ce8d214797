"""CPU restatement of the reference's DynamicPageFilter evaluation — TEST INFRASTRUCTURE ONLY (like everything under oracle/).

Follows M/sql/gen/columnar/DynamicPageFilter.java: one filter per column Domain in the TupleDomain's order (:124-137), applied one
after another to the surviving positions (DynamicFilterEvaluator.evaluate :160-178), each watched by the EffectiveFilterProfiler
(:181-210: once a filter has seen >= 2047 input positions and passed more than selectivityThreshold of them it is skipped from the
next page on).  A Domain contains a row's value iff the value is NULL and nulls are allowed, or it is non-NULL and in the value set
(S/predicate/Domain.java includesNullableValue).  Pinned on the cases of T/sql/gen/TestDynamicPageFilter.java (tests/test_oracle_dynamic_filter.py).

A DOUBLE range (`double=True`) compares by value, as DoubleType.compare does: bounds and column values are raw IEEE bits (the
LongArrayBlock of a DOUBLE column), decoded to float64 first, so -0.0 == 0.0 and NaN lies in no range.
"""
import numpy as np

ALL, NONE, RANGE, DISCRETE = 0, 1, 2, 3
MIN_SAMPLE_POSITIONS = 2047


def _as_double(bits):
    return np.asarray(bits, dtype=np.int64).view(np.float64)


class Domain:
    def __init__(self, channel, kind, null_allowed=False, lo=0, hi=0, values=None, double=False):
        self.channel, self.kind, self.null_allowed, self.lo, self.hi, self.double = channel, kind, null_allowed, lo, hi, double
        self.values = None if values is None else np.asarray(sorted(values), dtype=np.int64)

    def contains(self, values, nulls):
        """boolean array: which positions of a column (values, nulls) the domain lets through"""
        n = len(values)
        if self.kind == ALL:
            ok = np.ones(n, dtype=bool)
        elif self.kind == NONE:
            ok = np.zeros(n, dtype=bool)
        elif self.kind == RANGE and self.double:
            x = _as_double(values)
            ok = (x >= _as_double([self.lo])[0]) & (x <= _as_double([self.hi])[0])     # NaN compares false both ways
        elif self.kind == RANGE:
            ok = (values >= self.lo) & (values <= self.hi)          # inclusive bounds; an exclusive integer bound arrives as bound - 1
        else:
            ok = np.isin(values, self.values)
        if nulls is not None:
            ok = np.where(nulls, self.null_allowed, ok)
        return ok


class DynamicFilterEvaluator:
    def __init__(self, domains, selectivity_threshold=1.0):
        self.domains = list(domains)
        self.threshold = selectivity_threshold
        self.input_positions = [0] * len(self.domains)
        self.output_positions = [0] * len(self.domains)
        self.ineffective = [False] * len(self.domains)

    def evaluate(self, columns):
        """columns: list of (values, nulls-or-None) per channel.  Returns the selected positions (ascending)."""
        n = len(columns[0][0])
        active = np.arange(n)
        for i, d in enumerate(self.domains):
            if self.ineffective[i]:
                continue
            if len(active) == 0:
                break
            values, nulls = columns[d.channel]
            ok = d.contains(np.asarray(values)[active], None if nulls is None else np.asarray(nulls)[active])
            selected = active[ok]
            self.input_positions[i] += len(active)
            self.output_positions[i] += len(selected)
            self.ineffective[i] = self.input_positions[i] >= MIN_SAMPLE_POSITIONS and self.output_positions[i] > self.threshold * self.input_positions[i]
            active = selected
        return active
