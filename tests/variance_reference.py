"""The variance family as the reference computes it, and exactly.

- `exact(values)`: the exact (count, mean, m2) of the input doubles with Fraction, and the four results rounded once to double.  This is
  the yardstick the device is held to (1e-6 relative, and exactly 0.0 for a group of identical values).
- `welford(values)`: VarianceState.update (M/operator/aggregation/state/VarianceState.java:35-41) restated in Python floats, applied
  row by row from the empty state, and `merge` (:43-59), Chan's combination.  `results(state)` is VarianceAggregation.java:52-116.

Values are Python floats (a BIGINT argument is `float(value)`, VarianceAggregation.bigintInput :41-45); None is NULL and is skipped."""
import math
from fractions import Fraction

FUNCTIONS = ("var_samp", "var_pop", "stddev_samp", "stddev_pop")


def update(state, x):
    """VarianceState.update: count += 1; delta = x - mean; mean += delta / count; m2 += delta * (x - mean)"""
    n, mean, m2 = state
    n += 1
    delta = x - mean
    mean = mean + delta / n
    m2 = m2 + delta * (x - mean)
    return n, mean, m2


def merge(state, other):
    """VarianceState.merge as the reference writes it: a merge with count == 0 leaves the state unchanged"""
    n, mean, m2 = state
    nb, mb, qb = other
    if nb == 0:
        return state
    nt = nb + n
    new_mean = ((nb * mb) + (n * mean)) / float(nt)
    delta = mb - mean
    return nt, new_mean, m2 + qb + delta * delta * nb * n / float(nt)


def welford(values):
    state = (0, 0.0, 0.0)
    for v in values:
        if v is not None:
            state = update(state, float(v))
    return state


def results(state):
    """(var_samp, var_pop, stddev_samp, stddev_pop) of a state; None = NULL"""
    n, _, m2 = state
    samp = m2 / (n - 1) if n >= 2 else None
    pop = m2 / n if n >= 1 else None
    return (samp, pop, None if samp is None else math.sqrt(samp), None if pop is None else math.sqrt(pop))


def exact(values):
    """the four results of the exact variance of the non-NULL values (every value finite), each rounded once to double"""
    xs = [Fraction(float(v)) for v in values if v is not None]
    n = len(xs)
    if n == 0:
        return (None, None, None, None)
    mean = sum(xs) / n
    m2 = sum((x - mean) ** 2 for x in xs)
    samp = m2 / (n - 1) if n >= 2 else None
    pop = m2 / n
    return (None if samp is None else float(samp), float(pop), None if samp is None else _sqrt(samp), _sqrt(pop))


def _sqrt(q):
    """sqrt of a non-negative Fraction, correctly rounded to double"""
    if q == 0:
        return 0.0
    r = math.sqrt(float(q))
    # the float sqrt is within one ulp: keep the neighbour whose square is nearest q
    best = min((r, math.nextafter(r, math.inf), math.nextafter(r, 0.0)), key=lambda c: abs(Fraction(c) ** 2 - q))
    return best


def expected(values):
    """what the device must return: NaN where a non-finite input reaches a result, else the exact results"""
    finite = [v for v in values if v is not None]
    if any(not math.isfinite(float(v)) for v in finite):
        n = len(finite)
        nan = float("nan")
        return (nan if n >= 2 else None, nan, nan if n >= 2 else None, nan)
    return exact(values)


def close(got, want, rel=1e-6):
    """got within `rel` of want; NULL only where NULL; NaN only where NaN; an exact zero only as an exact zero"""
    if want is None or got is None:
        return got is None and want is None
    if want != want:
        return got != got
    if want == 0.0:
        return got == 0.0
    return abs(got - want) <= rel * abs(want)
