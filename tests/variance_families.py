"""Data families for the variance family's tests.  Each family(seed) returns a list of groups, each a list of floats or None (NULL)."""
import numpy as np


def well_conditioned(n, seed):
    return list(np.random.default_rng(seed).normal(100.0, 15.0, n))


def large_mean(n, seed):
    """1e9 + k/1024: a spread of 4 around a mean of 1e9, where Σx² − (Σx)²/n cancels catastrophically"""
    return [1e9 + k / 1024 for k in np.random.default_rng(seed).integers(0, 4096, n).tolist()]


def outlier_first(n, seed):
    rng = np.random.default_rng(seed)
    return [1e7] + list(rng.normal(0.0, 1.0, n - 1))


def _with_nulls(vals, seed, frac=0.2):
    rng = np.random.default_rng(seed + 1000)
    return [None if rng.random() < frac else v for v in vals]


FAMILIES = {
    "well_conditioned": lambda s: [well_conditioned(5000, s), _with_nulls(well_conditioned(3000, s), s)],
    "large_mean": lambda s: [large_mean(5000, s), _with_nulls(large_mean(3000, s), s)],
    "outlier_first": lambda s: [outlier_first(5000, s)],
    "constant": lambda s: [[42.5] * 4000, [float(-7 - s)] * 17, _with_nulls([3.0] * 1000, s)],
    "one_row": lambda s: [[float(s) + 0.25], [None, float(s) * 3, None]],
    "all_null": lambda s: [[None] * 50, []],
    "nonfinite": lambda s: [well_conditioned(100, s) + [float("nan")], [float("inf")] + well_conditioned(50, s), [float("-inf")],
                            [float("inf"), float("-inf")], _with_nulls(well_conditioned(200, s) + [float("inf")], s)],
}
