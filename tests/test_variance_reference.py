"""tests/variance_reference.py against the reference's own variance cases (tests/golden/variance_cases.json), and the data families
tests/test_gpu_variance.py uses: on each, the reference's sequential Welford fold stays within 1e-9 of the exact variance (1e-7 on the
large-mean family), so holding the device to 1e-6 of exact is a meaningful yardstick."""
import json
import math
import os

import pytest

import variance_reference as vr
import variance_families as fam

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "variance_cases.json")
CASES = json.load(open(GOLDEN))["cases"]


@pytest.mark.parametrize("case", CASES, ids=lambda c: c["source"].split("/")[-1].split(".java")[0] + "-" + c["source"].split("(")[-1][:-1])
def test_reference_cases(case):
    i = vr.FUNCTIONS.index(case["function"])
    vals = [None if v is None else float(v) for v in case["values"]]
    assert vr.close(vr.exact(vals)[i], case["expected"], rel=0)
    assert vr.close(vr.results(vr.welford(vals))[i], case["expected"], rel=1e-15)


def test_hand_checked_values():
    # 0..4: m2 = 10; 2..5: m2 = 5; 0..9: m2 = 82.5
    assert vr.exact([0, 1, 2, 3, 4])[:2] == (2.5, 2.0)
    assert vr.exact([2, 3, 4, 5])[:2] == (5 / 3, 1.25)
    assert vr.exact(list(range(10)))[:2] == (82.5 / 9, 8.25)
    assert vr.exact([7.0]) == (None, 0.0, None, 0.0)
    assert vr.exact([None, None]) == (None, None, None, None)
    assert vr.exact([1, 2, 3, 4])[2] == math.sqrt(5 / 3)


def test_update_and_merge_restate_the_reference():
    assert vr.welford([-0.0]) == (1, 0.0, 0.0) and math.copysign(1, vr.welford([-0.0])[1]) == 1.0     # the mean of -0.0 is +0.0
    assert math.isnan(vr.welford([math.inf])[2])                                                       # var_pop({+Inf}) is NaN
    s = vr.welford([3.0, 3.0, 3.0])
    assert s == (3, 3.0, 0.0)
    assert vr.merge(s, (0, 0.0, 0.0)) is s
    a, b = vr.welford([1.0, 2.0]), vr.welford([3.0, 4.0, 5.0])
    n, mean, m2 = vr.merge(a, b)
    assert n == 5 and mean == 3.0 and m2 == 10.0


def test_naive_formula_fails_the_large_mean_family():
    """the sum-of-squares formula Σx² − (Σx)²/n loses every digit on the large-mean family: a kernel using it cannot pass"""
    vals = fam.large_mean(4096, seed=1)
    n = len(vals)
    naive = (sum(v * v for v in vals) - sum(vals) ** 2 / n) / n
    assert not vr.close(naive, vr.exact(vals)[1])


# The large-mean family's values are 1e9 + k/1024, whose spacing (1.2e-7) is a ten-millionth of their spread: every Welford delta carries
# that rounding, so the fold is held to 1e-7 there (still a tenth of the device's 1e-6), to 1e-9 everywhere else.
FOLD_REL = {"large_mean": 1e-7}


@pytest.mark.parametrize("name", sorted(fam.FAMILIES))
def test_sequential_fold_is_close_to_exact(name):
    rel = FOLD_REL.get(name, 1e-9)
    for seed in range(3):
        for vals in fam.FAMILIES[name](seed):
            want = vr.expected(vals)
            got = vr.results(vr.welford(vals))
            for g, w in zip(got, want):
                assert vr.close(g, w, rel=rel), (name, seed, g, w)
