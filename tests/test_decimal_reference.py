"""decimal_reference pinned on the reference's own operator cases (tests/golden/decimal_cases.json: TestDecimalOperators restated as data,
with file:line), and on properties of its rounding and overflow rules."""
import random

import pytest

import decimal_golden as dg
import decimal_reference as dref
from trino_b200 import abi



@pytest.mark.parametrize("case", dg.CASES, ids=[c["source"] for c in dg.CASES])
def test_reference_cases(case):
    """every restated case of the reference's own tests: the value, or the error status, and the result type it asserts"""
    dec, rt = dg.plan(case)
    if "result_type" in case and rt is not None:
        assert rt == tuple(case["result_type"])
    want = dg.wanted(case)
    if "error" in case:
        with pytest.raises(dref.DecimalError) as exc:
            dg.expected(case)
        assert exc.value.status == want
    else:
        got = dg.expected(case)
        assert got == want and type(got) is type(want), (got, want)


def test_type_rules():
    # the TPC-H revenue expressions over decimal(12,2): 1 - l_discount, l_extendedprice * (1 - l_discount), * (1 + l_tax), Q6, ep / qty
    assert dref.decimal_result_type(abi.EX_SUB, (1, 0), (12, 2)) == (13, 2)
    assert dref.decimal_result_type(abi.EX_MUL, (12, 2), (13, 2)) == (26, 4)
    assert dref.decimal_result_type(abi.EX_MUL, (26, 4), (13, 2)) == (38, 6)
    assert dref.decimal_result_type(abi.EX_MUL, (12, 2), (12, 2)) == (25, 4)
    assert dref.decimal_result_type(abi.EX_DIV, (12, 2), (12, 2)) == (27, 15)
    assert dref.decimal_result_type(abi.EX_DIV, (12, 2), (12, 2), legacy=True) == (14, 2)
    assert dref.decimal_result_type(abi.EX_MUL, (12, 2), (12, 2), legacy=True) == (24, 4)


def test_type_rules_agree_with_the_library():
    """the restated rule sets against the ones PageProcessorProgram derives, over every pair of types"""
    from trino_b200.operators import decimal_result_type
    types = [(p, s) for p in range(1, 39) for s in range(0, p + 1, max(1, p // 6))]
    for legacy in (False, True):
        for op in (abi.EX_ADD, abi.EX_SUB, abi.EX_MUL, abi.EX_DIV):
            for a in types:
                for b in types[::3]:
                    assert dref.decimal_result_type(op, a, b, legacy) == decimal_result_type(op, a, b, legacy), (op, a, b, legacy)
    # legacy add / subtract
    assert dref.decimal_result_type(abi.EX_ADD, (12, 2), (10, 4), legacy=True) == (15, 4)
    assert dref.decimal_result_type(abi.EX_SUB, (38, 10), (38, 0), legacy=True) == (38, 10)
    assert dref.decimal_result_type(abi.EX_SUB, (38, 10), (38, 0)) == (38, 0)
    assert dref.decimal_result_type(abi.EX_ADD, (38, 10), (28, 10)) == (38, 10)


def test_rounding_and_wraparound():
    # HALF_UP on the magnitude, both signs
    assert dref.scale_down_round_up(15, 1) == 2 and dref.scale_down_round_up(-15, 1) == -2 and dref.scale_down_round_up(14, 1) == 1
    assert dref.decimal_to_bigint(250, (12, 2)) == 3 and dref.decimal_to_bigint(-250, (12, 2)) == -3
    assert dref.decimal_to_decimal(1250, (18, 4), (12, 2)) == 13 and dref.decimal_to_decimal(-1250, (18, 4), (12, 2)) == -13
    # unchecked short arithmetic wraps as Java's long does
    assert dref.add_sub(abi.EX_ADD, 9 * 10 ** 17, (18, 0), 9 * 10 ** 17, (18, 0), (18, 0)) == dref.wrap64(18 * 10 ** 17)
    # the short DOUBLE cast rounds twice, the long one once
    v = 2 ** 53 + 1
    assert dref.decimal_to_double(v, (18, 0)) == float(v)
    assert dref.decimal_to_double(v * 10 + 5, (19, 1)) == 9007199254740994.0
    rng = random.Random(3)
    for _ in range(2000):
        x, s = rng.randrange(-10 ** 38 + 1, 10 ** 38), rng.randrange(0, 39)
        d = dref.decimal_to_double(x, (38, s))
        assert abs(d - x / 10 ** s) <= abs(x / 10 ** s) * 2 ** -52


def test_overflow_rules():
    big = 10 ** 38 - 1
    with pytest.raises(dref.DecimalError):
        dref.mul(big, (38, 0), big, (38, 0), (38, 0))
    with pytest.raises(dref.DecimalError):
        dref.add_sub(abi.EX_ADD, big, (38, 0), 1, (1, 0), (38, 0))
    with pytest.raises(dref.DecimalError) as exc:
        dref.div(1, (12, 2), 0, (12, 2), (27, 15))
    assert exc.value.status == abi.ERR_DIVISION_BY_ZERO
    with pytest.raises(dref.DecimalError) as exc:
        dref.bigint_to_decimal(10 ** 10, (12, 2))
    assert exc.value.status == abi.ERR_INVALID_CAST_ARGUMENT
