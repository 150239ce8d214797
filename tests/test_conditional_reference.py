"""conditional_reference against the reference's written-out results (tests/golden/conditional_cases.json) and on the order of errors: a
branch, WHEN operand or argument the reference never evaluates raises nothing, and the converse of each case raises."""
import json
import os

import pytest

import conditional_reference as cr
import expr_reference as ref
from trino_b200 import abi
from trino_b200 import operators as ops

B, D, BOOL, DEC = abi.V_BIGINT, abi.V_DOUBLE, abi.V_BOOLEAN, abi.V_DECIMAL
GOLDEN = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "conditional_cases.json")))


@pytest.mark.parametrize("k", range(len(GOLDEN["cases"])))
def test_golden_case(k):
    c = GOLDEN["cases"][k]
    e = cr.from_json(c["expr"])
    got, err = cr.try_evaluate(e, [])
    assert err is None, (c["source"], c["sql"])
    want = cr.json_want(c["want"])
    assert got == want and type(got) is type(want), (c["source"], c["sql"], got, want)
    if isinstance(c["want"], list):
        assert tuple(e.dtype) == tuple(c["want"][2:]), (c["source"], e.dtype)


def test_golden_file_names_its_sources():
    assert len(GOLDEN["cases"]) >= 40
    for c in GOLDEN["cases"] + GOLDEN["skipped"]:
        assert c["source"].split(":")[0].endswith(".java") and c["source"].split(":")[1][0].isdigit()


# x = 0 on the row: y / x raises DIVISION_BY_ZERO wherever it is evaluated
X, Y, N = ops.Col(0, B), ops.Col(1, B), ops.Col(2, B)
ROW = [0, 10, None]
K = lambda v: ops.Const(v, B)
DIV = ops.Call(abi.EX_DIV, Y, X)
NONZERO, IS_ZERO = ops.Call(abi.EX_NE, X, K(0)), ops.Call(abi.EX_EQ, X, K(0))
DBZ = abi.ERR_DIVISION_BY_ZERO

ERROR_ORDER = {
    # never evaluated: no error
    "guarded_then": (ops.Case([(NONZERO, DIV)], K(0)), 0, None),
    "guarded_else": (ops.If(IS_ZERO, K(-1), DIV), -1, None),
    "guarded_later_when": (ops.Case([(IS_ZERO, K(7)), (ops.Call(abi.EX_GT, DIV, K(1)), K(8))], K(9)), 7, None),
    "if_without_else": (ops.If(NONZERO, DIV), None, None),
    "coalesce_non_null_first": (ops.Coalesce(Y, DIV), 10, None),
    "coalesce_stops_at_second": (ops.Coalesce(N, K(3), DIV), 3, None),
    "nullif_null_first": (ops.NullIf(N, DIV), None, None),
    "switch_null_value": (ops.Switch(N, [(DIV, K(1))], K(2)), 2, None),
    "switch_earlier_when_matches": (ops.Switch(X, [(K(0), K(5)), (DIV, K(6))]), 5, None),
    "null_condition_is_false": (ops.If(ops.Call(abi.EX_EQ, N, K(1)), DIV, K(4)), 4, None),
    # the converses: evaluated, so they raise
    "taken_then": (ops.Case([(IS_ZERO, DIV)], K(0)), None, DBZ),
    "taken_else": (ops.If(NONZERO, K(-1), DIV), None, DBZ),
    "condition_raises": (ops.Case([(ops.Call(abi.EX_GT, DIV, K(1)), K(8))], K(9)), None, DBZ),
    "coalesce_null_first": (ops.Coalesce(N, DIV), None, DBZ),
    "coalesce_error_first": (ops.Coalesce(DIV, Y), None, DBZ),
    "nullif_second_evaluated": (ops.NullIf(Y, DIV), None, DBZ),
    "nullif_first_raises": (ops.NullIf(DIV, N), None, DBZ),
    "switch_value_raises": (ops.Switch(DIV, [(N, K(1))], K(2)), None, DBZ),
    "switch_when_evaluated": (ops.Switch(X, [(DIV, K(1))], K(2)), None, DBZ),
    "switch_taken_result": (ops.Switch(X, [(K(0), DIV)], K(2)), None, DBZ),
}


@pytest.mark.parametrize("name", sorted(ERROR_ORDER))
def test_error_order(name):
    e, want, want_err = ERROR_ORDER[name]
    assert cr.try_evaluate(e, ROW) == (want, want_err)


def test_operands_of_every_module():
    """DECIMAL, VARCHAR and plain operands are evaluated by their own modules, inside and around the forms"""
    d = ops.Col(0, DEC, (12, 2))
    s = ops.Col(1, abi.V_VARCHAR)
    row = [1250, b"PROMO BRUSHED", 3]
    promo = ops.Call(abi.EX_LIKE, s, pattern="PROMO%")
    q14 = ops.If(promo, ops.Call(abi.EX_MUL, d, ops.Call(abi.EX_SUB, ops.Const(1, DEC, (1, 0)), ops.Const(5, DEC, (12, 2)))),
                 ops.Const(0, DEC, (25, 4)))
    assert cr.evaluate(q14, row) == 1250 * 95
    assert cr.evaluate(ops.Call(abi.EX_ADD, ops.Coalesce(ops.Null(B), ops.Col(2, B)), K(1)), row) == 4
    assert cr.evaluate(ops.Call(abi.EX_AND, ops.Const(False, BOOL), ops.Call(abi.EX_GT, ops.If(promo, DIV, K(0)), K(1))), [0, 1]) is False
    with pytest.raises(ref.ExprError):
        cr.evaluate(ops.If(ops.Const(True, BOOL), ops.Call(abi.EX_DIV, d, ops.Const(0, DEC, (12, 2))), ops.Null(DEC, (12, 2))), row)


def test_switch_compares_doubles_with_equal():
    """NaN matches no WHEN (equal(NaN, NaN) is false) and -0.0 matches 0.0"""
    v = ops.Col(0, D)
    e = ops.Switch(v, [(ops.Const(float("nan"), D), K(1)), (ops.Const(0.0, D), K(2))], K(3))
    assert cr.evaluate(e, [float("nan")]) == 3
    assert cr.evaluate(e, [-0.0]) == 2
