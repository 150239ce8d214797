"""The cases of tests/golden/decimal_cases.json as the planner would hand them to the library: integer operands of a decimal operation are
coerced to DECIMAL(19, 0) (BIGINT) or DECIMAL(10, 0) (INTEGER), compared operands to their common super type, and the result type of
+ - * / follows the default rules.  expected() evaluates a case with decimal_reference; expression() builds it for the device."""
import json
import os

import decimal_reference as dref
from trino_b200 import abi
from trino_b200 import operators as ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = json.load(open(os.path.join(ROOT, "tests", "golden", "decimal_cases.json")))["cases"]
ARITH = {"add": abi.EX_ADD, "subtract": abi.EX_SUB, "multiply": abi.EX_MUL, "divide": abi.EX_DIV}
CMP = {"eq": abi.EX_EQ, "ne": abi.EX_NE, "lt": abi.EX_LT, "le": abi.EX_LE, "gt": abi.EX_GT, "ge": abi.EX_GE}
INT_AS_DECIMAL = {"bigint": (19, 0), "integer": (10, 0)}
ERRORS = {"NUMERIC_VALUE_OUT_OF_RANGE": abi.ERR_NUMERIC_VALUE_OUT_OF_RANGE, "DIVISION_BY_ZERO": abi.ERR_DIVISION_BY_ZERO,
          "INVALID_CAST_ARGUMENT": abi.ERR_INVALID_CAST_ARGUMENT}


def arg_type(a):
    return tuple(a["type"]) if isinstance(a["type"], list) else a["type"]


def _super(types):
    whole = max(p - s for p, s in types)
    scale = max(s for _, s in types)
    return min(38, whole + scale), scale


def plan(case):
    """(operand decimal types after coercion, result type or None)"""
    op = case["op"]
    raw = [arg_type(a) for a in case["args"]]
    dec = [INT_AS_DECIMAL[t] if isinstance(t, str) else t for t in raw]
    if op in ARITH:
        return dec, dref.decimal_result_type(ARITH[op], dec[0], dec[1])
    if op == "negate":
        return dec, dec[0]
    if op in CMP or op == "between":
        t = _super(dec)
        return [t] * len(dec), None
    return raw, tuple(case["target"]) if isinstance(case["target"], list) else None


def expected(case):
    """the reference's value (int, bool, float or None) or DecimalError"""
    dec, rt = plan(case)
    op = case["op"]
    vals = [None if a["value"] is None else int(a["value"]) for a in case["args"]]
    if op == "cast":
        v, t = vals[0], arg_type(case["args"][0])
        if v is None:
            return None
        if case["target"] == "BIGINT":
            return dref.decimal_to_bigint(v, t)
        if case["target"] == "DOUBLE":
            return dref.decimal_to_double(v, t)
        return dref.bigint_to_decimal(v, rt) if isinstance(t, str) else dref.decimal_to_decimal(v, t, rt)
    coerced = []
    for v, a, t in zip(vals, case["args"], dec):
        src = arg_type(a)
        if v is None:
            coerced.append(None)
        elif isinstance(src, str):
            coerced.append(dref.bigint_to_decimal(v, t))
        else:
            coerced.append(dref.decimal_to_decimal(v, src, t) if src != t else v)
    if op == "between":
        a, b, c = coerced
        if a is None:
            return None
        f1, f2 = b is not None and a < b, c is not None and a > c
        return False if f1 or f2 else (None if b is None or c is None else True)
    if any(v is None for v in coerced):
        return None
    if op in ARITH:
        return dref.apply(ARITH[op], abi.V_DECIMAL, (dec[0], dec[1], None, rt), *coerced)
    if op == "negate":
        return dref.neg(coerced[0], dec[0])
    return dref.compare(CMP[op], *coerced)


def wanted(case):
    """the value the reference's test asserts (int, bool, float or None), or the error status"""
    if "error" in case:
        return ERRORS[case["error"]]
    if "result_double" in case:
        return float(case["result_double"])
    r = case["result"]
    return r if r is None or isinstance(r, bool) else int(r)


def expression(case, operands):
    """the case as an expression over `operands` (one expression per argument, of the argument's own type)"""
    dec, rt = plan(case)
    op = case["op"]
    if op == "cast":
        a = operands[0]
        if case["target"] == "BIGINT":
            return ops.Call(abi.EX_CAST_DECIMAL_TO_BIGINT, a)
        if case["target"] == "DOUBLE":
            return ops.Call(abi.EX_CAST_DECIMAL_TO_DOUBLE, a)
        return ops.Call(abi.EX_CAST_TO_DECIMAL, a, result_dtype=rt)
    args = []
    for e, a, t in zip(operands, case["args"], dec):
        if arg_type(a) != t:
            e = ops.Call(abi.EX_CAST_TO_DECIMAL, e, result_dtype=t)
        args.append(e)
    if op in ARITH:
        return ops.Call(ARITH[op], *args)
    if op == "negate":
        return ops.Call(abi.EX_NEG, *args)
    if op == "between":
        return ops.Call(abi.EX_BETWEEN, *args)
    return ops.Call(CMP[op], *args)


def operand_expr(a, k, as_column):
    """argument a as channel k (as_column) or as a constant / NULL"""
    t = arg_type(a)
    vt, dt = (abi.V_BIGINT, None) if isinstance(t, str) else (abi.V_DECIMAL, t)
    if as_column:
        return ops.Col(k, vt, dt)
    if a["value"] is None:
        return ops.Null(vt, dt)
    return ops.Const(int(a["value"]), vt, dt)
