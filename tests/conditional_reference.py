"""expr_reference.evaluate extended to the conditional special forms (If, Case, Switch, Coalesce, NullIf of trino_b200.operators) and to
DECIMAL operations, without touching it.

The forms are evaluated as written, by the reference's code generators, never through the IF / COALESCE lowering PageProcessorProgram
compiles them to:
- IF / searched CASE (IfCodeGenerator.java:47-62): the condition first; a NULL condition counts as FALSE; then only the chosen branch.
  A missing ELSE is NULL.
- simple CASE (SwitchCodeGenerator.java:77-169): the value first; a NULL value goes to ELSE without evaluating any WHEN operand;
  otherwise the WHEN operands in order, each compared with `equal` (a NULL comparison counts as false), and only the chosen result.
- COALESCE (CoalesceCodeGenerator.java:45-75): the arguments left to right, stopping at the first non-NULL one.
- NULLIF (NullIfCodeGenerator.java:62-105): a; NULL when a is NULL (b is not evaluated); then cast(a), b, cast(b) to the comparison's type,
  and `equal`: equal gives NULL, NULL or not equal gives the uncast a.
So an operand the reference skips is never evaluated here and raises nothing.

Operands go to the module that knows them: DECIMAL calls are NEVER_NULL calls over decimal_reference.apply, VARCHAR predicates go to
varchar_reference, and every other call to expr_reference with its operands wrapped as lazy constants, so AND / OR short-circuit and
the order of errors stay expr_reference's.  A DECIMAL value is its unscaled int; a DECIMAL error is raised as expr_reference.ExprError.
"""
import copy

import decimal_reference as dref
import expr_reference as ref
import varchar_reference as vr
from trino_b200 import abi
from trino_b200 import operators as ops

B, D, BOOL, DEC = abi.V_BIGINT, abi.V_DOUBLE, abi.V_BOOLEAN, abi.V_DECIMAL
_CONDITIONAL = (ops.If, ops.Case, ops.Switch, ops.Coalesce, ops.NullIf)


class _Lazy(ops.Const):
    """an operand expr_reference reads as a constant; its value is computed (by this module) when read"""

    def __init__(self, expr, row):          # noqa: super().__init__ would store `value`
        self.expr, self.row, self.vtype, self.dtype = expr, row, expr.vtype, getattr(expr, "dtype", None)

    @property
    def value(self):
        return evaluate(self.expr, self.row)


def _decimal_call(e):
    return isinstance(e, ops.Call) and (e.operand_vtype == DEC or e.op == abi.EX_CAST_TO_DECIMAL)


def _cast_value(v, from_vt, from_dt, to_vt, to_dt):
    """the value of the cast NullIf puts around a comparison operand"""
    if from_vt == to_vt and (to_vt != DEC or tuple(from_dt) == tuple(to_dt)):
        return v
    try:
        if to_vt == D:
            return float(v) if from_vt == B else dref.decimal_to_double(v, from_dt)
        if to_vt == DEC:
            return dref.bigint_to_decimal(v, to_dt) if from_vt == B else dref.decimal_to_decimal(v, from_dt, to_dt)
    except dref.DecimalError as err:
        raise ref.ExprError(err.status)
    raise ValueError("no cast from vtype %d to vtype %d" % (from_vt, to_vt))


def _evaluate_decimal(e, row):
    op, args = e.op, e.args
    if op == abi.EX_IS_NULL:
        return evaluate(args[0], row) is None
    if op == abi.EX_IS_NOT_NULL:
        return evaluate(args[0], row) is not None
    if op == abi.EX_BETWEEN:
        v = evaluate(args[0], row)
        if v is None:
            return None
        lo = evaluate(args[1], row)
        left = None if lo is None else lo <= v
        if left is False:
            return False
        hi = evaluate(args[2], row)
        right = None if hi is None else v <= hi
        if right is False:
            return False
        return None if left is None or right is None else True
    vals = []
    for a in args:       # NEVER_NULL: in order, stop at the first NULL
        v = evaluate(a, row)
        if v is None:
            return None
        vals.append(v)
    if op == abi.EX_IN:
        return vals[0] in [int(c) for c in e.in_list]
    dts = (e.operand_dtypes + [None, None, None])[:3] if e.operand_vtype == DEC else [None, None, None]
    try:
        return dref.apply(op, e.operand_vtype, (dts[0], dts[1], dts[2], e.dtype), *vals)
    except dref.DecimalError as err:
        raise ref.ExprError(err.status)


def evaluate(e, row):
    """Value of `e` on `row` (channel -> int / float / bool / bytes / None; a DECIMAL channel holds the unscaled int); raises
    expr_reference.ExprError"""
    if isinstance(e, ops.If):
        return evaluate(e.then, row) if evaluate(e.cond, row) is True else evaluate(e.else_, row)
    if isinstance(e, ops.Case):
        for cond, result in e.whens:
            if evaluate(cond, row) is True:
                return evaluate(result, row)
        return None if e.else_ is None else evaluate(e.else_, row)
    if isinstance(e, ops.Switch):
        v = evaluate(e.value, row)
        if v is not None:
            for w, result in e.whens:
                x = evaluate(w, row)
                if x is not None and x == v:
                    return evaluate(result, row)
        return None if e.else_ is None else evaluate(e.else_, row)
    if isinstance(e, ops.Coalesce):
        for a in e.args:
            v = evaluate(a, row)
            if v is not None:
                return v
        return None
    if isinstance(e, ops.NullIf):
        a = evaluate(e.a, row)
        if a is None:
            return None
        cv, cd = e.compare_as
        ca = _cast_value(a, e.a.vtype, getattr(e.a, "dtype", None), cv, cd)
        b = evaluate(e.b, row)
        if b is None:
            return a
        cb = _cast_value(b, e.b.vtype, getattr(e.b, "dtype", None), cv, cd)
        return None if ca == cb else a
    if _decimal_call(e):
        return _evaluate_decimal(e, row)
    if vr._is_string_call(e):
        return vr.evaluate(e, row)          # VARCHAR operands hold no conditional
    if isinstance(e, ops.Call):
        c = copy.copy(e)
        c.args = [_Lazy(a, row) for a in e.args]
        return ref.evaluate(c, row)
    if isinstance(e, ops.Const) and e.vtype == DEC:
        return int(e.value)
    return vr.evaluate(e, row)


def try_evaluate(e, row):
    """(value, error code or None)"""
    try:
        return evaluate(e, row), None
    except ref.ExprError as err:
        return None, err.code


# ---- the JSON form of tests/golden/conditional_cases.json ------------------------------------------------------------------------
_TYPES = {"bigint": B, "double": D, "boolean": BOOL}


def from_json(t):
    """see the "about" entry of tests/golden/conditional_cases.json"""
    head = t[0]
    if head == "decimal":
        return ops.Const(int(t[1]), DEC, (t[2], t[3]))
    if head == "null_decimal":
        return ops.Null(DEC, (t[1], t[2]))
    if head == "if":
        return ops.If(*[from_json(a) for a in t[1:]])
    if head == "case":
        return ops.Case([(from_json(c), from_json(r)) for c, r in t[1]], from_json(t[2]) if len(t) > 2 else None)
    if head == "switch":
        return ops.Switch(from_json(t[1]), [(from_json(w), from_json(r)) for w, r in t[2]], from_json(t[3]) if len(t) > 3 else None)
    if head == "coalesce":
        return ops.Coalesce(*[from_json(a) for a in t[1:]])
    if head == "nullif":
        cmp = None
        if len(t) > 3:
            cmp = (D, None) if t[3][0] == "double" else (DEC, (t[3][1], t[3][2]))
        return ops.NullIf(from_json(t[1]), from_json(t[2]), compare_as=cmp)
    if head in _TYPES or head in ("null", "in") or head in ref._OPS:
        if head in ("null", "in") or head in _TYPES:
            return ref.from_json(t)
        return ops.Call(ref._OPS[head], *[from_json(a) for a in t[1:]])
    raise ValueError(head)


def json_want(w):
    """the 'want' of a golden case as a value of evaluate"""
    if isinstance(w, list) and w and w[0] == "decimal":
        return int(w[1])
    return w
