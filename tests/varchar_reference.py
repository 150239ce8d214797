"""expr_reference.evaluate extended to VARCHAR operands, without touching it.

A VARCHAR value is bytes (None = NULL).  `=` / `<>` compare the bytes; order is Slice.compareTo (unsigned bytes, lexicographic, a proper
prefix first: S/type/AbstractVariableWidthType.java:403-410), which is Python's order on bytes.  IN, LIKE and the comparisons are NEVER_NULL
calls (NULL in, NULL out); IS [NOT] NULL and BETWEEN follow expr_reference.  LIKE is like_reference.  A string operation never raises.

Every other node is handed to expr_reference.evaluate with its operands wrapped as lazy constants: the wrapped operand is evaluated (by
this module) only when expr_reference reads it, so AND / OR short-circuit and the order of errors are exactly expr_reference's.
"""
import copy

import expr_reference as ref
import like_reference as lr
from trino_b200 import abi
from trino_b200 import operators as ops

_CMP = {abi.EX_EQ: lambda x, y: x == y, abi.EX_NE: lambda x, y: x != y, abi.EX_LT: lambda x, y: x < y,
        abi.EX_LE: lambda x, y: x <= y, abi.EX_GT: lambda x, y: x > y, abi.EX_GE: lambda x, y: x >= y}


def _bytes(v):
    return v.encode() if isinstance(v, str) else bytes(v)


class _Lazy(ops.Const):
    """an operand expr_reference reads as a constant; its value is computed when read"""

    def __init__(self, expr, row):          # noqa: super().__init__ would store `value`
        self.expr, self.row, self.vtype = expr, row, expr.vtype

    @property
    def value(self):
        return evaluate(self.expr, self.row)


def _is_string_call(e):
    return isinstance(e, ops.Call) and (e.op == abi.EX_LIKE or e.operand_vtype == abi.V_VARCHAR)


def evaluate(e, row):
    """Value of `e` on `row` (channel -> int / float / bytes / None); raises expr_reference.ExprError"""
    if isinstance(e, ops.Col) and e.vtype == abi.V_VARCHAR:
        v = row[e.channel]
        return None if v is None else _bytes(v)
    if isinstance(e, ops.Const) and not isinstance(e, _Lazy) and e.vtype == abi.V_VARCHAR:
        return _bytes(e.value)
    if isinstance(e, ops.Null) and e.vtype == abi.V_VARCHAR:
        return None
    if _is_string_call(e):
        op, args = e.op, e.args
        if op == abi.EX_IS_NULL:
            return evaluate(args[0], row) is None
        if op == abi.EX_IS_NOT_NULL:
            return evaluate(args[0], row) is not None
        if op == abi.EX_BETWEEN:
            v = evaluate(args[0], row)
            if v is None:
                return None
            lo, hi = evaluate(args[1], row), evaluate(args[2], row)
            left = None if lo is None else lo <= v
            right = None if hi is None else v <= hi
            if left is False or right is False:
                return False
            return None if left is None or right is None else True
        vals = []
        for a in args:
            v = evaluate(a, row)
            if v is None:
                return None
            vals.append(v)
        if op == abi.EX_LIKE:
            return lr.like(vals[0], e.pattern, e.escape)
        if op == abi.EX_IN:
            return vals[0] in {_bytes(c) for c in e.in_list}
        return _CMP[op](vals[0], vals[1])
    if isinstance(e, ops.Call):
        c = copy.copy(e)
        c.args = [_Lazy(a, row) for a in e.args]
        return ref.evaluate(c, row)
    return ref.evaluate(e, row)


def try_evaluate(e, row):
    """(value, error code or None)"""
    try:
        return evaluate(e, row), None
    except ref.ExprError as err:
        return None, err.code
