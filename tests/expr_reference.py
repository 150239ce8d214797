"""Exact host-side evaluator of the expression trees of trino_b200.operators (Col / Const / Null / Call).

It evaluates the TREES, not the three-address code PageProcessorProgram compiles them to, so a bug in that compiler or in any GPU
form of the evaluator cannot hide in it.  Semantics are the reference's:

- BIGINT is a Python int with an explicit range check after every operation (Math.addExact / subtractExact / multiplyExact /
  negateExact, M/type/BigintOperators.java); division and modulus truncate toward zero as Java does.
- DOUBLE is a Python float: IEEE-754 binary64, round to nearest, every operation rounded on its own (no fused multiply-add).
  `%` is math.fmod, which is Java's `%` on doubles.
- CAST(DOUBLE AS BIGINT) is DoubleMath.roundToLong(x, HALF_UP) (M/type/DoubleOperators.java:159-167): the input must satisfy
  -2^63 <= x < 2^63, else INVALID_CAST_ARGUMENT; NaN and +-Infinity fail the same test.
- Boolean logic is Kleene three-valued.

Evaluation order, which decides which errors are raised:
- AND / OR evaluate left to right and stop at the first FALSE / TRUE (M/sql/gen/AndCodeGenerator.java:56-75,
  OrCodeGenerator.java:69-70).
- A call whose arguments are NEVER_NULL evaluates them in order and skips the remaining ones once one is NULL
  (M/sql/gen/BytecodeUtils.java:303-306).
- value BETWEEN min AND max: NULL when the value is NULL (min and max are not evaluated), otherwise
  `min <= value AND value <= max` with AND's short circuit (M/sql/gen/BetweenCodeGenerator.java:62-80).

A row's result is a value, NULL (None) or the first error it raises (ExprError).  A page's result follows PageProcessor: the filter
runs on every row and any error there fails the page; the projections run only on the selected rows.

In a filter, `NULL AND <error>` raises here, as the row-wise code generator does.  The reference's columnar filter path
(M/sql/gen/columnar/AndFilterEvaluator.java:71-78) evaluates the right conjunct only on the rows the left one selected, so it would
skip that error.  The two reference paths disagree on this one case; the library follows the row-wise one.
"""
import decimal
import math

from trino_b200 import abi

INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1

ERROR_NAMES = {abi.ERR_NUMERIC_VALUE_OUT_OF_RANGE: "NUMERIC_VALUE_OUT_OF_RANGE", abi.ERR_DIVISION_BY_ZERO: "DIVISION_BY_ZERO",
               abi.ERR_INVALID_CAST_ARGUMENT: "INVALID_CAST_ARGUMENT"}
ERROR_CODES = {v: k for k, v in ERROR_NAMES.items()}


class ExprError(Exception):
    def __init__(self, code):
        super().__init__(ERROR_NAMES[code])
        self.code = code


def _check(v):
    if v < INT64_MIN or v > INT64_MAX:
        raise ExprError(abi.ERR_NUMERIC_VALUE_OUT_OF_RANGE)
    return v


def _bigint(op, x, y):
    if op == abi.EX_ADD:
        return _check(x + y)
    if op == abi.EX_SUB:
        return _check(x - y)
    if op == abi.EX_MUL:
        return _check(x * y)
    if y == 0:
        raise ExprError(abi.ERR_DIVISION_BY_ZERO)
    q = abs(x) // abs(y)
    if (x < 0) != (y < 0):
        q = -q
    if op == abi.EX_DIV:
        return _check(q)          # only INT64_MIN / -1 leaves the range
    return x - y * q


def _double(op, x, y):
    if op == abi.EX_ADD:
        return x + y
    if op == abi.EX_SUB:
        return x - y
    if op == abi.EX_MUL:
        return x * y
    if op == abi.EX_DIV:
        if y == 0.0:
            if x == 0.0 or x != x:
                return math.nan
            return math.copysign(math.inf, x) * math.copysign(1.0, y)
        return x / y
    try:
        return math.fmod(x, y)
    except ValueError:            # y == 0 or x infinite: Java's % gives NaN
        return math.nan


def cast_double_to_bigint(x):
    if not (-2.0 ** 63 <= x < 2.0 ** 63):       # also false for NaN
        raise ExprError(abi.ERR_INVALID_CAST_ARGUMENT)
    return int(decimal.Decimal(x).quantize(decimal.Decimal(1), rounding=decimal.ROUND_HALF_UP))


_CMP = {abi.EX_EQ: lambda x, y: x == y, abi.EX_NE: lambda x, y: x != y, abi.EX_LT: lambda x, y: x < y,
        abi.EX_LE: lambda x, y: x <= y, abi.EX_GT: lambda x, y: x > y, abi.EX_GE: lambda x, y: x >= y}


def _typed(v, vtype):
    if v is None:
        return None
    if vtype == abi.V_DOUBLE:
        return float(v)
    if vtype == abi.V_BOOLEAN:
        return bool(v)
    return int(v)


def evaluate(e, row):
    """Value of expression `e` on `row` (a sequence indexed by channel, None = NULL): int / float / bool / None; raises ExprError."""
    from trino_b200 import operators as ops
    if isinstance(e, ops.Col):
        return _typed(row[e.channel], e.vtype)
    if isinstance(e, ops.Const):
        return _typed(e.value, e.vtype)
    if isinstance(e, ops.Null):
        return None
    op, args, vt = e.op, e.args, e.operand_vtype
    if op == abi.EX_AND or op == abi.EX_OR:
        stop = op == abi.EX_OR                     # the value that decides the result on its own
        left = evaluate(args[0], row)
        if left is stop:
            return stop
        right = evaluate(args[1], row)
        if right is stop:
            return stop
        return None if left is None or right is None else (not stop)
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
    if op == abi.EX_IS_NULL:
        return evaluate(args[0], row) is None
    if op == abi.EX_IS_NOT_NULL:
        return evaluate(args[0], row) is not None
    if op == abi.EX_MOV:
        return evaluate(args[0], row)
    # NEVER_NULL arguments: in order, stop at the first NULL
    vals = []
    for a in args:
        v = evaluate(a, row)
        if v is None:
            return None
        vals.append(v)
    x = vals[0]
    if op == abi.EX_IN:
        return any(x == _typed(c, vt) for c in e.in_list)
    if op == abi.EX_NOT:
        return not x
    if op == abi.EX_NEG:
        return -x if vt == abi.V_DOUBLE else _check(-x)
    if op == abi.EX_CAST_BIGINT_TO_DOUBLE:
        return float(x)
    if op == abi.EX_CAST_DOUBLE_TO_BIGINT:
        return cast_double_to_bigint(x)
    if op in _CMP:
        return _CMP[op](x, vals[1])
    if vt == abi.V_DOUBLE:
        return _double(op, x, vals[1])
    return _bigint(op, x, vals[1])


def try_evaluate(e, row):
    """(value, error code or None)"""
    try:
        return evaluate(e, row), None
    except ExprError as err:
        return None, err.code


def process_rows(filter_expr, projections, rows):
    """PageProcessor over `rows`: (selected row indices, projected values [projection][selected row], error codes).
    `projections`: expressions (pass-through channels are the caller's business).  When the filter raises on any row the page
    fails there: no projection runs and the errors are the filter's.  Otherwise the errors are those the projections raise on the
    selected rows.  Which row's error is reported first is not defined, so every code raised is returned."""
    selected, errors = [], set()
    for i, r in enumerate(rows):
        if filter_expr is None:
            selected.append(i)
            continue
        v, err = try_evaluate(filter_expr, r)
        if err is not None:
            errors.add(err)
        elif v is True:
            selected.append(i)
    if errors:
        return selected, None, errors
    out = []
    for p in projections:
        col = []
        for i in selected:
            v, err = try_evaluate(p, rows[i])
            if err is not None:
                errors.add(err)
            col.append(v)
        out.append(col)
    return selected, out, errors


# ---- the JSON form of expressions used by tests/golden/expressions.json --------------------------------------------------
_OPS = {"add": abi.EX_ADD, "sub": abi.EX_SUB, "mul": abi.EX_MUL, "div": abi.EX_DIV, "mod": abi.EX_MOD, "neg": abi.EX_NEG,
        "eq": abi.EX_EQ, "ne": abi.EX_NE, "lt": abi.EX_LT, "le": abi.EX_LE, "gt": abi.EX_GT, "ge": abi.EX_GE,
        "and": abi.EX_AND, "or": abi.EX_OR, "not": abi.EX_NOT, "is_null": abi.EX_IS_NULL, "is_not_null": abi.EX_IS_NOT_NULL,
        "between": abi.EX_BETWEEN, "cast_double": abi.EX_CAST_BIGINT_TO_DOUBLE, "cast_bigint": abi.EX_CAST_DOUBLE_TO_BIGINT}
_TYPES = {"bigint": abi.V_BIGINT, "double": abi.V_DOUBLE, "boolean": abi.V_BOOLEAN}


def json_double(v):
    """JSON number, or a string float.fromhex reads ("0x1.0p+63", "nan", "-inf", "-0x0p+0")"""
    return float.fromhex(v) if isinstance(v, str) else float(v)


def from_json(t):
    """["bigint", 5] / ["double", "0x1.8p+0"] / ["boolean", true] / ["null", "bigint"] / ["in", x, [values]] / [op, args...]"""
    from trino_b200 import operators as ops
    head = t[0]
    if head in _TYPES:
        vt = _TYPES[head]
        return ops.Const(json_double(t[1]) if vt == abi.V_DOUBLE else t[1], vt)
    if head == "null":
        return ops.Null(_TYPES[t[1]])
    if head == "in":
        x = from_json(t[1])
        vals = [json_double(v) if x.vtype == abi.V_DOUBLE else v for v in t[2]]
        return ops.Call(abi.EX_IN, x, in_list=vals)
    return ops.Call(_OPS[head], *[from_json(a) for a in t[1:]])
