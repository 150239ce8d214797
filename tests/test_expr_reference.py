"""The exact reference evaluator (expr_reference.py) against known answers of the reference's own tests, and the coverage of the
seeded program generator (expr_cases.py).  Host only."""
import json
import math
import os

import pytest

import expr_cases as ec
import expr_reference as ref
from helpers import GOLDEN
from trino_b200 import abi
from trino_b200 import operators as ops

with open(os.path.join(GOLDEN, "expressions.json")) as _f:
    KNOWN = json.load(_f)


def _want(case, result_vtype):
    w = case["want"]
    if isinstance(w, dict):
        return w
    if w is None or result_vtype != abi.V_DOUBLE:
        return w
    return ref.json_double(w)


@pytest.mark.parametrize("i", range(len(KNOWN)), ids=[f"{c['source']}:{json.dumps(c['expr'])}" for c in KNOWN])
def test_known_answers(i):
    case = KNOWN[i]
    expr = ref.from_json(case["expr"])
    want = _want(case, expr.vtype)
    value, err = ref.try_evaluate(expr, ())
    if isinstance(want, dict):
        assert err is not None and ref.ERROR_NAMES[err] == want["error"], (value, err)
        return
    assert err is None, ref.ERROR_NAMES[err]
    if isinstance(want, float):
        assert isinstance(value, float)
        assert (math.isnan(want) and math.isnan(value)) or (value == want and math.copysign(1, value) == math.copysign(1, want)), (value, want)
    else:
        assert value == want and type(value) is type(want), (value, want)


def test_page_semantics_follow_page_processor():
    """filter errors count on every row and stop the page; projection errors only on the selected rows"""
    x, y = ops.Col(0, abi.V_BIGINT), ops.Col(1, abi.V_BIGINT)
    div = ops.Call(abi.EX_DIV, y, x)
    rows = [(0, 5), (1, 5), (2, 5)]
    keep_nonzero = ops.Call(abi.EX_NE, x, ops.Const(0, abi.V_BIGINT))
    sel, out, errors = ref.process_rows(keep_nonzero, [div], rows)
    assert sel == [1, 2] and out == [[5, 2]] and not errors
    sel, out, errors = ref.process_rows(ops.Call(abi.EX_GT, div, ops.Const(0, abi.V_BIGINT)), [x], rows)
    assert out is None and errors == {abi.ERR_DIVISION_BY_ZERO}
    sel, out, errors = ref.process_rows(None, [div], rows)
    assert errors == {abi.ERR_DIVISION_BY_ZERO} and out == [[None, 5, 2]]


def test_generator_covers_every_op_and_operand_type():
    cases, seen = ec.random_cases()
    assert set(seen) >= ec.OP_PAIRS, sorted(ec.OP_PAIRS - set(seen))
    for case in cases:
        prog = ops.PageProcessorProgram(case.filt, case.projs)
        assert len(prog.insns) <= 64
        assert max(d for _, _, d, *_ in prog.insns) < 8
    # the compiled programs, not only the trees, hold every pair (a MOV may also come from the compiler)
    compiled = {(op, vt) for case in cases for op, vt, *_ in ops.PageProcessorProgram(case.filt, case.projs).insns}
    assert compiled >= ec.OP_PAIRS, sorted(ec.OP_PAIRS - compiled)


def test_generator_pages_cover_sizes_encodings_and_null_modes():
    cases, _ = ec.random_cases()
    sizes = {len(p) for c in cases for p in c.pages}
    assert sizes >= set(ec.SIZES) | {ec.BIG_PAGE}
    enc = {(c.type, col_enc) for case in cases for c, col_enc in ((c, c.encoding) for c in case.columns[:case.key])}
    assert {e for _, e in enc} == {"flat", "dict", "rle"}
    modes = {ec._null_mode(c) for case in cases for c in case.columns[:case.key]}
    assert modes == {"non-null", "nullable", "all-null"}
    filters = {case.name.rsplit("-", 1)[1] for case in cases}
    assert filters == {"some", "none", "all"}


def test_generated_cases_hit_values_nulls_and_errors():
    """the random cases are not all error pages: most produce values, some raise each error code"""
    cases, _ = ec.random_cases()
    codes, valued = set(), 0
    for case in cases:
        for p in case.projs:
            vals, errs = case.evaluate(p)
            codes |= {e for e in errs if e}
            valued += sum(1 for v, e in zip(vals, errs) if e is None and v is not None) > len(vals) // 4
    assert codes == set(ref.ERROR_NAMES)
    assert valued >= len(cases)
