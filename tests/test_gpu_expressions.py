"""Every form of the expression evaluator against the exact reference evaluator (expr_reference.py).

Forms, each fed the same cases:
- chunked:            FilterAndProject with fixed-width pass-through channels (the two-pass form without a selection vector)
- selection_vector:   the same program with TGPU_FP_SELECTION_VECTOR=1 (filter kernel, selected positions, project kernel)
- varchar_passthrough: a VARCHAR pass-through channel, which only the selection-vector form handles
- no_filter:          a program without a filter (project kernel over every row)
- aggregation:        HashAggregationOperator with the program as its fused pre-stage, on the small-group path
test_interpreter_forms_in_child_process runs all of it again in a process started with TGPU_DISABLE_JIT=1: the interpreter kernels.

Values: BIGINT / BOOLEAN and NULL positions exact, DOUBLE bit-exact including the sign of zero (any NaN matches any NaN), row order
exact.  Errors: where the reference raises on a page, the operator must raise TrinoGpuError with that code (any of the codes when
rows raise different ones); the rows that raise nothing are then run again as their own pages and must match exactly.
"""
import math
import os
import subprocess
import sys

import numpy as np
import pytest

import expr_cases as ec
import expr_reference as ref
from helpers import oracle_agg_rows
from trino_b200 import abi
from trino_b200 import operators as ops
from trino_b200.page import Block, Page

pytestmark = pytest.mark.gpu
B, D, BOOL = abi.V_BIGINT, abi.V_DOUBLE, abi.V_BOOLEAN
FORMS = ("chunked", "selection_vector", "varchar_passthrough", "no_filter", "aggregation")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NO_JIT = bool(os.environ.get("TGPU_DISABLE_JIT"))


# ---- expected results -------------------------------------------------------------------------------------------------------
class Expected:
    """Reference results of one expression over the pool rows of a case, as arrays"""

    def __init__(self, case, expr):
        vals, errs = case.evaluate(expr)
        self.vtype = expr.vtype
        self.err = np.array([e or 0 for e in errs], dtype=np.int64)
        self.nulls = np.array([v is None for v in vals], dtype=bool)
        if self.vtype == D:
            self.values = np.array([0.0 if v is None else v for v in vals], dtype=np.float64)
        else:
            self.values = np.array([0 if v is None else int(v) for v in vals], dtype=np.int64)


def form_program(case, form):
    """(filter or None, outputs): outputs are ("pass", channel) or ("expr", expression)"""
    filt = case.filt if case.filt is not None or form in ("no_filter", "aggregation") else ops.Const(True, BOOL)
    exprs = [("expr", p) for p in case.projs]
    if form in ("chunked", "selection_vector"):
        return filt, [("pass", c) for c in case.fixed] + exprs
    if form == "varchar_passthrough":
        return filt, [("pass", case.varchar)] + exprs + [("pass", case.fixed[0])]
    if form == "no_filter":
        return None, exprs + [("pass", case.fixed[0])]
    return case.filt, [("pass", case.key)] + exprs


def page_outcome(case, filt, outputs, idx):
    """(error codes the page raises, pool rows of the page that raise nothing, pool rows selected among those)"""
    k = len(case.rows)
    if filt is not None:
        f = Expected(case, filt)
        f_err, f_true = f.err, ~f.nulls & (f.values != 0) & (f.err == 0)
    else:
        f_err, f_true = np.zeros(k, np.int64), np.ones(k, bool)
    p_err = np.zeros(k, np.int64)
    for kind, e in outputs:
        if kind == "expr":
            pe = Expected(case, e).err
            p_err = np.where(p_err != 0, p_err, pe)
    fe = f_err[idx]
    sel = f_true[idx]
    errors = set(np.unique(fe[fe != 0]).tolist())
    if not errors:
        pe = p_err[idx][sel]
        errors = set(np.unique(pe[pe != 0]).tolist())
    clean = idx[(fe == 0) & ~(sel & (p_err[idx] != 0))]
    return errors, clean, clean[f_true[clean]]


def build_program(filt, outputs):
    return ops.PageProcessorProgram(filt, [e for _, e in outputs])      # an int passes that channel through


def _concat(pages, c, n):
    if not pages:
        return None
    blocks = [p.get_block(c) for p in pages]
    if blocks[0].type == abi.UTF8:
        return [v for b in blocks for v in b.to_pylist()]
    vals = np.concatenate([b.values for b in blocks])
    nulls = np.concatenate([b.nulls if b.nulls is not None else np.zeros(len(b.values), bool) for b in blocks])
    return vals, nulls


def _fail(case, form, what, row, pool_row, want, got):
    raise AssertionError(f"{form}: {what} differs at output row {row} (pool row {pool_row}: "
                         f"{dict(enumerate(case.rows[pool_row]))})\n  want {want!r}\n  got  {got!r}\n{case.describe()}")


def compare_columns(case, form, outputs, sel_rows, pages):
    n = len(sel_rows)
    got_n = sum(p.position_count for p in pages)
    assert got_n == n, f"{form}: {got_n} rows, want {n}\n{case.describe()}"
    if n == 0:
        return
    for c, (kind, e) in enumerate(outputs):
        got = _concat(pages, c, n)
        if kind == "pass":
            col = case.columns[e]
            if col.type == abi.UTF8:
                want = [None if col.nulls[i] else col.values[i].encode() for i in sel_rows.tolist()]
                if got != want:
                    r = next(i for i, (a, b) in enumerate(zip(want, got)) if a != b)
                    _fail(case, form, f"pass-through c{e}", r, int(sel_rows[r]), want[r], got[r])
                continue
            w_vals, w_nulls, vt = col.values[sel_rows], col.nulls[sel_rows], D if col.type == abi.FLOAT64 else B
            what = f"pass-through c{e}"
        else:
            x = Expected(case, e)
            w_vals, w_nulls, vt = x.values[sel_rows], x.nulls[sel_rows], x.vtype
            what = f"projection {ec.show(e)}"
        g_vals, g_nulls = got
        bad = g_nulls != w_nulls
        if vt == D:
            wb, gb = w_vals.astype(np.float64).view(np.int64), g_vals.astype(np.float64).view(np.int64)
            bad |= ~w_nulls & (wb != gb) & ~(np.isnan(w_vals) & np.isnan(g_vals))
        else:
            bad |= ~w_nulls & (w_vals.astype(np.int64) != g_vals.astype(np.int64))
        if bad.any():
            r = int(np.argmax(bad))
            fmt = (lambda v, isn: None if isn else (float(v) if vt == D else int(v)))
            _fail(case, form, what, r, int(sel_rows[r]), fmt(w_vals[r], w_nulls[r]), fmt(g_vals[r], g_nulls[r]))


# ---- running the forms --------------------------------------------------------------------------------------------------------
def run_fp(ctx, prog, pages):
    op = ops.FilterAndProjectOperatorFactory(ctx, prog).create_operator()
    try:
        return ops.drive(op, pages)
    finally:
        op.close()


def agg_plan(case, outputs, sel_rows):
    """aggregators over the computed outputs: SUM / MIN / MAX / COUNT of BIGINT and DOUBLE, COUNT of BOOLEAN.  A BIGINT SUM whose
    running total could leave the range is left out: the reference raises at the first overflowing addition, in row order."""
    aggs = []
    for c, (kind, e) in enumerate(outputs):
        if kind != "expr":
            continue
        if e.vtype == BOOL:
            aggs.append((abi.AGG_COUNT, c, -1))
            continue
        x = Expected(case, e)
        fns = [abi.AGG_MIN, abi.AGG_MAX, abi.AGG_COUNT]
        vals = x.values[sel_rows][~x.nulls[sel_rows]]
        if e.vtype == D or sum(abs(v) for v in vals.tolist()) <= ec.I64_MAX:
            fns.insert(0, abi.AGG_SUM)
        aggs += [(fn, c, -1) for fn in fns]
    return aggs


def run_agg(ctx, prog, aggs, pages):
    fac = ops.HashAggregationOperatorFactory(ctx, [0], abi.STEP_SINGLE, [ops.Aggregator(fn, ch, m) for fn, ch, m in aggs], expected_groups=16, pre=prog)
    op = fac.create_operator()
    try:
        return [r for p in ops.drive(op, pages) for r in p.rows()]
    finally:
        op.close()


def reference_output_page(case, outputs, sel_rows):
    blocks = []
    for kind, e in outputs:
        if kind == "pass":
            col = case.columns[e]
            blocks.append(Block.tinyint(col.values[sel_rows], col.nulls[sel_rows]))
        else:
            x = Expected(case, e)
            v, n = x.values[sel_rows], x.nulls[sel_rows]
            blocks.append(Block.double(v, n) if e.vtype == D else Block.boolean(v.astype(np.int8), n) if e.vtype == BOOL else Block.bigint(v, n))
    return Page(*blocks, position_count=len(sel_rows))


def compare_agg(case, outputs, aggs, sel_rows, got):
    want = oracle_agg_rows([reference_output_page(case, outputs, sel_rows)], [0], aggs) if len(sel_rows) else []
    order = lambda r: (r[0] is not None, r[0] if r[0] is not None else 0)
    want, got = sorted(want, key=order), sorted(got, key=order)
    msg = f"aggregation over {[(fn, ch) for fn, ch, _ in aggs]}\n  want {want[:8]}\n  got  {got[:8]}\n{case.describe()}"
    assert len(want) == len(got), msg
    keys = case.columns[case.key]
    for w, g in zip(want, got):
        assert w[0] == g[0], msg
        in_group = sel_rows[(keys.nulls[sel_rows]) if w[0] is None else (~keys.nulls[sel_rows] & (keys.values[sel_rows] == w[0]))]
        for (fn, ch, _), a, b in zip(aggs, w[1:], g[1:]):
            if a is None or b is None or not isinstance(a, float):
                assert a == b, f"group {w[0]} fn {fn} c{ch}: {a!r} vs {b!r}\n" + msg
                continue
            if math.isnan(a):
                assert math.isnan(b), f"group {w[0]} fn {fn} c{ch}: {a!r} vs {b!r}\n" + msg
                continue
            if fn != abi.AGG_SUM or math.isinf(a):
                assert a == b, f"group {w[0]} fn {fn} c{ch}: {a!r} vs {b!r}\n" + msg
                continue
            # a sum in another order: within the rounding bound of the magnitudes summed (unbounded when they overflow: then skipped)
            x = Expected(case, outputs[ch][1])
            mags = np.abs(x.values[in_group][~x.nulls[in_group]])
            bound = float(np.sum(mags))
            if math.isfinite(bound):
                assert abs(a - b) <= 1e-9 * max(abs(a), bound), f"group {w[0]} sum c{ch}: {a!r} vs {b!r}\n" + msg


def check_form(ctx, case, form, monkeypatch):
    if form == "selection_vector":
        monkeypatch.setenv("TGPU_FP_SELECTION_VECTOR", "1")
    filt, outputs = form_program(case, form)
    prog = build_program(filt, outputs)
    varchar = form == "varchar_passthrough"
    clean_pages, selected = [], []
    aggs = None
    for idx in case.pages:
        errors, clean, sel = page_outcome(case, filt, outputs, idx)
        if errors:
            page = case.page(idx, varchar)
            with pytest.raises(abi.TrinoGpuError) as exc:
                if form == "aggregation":
                    run_agg(ctx, prog, agg_plan(case, outputs, sel), [page])
                else:
                    run_fp(ctx, prog, [page])
            assert exc.value.code in errors, (f"{form}: page of {len(idx)} rows raised {exc.value}, want one of "
                                              f"{sorted(ref.ERROR_NAMES[e] for e in errors)}\n{case.describe()}")
        if len(clean):
            clean_pages.append(case.page(clean, varchar))
            selected.append(sel)
    sel_rows = np.concatenate(selected) if selected else np.zeros(0, np.int64)
    if form == "aggregation":
        aggs = agg_plan(case, outputs, sel_rows)
        compare_agg(case, outputs, aggs, sel_rows, run_agg(ctx, prog, aggs, clean_pages))
    else:
        compare_columns(case, form, outputs, sel_rows, run_fp(ctx, prog, clean_pages))


_RANDOM = None


def random_cases():
    global _RANDOM
    if _RANDOM is None:
        _RANDOM = ec.random_cases()[0]
    return _RANDOM


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("index", range(16))
def test_random_programs(ctx, index, form, monkeypatch):
    check_form(ctx, random_cases()[index], form, monkeypatch)


# ---- directed cases ---------------------------------------------------------------------------------------------------------------
def _col(type_, values):
    nulls = [v is None for v in values]
    vals = [0 if v is None else v for v in values]
    return ec.Column(type_, vals, nulls)


def directed_case(name, columns, filt, projs, repeat=1):
    n = len(columns[0].values)
    pages = [np.tile(np.arange(n), repeat)]
    return ec.Case(name, columns, filt, projs, pages)


X, Y, N, V = ops.Col(0, B), ops.Col(1, B), ops.Col(2, B), ops.Col(3, B)


def _c(v, vt=B):
    return ops.Const(v, vt)


def _div_guard_columns():
    # x has zeros; y / x is only safe where x <> 0; n is NULL everywhere; v is NULL where x = 0 and below 10 elsewhere
    x = [0, 1, 2, 0, 5, -3, 0, 7]
    return [_col(abi.INT64, x), _col(abi.INT32, [10, 10, 1, 3, 20, 9, -4, 22]), _col(abi.INT64, [None] * 8),
            _col(abi.INT16, [None if xi == 0 else 4 for xi in x])]


def _guarded(case_name, filt, projs):
    return directed_case(case_name, _div_guard_columns(), filt, projs, repeat=200)


DIV = ops.Call(abi.EX_DIV, Y, X)
NONZERO = ops.Call(abi.EX_NE, X, _c(0))
IS_ZERO = ops.Call(abi.EX_EQ, X, _c(0))
DIV_GT_2 = ops.Call(abi.EX_GT, DIV, _c(2))
SHORT_CIRCUIT = {
    "and_filter": (ops.Call(abi.EX_AND, NONZERO, DIV_GT_2), [X], None),
    "and_projection": (None, [ops.Call(abi.EX_AND, NONZERO, DIV_GT_2)], None),
    "or_filter": (ops.Call(abi.EX_OR, IS_ZERO, DIV_GT_2), [Y], None),
    "or_projection": (None, [ops.Call(abi.EX_OR, IS_ZERO, DIV_GT_2)], None),
    "null_operand_skips_the_rest": (None, [ops.Call(abi.EX_ADD, N, DIV)], None),
    "null_constant_skips_the_rest": (None, [ops.Call(abi.EX_MUL, ops.Null(B), DIV)], None),
    "between_null_value": (None, [ops.Call(abi.EX_BETWEEN, V, DIV, _c(100))], None),
    "between_failing_lower_bound": (ops.Call(abi.EX_NOT, ops.Call(abi.EX_BETWEEN, ops.Call(abi.EX_ADD, X, _c(1)), _c(10), DIV)), [X], None),
    # the converse: the operand that raises is evaluated first, or nothing stops the evaluation
    "and_error_first": (ops.Call(abi.EX_AND, DIV_GT_2, NONZERO), [X], abi.ERR_DIVISION_BY_ZERO),
    "or_error_first": (None, [ops.Call(abi.EX_OR, DIV_GT_2, IS_ZERO)], abi.ERR_DIVISION_BY_ZERO),
    "null_operand_after_error": (None, [ops.Call(abi.EX_ADD, DIV, N)], abi.ERR_DIVISION_BY_ZERO),
    # NULL AND <error> raises, as in the reference's row-wise code generator (see expr_reference)
    "and_with_null_left": (ops.Call(abi.EX_AND, ops.Call(abi.EX_EQ, N, _c(1)), DIV_GT_2), [X], abi.ERR_DIVISION_BY_ZERO),
    "between_bound_evaluated": (None, [ops.Call(abi.EX_BETWEEN, X, ops.Call(abi.EX_SUB, X, _c(1)), DIV)], abi.ERR_DIVISION_BY_ZERO),
}


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("name", sorted(SHORT_CIRCUIT))
def test_short_circuit(ctx, name, form, monkeypatch):
    filt, projs, want_error = SHORT_CIRCUIT[name]
    case = _guarded(name, filt, projs)
    errors, _, _ = page_outcome(case, filt, [("expr", p) for p in projs], case.pages[0])
    assert errors == ({want_error} if want_error else set()), errors      # the reference itself, before any GPU form
    check_form(ctx, case, form, monkeypatch)


I64_MIN, I64_MAX = ec.I64_MIN, ec.I64_MAX
ARITHMETIC = {
    "min_div_minus_one": (ops.Call(abi.EX_DIV, X, Y), [I64_MIN], [-1], abi.ERR_NUMERIC_VALUE_OUT_OF_RANGE),
    "min_mod_minus_one": (ops.Call(abi.EX_MOD, X, Y), [I64_MIN, 7, -7, I64_MAX], [-1, -1, -1, -1], None),
    "mod_zero": (ops.Call(abi.EX_MOD, X, Y), [5], [0], abi.ERR_DIVISION_BY_ZERO),
    "negate_min": (ops.Call(abi.EX_NEG, X), [I64_MIN], [0], abi.ERR_NUMERIC_VALUE_OUT_OF_RANGE),
    "square_3037000499": (ops.Call(abi.EX_MUL, X, Y), [3037000499, -3037000499], [3037000499, 3037000499], None),
    "square_3037000500": (ops.Call(abi.EX_MUL, X, Y), [3037000500], [3037000500], abi.ERR_NUMERIC_VALUE_OUT_OF_RANGE),
    "min_times_minus_one": (ops.Call(abi.EX_MUL, X, Y), [I64_MIN], [-1], abi.ERR_NUMERIC_VALUE_OUT_OF_RANGE),
    "minus_one_times_min": (ops.Call(abi.EX_MUL, X, Y), [-1], [I64_MIN], abi.ERR_NUMERIC_VALUE_OUT_OF_RANGE),
    "min_times_one": (ops.Call(abi.EX_MUL, X, Y), [I64_MIN, I64_MAX], [1, 1], None),
}


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("name", sorted(ARITHMETIC))
def test_bigint_boundaries(ctx, name, form, monkeypatch):
    expr, xs, ys, want_error = ARITHMETIC[name]
    case = directed_case(name, [_col(abi.INT64, xs), _col(abi.INT64, ys)], None, [expr], repeat=3)
    errors, _, _ = page_outcome(case, None, [("expr", expr)], case.pages[0])
    assert errors == ({want_error} if want_error else set()), errors
    check_form(ctx, case, form, monkeypatch)


CAST_TABLE = [(float.fromhex(c["expr"][1][1]) if isinstance(c["expr"][1][1], str) else float(c["expr"][1][1]), c["want"])
              for c in __import__("json").load(open(os.path.join(os.path.dirname(__file__), "golden", "expressions.json")))
              if c["expr"][0] == "cast_bigint" and c["expr"][1][0] == "double"]


@pytest.mark.parametrize("form", FORMS)
def test_double_to_bigint_cast_table(ctx, form, monkeypatch):
    """TestDoubleOperators.testCastToBigint and HALF_UP rounding: the values in range in one page, every failing value in a page of its own"""
    cast = ops.Call(abi.EX_CAST_DOUBLE_TO_BIGINT, ops.Col(0, D))
    good = [(v, w) for v, w in CAST_TABLE if not isinstance(w, dict)]
    case = directed_case("cast in range", [_col(abi.FLOAT64, [v for v, _ in good])], None, [cast])
    assert Expected(case, cast).values.tolist() == [w for _, w in good]
    check_form(ctx, case, form, monkeypatch)
    for v, w in CAST_TABLE:
        if isinstance(w, dict):
            case = directed_case(f"cast {v!r}", [_col(abi.FLOAT64, [1.0, v, 2.0])], None, [cast])
            errors, _, _ = page_outcome(case, None, [("expr", cast)], case.pages[0])
            assert errors == {abi.ERR_INVALID_CAST_ARGUMENT}
            check_form(ctx, case, form, monkeypatch)


def test_narrow_integer_columns_are_sign_extended(ctx, monkeypatch):
    """TINYINT / SMALLINT / INTEGER channels enter expressions sign-extended (tg_load_i64, tg_load_elem)"""
    cols = [_col(abi.INT8, [-128, -1, 127, None]), _col(abi.INT16, [-32768, -1, 32767, 5]), _col(abi.INT32, [-2 ** 31, -1, 2 ** 31 - 1, None])]
    exprs = [ops.Call(abi.EX_ADD, ops.Col(c, B), _c(0)) for c in range(3)] + [ops.Call(abi.EX_LT, ops.Col(1, B), _c(0))]
    case = directed_case("sign extension", cols, ops.Call(abi.EX_IS_NOT_NULL, ops.Col(1, B)), exprs, repeat=300)
    assert Expected(case, exprs[1]).values.tolist() == [-32768, -1, 32767, 5]
    for form in FORMS:
        check_form(ctx, case, form, monkeypatch)


def test_interpreter_forms_in_child_process():
    """The kernels that run where NVRTC is missing (fp_filter_kernel, fp_project_kernel, the pre-stage of agg_small_kernel): no other
    test reaches them, because the choice is made once per process."""
    if NO_JIT:
        pytest.skip("already the child")
    env = dict(os.environ, TGPU_DISABLE_JIT="1")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", "-p", "no:cacheprovider", os.path.abspath(__file__)],
                       cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-6000:]
    assert " passed" in r.stdout and "1 skipped" in r.stdout, r.stdout[-2000:]


def test_jit_state_of_this_process():
    """In the child the NVRTC path must really be off (else the child test would run the specialised kernels a second time)"""
    import ctypes as C

    from q1 import q1_program
    lib = abi.load_library()
    types = (C.c_int32 * 7)(abi.INT32, abi.INT8, abi.INT8, abi.FLOAT64, abi.FLOAT64, abi.FLOAT64, abi.FLOAT64)
    n = C.c_int64()
    buf = C.create_string_buffer(1 << 16)
    st = lib.tgpu_jit_selftest_filter_project(C.byref(q1_program().struct), types, 7, 0, C.byref(n), buf, len(buf))
    assert st == (abi.ERR_NOT_SUPPORTED if NO_JIT else 0), buf.value.decode()[-500:]
