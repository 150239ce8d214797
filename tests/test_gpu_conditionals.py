"""IF, CASE, the simple CASE, COALESCE and NULLIF on the GPU against the exact reference (conditional_reference.py).

- Seeded random programs (ConditionalProgramGen: conditional nodes at any depth, as conditions and inside arithmetic) run through the
  five forms of test_gpu_expressions: chunked, selection vector, VARCHAR pass-through, no filter and the fused small-path aggregation,
  at page sizes of 1 row, a tile +- 1 and several chunks, over flat, dictionary and RLE blocks.
- Directed: the order of errors (a branch, WHEN operand or argument the reference skips raises nothing; the converses raise); short and
  long DECIMAL branches, COALESCE and NULLIF; VARCHAR conditions (=, IN, LIKE) with numeric results; count(IF(c, x, NULL)) and
  count(COALESCE(x, y)) through path S, path G and the global aggregation (the never-NULL rule that lets count(x) alias count(*));
  Q12- and Q14-shaped FilterAndProject -> HashAggregationOperator pipelines.
test_interpreter_forms_in_child_process runs the file again with TGPU_DISABLE_JIT=1.  Values, NULLs and row order are exact, DOUBLE bit for
bit; a page that raises must fail with one of the reference's codes."""
import math
import os
import random
import struct
import subprocess
import sys

import numpy as np
import pytest

import agg_reference
import conditional_reference as cr
import expr_cases as ec
import test_conditional_reference as tcr
from test_gpu_expressions import FORMS, _div_guard_columns, check_form, page_outcome
from trino_b200 import abi
from trino_b200 import operators as ops
from trino_b200.page import Block, DictionaryBlock, Page, RunLengthEncodedBlock

pytestmark = pytest.mark.gpu
B, D, BOOL, S, DEC = abi.V_BIGINT, abi.V_DOUBLE, abi.V_BOOLEAN, abi.V_VARCHAR, abi.V_DECIMAL
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NO_JIT = bool(os.environ.get("TGPU_DISABLE_JIT"))
call = ops.Call


# ---- random programs ------------------------------------------------------------------------------------------------------------------
class ConditionalProgramGen(ec.ProgramGen):
    """ec.ProgramGen whose trees also hold IF, CASE, the simple CASE, COALESCE and NULLIF of every numeric and BOOLEAN type, at any
    depth (so as conditions, WHEN operands and arithmetic operands too)"""

    def expr(self, vt, depth):
        r = self.rng
        if depth <= 0 or r.random() >= 0.35:
            return super().expr(vt, depth)
        kind = ["if", "case", "switch", "coalesce", "nullif"][int(r.integers(0, 5))]
        self.seen[(kind, vt)] = self.seen.get((kind, vt), 0) + 1
        sub = lambda t: self.expr(t, depth - 1)
        if kind == "if":
            return ops.If(sub(BOOL), sub(vt), sub(vt) if r.random() < 0.7 else None)
        if kind == "case":
            whens = [(sub(BOOL), sub(vt)) for _ in range(int(r.integers(1, 3)))]
            return ops.Case(whens, sub(vt) if r.random() < 0.7 else None)
        if kind == "switch":
            wt = [B, D, BOOL][int(r.integers(0, 3))]
            whens = [(self.leaf(wt) if r.random() < 0.6 else sub(wt), sub(vt)) for _ in range(int(r.integers(1, 3)))]
            return ops.Switch(sub(wt), whens, sub(vt) if r.random() < 0.7 else None)
        if kind == "coalesce":
            return ops.Coalesce(*[sub(vt) for _ in range(int(r.integers(2, 4)))])
        if vt == D and r.random() < 0.4:
            return ops.NullIf(sub(D), sub(B), compare_as=D)
        return ops.NullIf(sub(vt), sub(vt))


_EC_SHOW = ec.show
_OPNAME = {abi.EX_ADD: "+", abi.EX_SUB: "-", abi.EX_MUL: "*", abi.EX_DIV: "/", abi.EX_MOD: "%", abi.EX_EQ: "=", abi.EX_NE: "<>",
           abi.EX_LT: "<", abi.EX_LE: "<=", abi.EX_GT: ">", abi.EX_GE: ">=", abi.EX_AND: "AND", abi.EX_OR: "OR"}


def show(e):
    """ec.show extended to the conditional forms"""
    if isinstance(e, ops.If):
        return f"IF({show(e.cond)}, {show(e.then)}, {show(e.else_)})"
    if isinstance(e, ops.Case):
        return "CASE " + " ".join(f"WHEN {show(c)} THEN {show(v)}" for c, v in e.whens) + (f" ELSE {show(e.else_)}" if e.else_ is not None else "") + " END"
    if isinstance(e, ops.Switch):
        return (f"CASE {show(e.value)} " + " ".join(f"WHEN {show(c)} THEN {show(v)}" for c, v in e.whens)
                + (f" ELSE {show(e.else_)}" if e.else_ is not None else "") + " END")
    if isinstance(e, ops.Coalesce):
        return "COALESCE(" + ", ".join(show(a) for a in e.args) + ")"
    if isinstance(e, ops.NullIf):
        return f"NULLIF({show(e.a)}, {show(e.b)})"
    if isinstance(e, ops.Call):
        a = [show(x) for x in e.args]
        if e.op in _OPNAME:
            return f"({a[0]} {_OPNAME[e.op]} {a[1]})"
        return f"op{e.op}({', '.join(a)})"
    return _EC_SHOW(e)


class CondCase(ec.Case):
    """an ec.Case evaluated by conditional_reference"""

    def evaluate(self, expr):
        key = id(expr)
        if key not in self._memo:
            vals, errs = [], []
            for r in self.rows:
                v, e = cr.try_evaluate(expr, r)
                vals.append(v)
                errs.append(e)
            self._memo[key] = (expr, vals, errs)
        return self._memo[key][1:]

    def describe(self):
        s = f"case {self.name}\n  filter: {show(self.filt) if self.filt is not None else '-'}\n"
        return s + "".join(f"  projection {i}: {show(p)}\n" for i, p in enumerate(self.projs)) + "  page sizes: " + ", ".join(str(len(p)) for p in self.pages)


def random_case(seed, seen, sizes=None):
    rng = np.random.default_rng(seed)
    k = ec.POOL
    columns = []
    for t in ec.RANDOM_TYPES:
        null_mode = rng.choice(["none", "some", "all"], p=[0.45, 0.45, 0.1])
        enc = rng.choice(["flat", "dict", "rle"], p=[0.6, 0.3, 0.1])
        columns.append(ec.random_column(rng, t, k, null_mode, enc))
    by_vt = {B: [], D: [], BOOL: []}
    for c, t in enumerate(ec.RANDOM_TYPES):
        by_vt[ec.VTYPE_OF[t]].append(c)
    gen = ConditionalProgramGen(rng, by_vt, seen, [c for c, t in enumerate(ec.RANDOM_TYPES) if t == abi.INT64])
    filt, projs = gen.program(max_depth=4)
    sizes = sizes or [ec.SIZES[seed % len(ec.SIZES)], ec.SIZES[(seed + 3) % len(ec.SIZES)]]
    pages = [rng.integers(0, k, n) for n in sizes]
    return CondCase(f"conditional-{seed}", columns, filt, projs, pages, seed=seed)


_RANDOM = None


def random_cases():
    global _RANDOM
    if _RANDOM is None:
        seen = {}
        _RANDOM = [random_case(7000 + s, seen, [ec.BIG_PAGE, 1023] if s == 3 else None) for s in range(12)]
    return _RANDOM


@pytest.fixture
def conditional_show(monkeypatch):
    monkeypatch.setattr(ec, "show", show)      # check_form names a failing projection with ec.show


def test_random_programs_hold_every_form():
    seen = {}
    for s in range(12):
        random_case(7000 + s, seen)
    for kind in ("if", "case", "switch", "coalesce", "nullif"):
        assert any(k == kind for k, _ in seen), kind


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("index", range(12))
def test_random_programs(ctx, index, form, monkeypatch, conditional_show):
    check_form(ctx, random_cases()[index], form, monkeypatch)


# ---- directed: the order of errors ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("name", sorted(tcr.ERROR_ORDER))
def test_error_order(ctx, name, form, monkeypatch, conditional_show):
    """x holds zeros, y / x raises there: a skipped branch raises nothing, an evaluated one raises DIVISION_BY_ZERO"""
    e, _, want_error = tcr.ERROR_ORDER[name]
    for filt, projs in ((None, [e]), (call(abi.EX_IS_NOT_NULL, e), [ops.Col(0, B)])):
        case = CondCase(name, _div_guard_columns(), filt, projs, [np.tile(np.arange(8), 200)])
        errors, _, _ = page_outcome(case, filt, [("expr", p) for p in projs], case.pages[0])
        assert errors == ({want_error} if want_error else set()), errors
        check_form(ctx, case, form, monkeypatch)


# ---- directed: pages built by hand ------------------------------------------------------------------------------------------------------
def _fp(ctx, monkeypatch, prog, pages, form):
    if form == "selection_vector":
        monkeypatch.setenv("TGPU_FP_SELECTION_VECTOR", "1")
    else:
        monkeypatch.delenv("TGPU_FP_SELECTION_VECTOR", raising=False)
    op = ops.FilterAndProjectOperatorFactory(ctx, prog).create_operator()
    try:
        return ops.drive(op, pages)
    finally:
        op.close()


def _bits(v):
    return struct.unpack("<q", struct.pack("<d", v))[0]


def _same(g, w, vt):
    if w is None or g is None:
        return g is None and w is None
    if vt == D:
        return (math.isnan(g) and math.isnan(w)) or _bits(g) == _bits(w)
    if vt == BOOL:
        return bool(g) == w
    return g == w


def _check_rows(ctx, monkeypatch, rows, page, filt, projs, forms=("chunked", "selection_vector", "no_filter")):
    """every form of FilterAndProject over one page against the reference row by row; a page that raises fails with one of its codes"""
    for form in forms:
        f = filt if form != "no_filter" else None
        if f is None and form != "no_filter":
            f = ops.Const(True, BOOL)
        sel, errors = [], set()
        for i, r in enumerate(rows):
            v, e = (True, None) if f is None else cr.try_evaluate(f, r)
            if e is not None:
                errors.add(e)
            elif v is True:
                sel.append(i)
        want = []
        if not errors:
            for p in projs:
                col = []
                for i in sel:
                    v, e = cr.try_evaluate(p, rows[i])
                    if e is not None:
                        errors.add(e)
                    col.append(v)
                want.append(col)
        prog = ops.PageProcessorProgram(f, projs)
        if errors:
            with pytest.raises(abi.TrinoGpuError) as exc:
                _fp(ctx, monkeypatch, prog, [page], form)
            assert exc.value.code in errors, (form, exc.value, errors)
            continue
        out = _fp(ctx, monkeypatch, prog, [page], form)
        for k, p in enumerate(projs):
            got = [v for o in out for v in o.get_block(k).to_pylist()]
            assert len(got) == len(sel), (form, k)
            for j, (g, w) in enumerate(zip(got, want[k])):
                assert _same(g, w, p.vtype), (form, show(p), "row", sel[j], rows[sel[j]], g, w)


def _dec_values(rng, p, n, nulls=0.1):
    m = 10 ** p - 1
    edges = [0, 1, -1, m, -m, 5, -5, 10 ** (p // 2)]
    r = random.Random(int(rng.integers(0, 1 << 30)))
    return [None if r.random() < nulls else (edges[i] if i < len(edges) else r.randint(-m, m)) for i in range(n)]


def _dec_block(p, values):
    if p <= 18:
        return Block.bigint([0 if v is None else v for v in values], [v is None for v in values])
    return Block.int128(values)


def test_decimal_branches(ctx, monkeypatch):
    """short (12, 2) and long (38, 6) branches of IF, CASE, COALESCE and NULLIF, against decimal_reference; a guarded DECIMAL division"""
    rng = np.random.default_rng(11)
    n = 700
    x = [None if rng.random() < 0.1 else int(rng.integers(-3, 4)) for _ in range(n)]
    a, b = _dec_values(rng, 12, n), _dec_values(rng, 12, n)
    c, d = _dec_values(rng, 38, n), _dec_values(rng, 38, n)
    b[0] = 0
    rows = list(zip(x, a, b, c, d))
    page = Page(Block.bigint([0 if v is None else v for v in x], [v is None for v in x]), _dec_block(12, a), _dec_block(12, b),
                _dec_block(38, c), _dec_block(38, d))
    X, A, Bc, Cc, Dc = ops.Col(0, B), ops.Col(1, DEC, (12, 2)), ops.Col(2, DEC, (12, 2)), ops.Col(3, DEC, (38, 6)), ops.Col(4, DEC, (38, 6))
    zero_s, zero_l = ops.Const(0, DEC, (12, 2)), ops.Const(0, DEC, (38, 6))
    pos = call(abi.EX_GT, X, ops.Const(0, B))
    quotient = call(abi.EX_DIV, A, Bc)
    projs = [ops.If(pos, A, Bc), ops.Coalesce(A, Bc, zero_s), ops.NullIf(A, Bc), ops.If(pos, Cc, Dc), ops.Coalesce(Cc, Dc),
             ops.Case([(pos, Cc), (call(abi.EX_LT, X, ops.Const(0, B)), ops.Const(-(10 ** 37), DEC, (38, 6)))]), ops.NullIf(Cc, zero_l),
             ops.If(call(abi.EX_NE, Bc, zero_s), quotient, ops.Const(0, DEC, quotient.dtype)),
             ops.Switch(A, [(zero_s, Cc), (Bc, Dc)], zero_l),
             call(abi.EX_GT, ops.Coalesce(Cc, Dc), zero_l)]
    for k in range(0, len(projs), 4):     # at most 8 temps: projection temps stay live to the end
        _check_rows(ctx, monkeypatch, rows, page, call(abi.EX_IS_NOT_NULL, ops.Coalesce(A, Bc)), projs[k:k + 4])
    # the converse: the division is the branch taken where b = 0, and raises
    _check_rows(ctx, monkeypatch, rows, page, None, [ops.If(call(abi.EX_EQ, Bc, zero_s), quotient, ops.Const(0, DEC, quotient.dtype))],
                forms=("no_filter",))


def test_boolean_channel_condition_of_decimal_if(ctx, monkeypatch):
    """a BOOLEAN channel (TGPU_INT8) as the condition of a short and a long DECIMAL IF, CASE and COALESCE-of-IF: the condition is a plain
    word, not a decimal operand, so create and add_input accept the page and every form matches the reference (the child run of this
    file repeats it through the interpreter kernels)"""
    rng = np.random.default_rng(16)
    n = 3000
    p = [None if rng.random() < 0.15 else bool(rng.integers(0, 2)) for _ in range(n)]
    a, c = _dec_values(rng, 12, n), _dec_values(rng, 38, n)
    rows = list(zip(p, a, c))
    page = Page(Block.boolean([0 if v is None else int(v) for v in p], [v is None for v in p]), _dec_block(12, a), _dec_block(38, c))
    P, A, Cc = ops.Col(0, BOOL), ops.Col(1, DEC, (12, 2)), ops.Col(2, DEC, (38, 6))
    projs = [ops.If(P, A, ops.Const(0, DEC, (12, 2))), ops.If(P, Cc), ops.Case([(P, Cc)], ops.Const(-1, DEC, (38, 6))),
             ops.Coalesce(ops.If(P, A), ops.Const(7, DEC, (12, 2)))]
    _check_rows(ctx, monkeypatch, rows, page, ops.Call(abi.EX_IS_NOT_NULL, ops.If(P, A, ops.Null(DEC, (12, 2)))), projs[:2])
    _check_rows(ctx, monkeypatch, rows, page, P, projs[2:])


@pytest.mark.parametrize("vt", ["bigint", "decimal"])
def test_if_condition_channel_must_be_boolean(ctx, monkeypatch, vt):
    """a DOUBLE or BIGINT channel named as IF's condition is refused at add_input instead of being read as raw bits"""
    r = ops.Col(1, DEC, (12, 2)) if vt == "decimal" else ops.Col(1, B)
    prog = ops.PageProcessorProgram(None, [ops.If(ops.Col(0, BOOL), r, ops.Null(r.vtype, getattr(r, "dtype", None)))])
    for cond in (Block.double([-0.0, 1.0]), Block.bigint([0, 1])):
        with pytest.raises(abi.TrinoGpuError) as exc:
            _fp(ctx, monkeypatch, prog, [Page(cond, Block.bigint([5, 6]))], "no_filter")
        assert exc.value.code == abi.ERR_INVALID_ARGUMENT
    out = _fp(ctx, monkeypatch, prog, [Page(Block.boolean([0, 1]), Block.bigint([5, 6]))], "no_filter")
    assert out[0].get_block(0).to_pylist() == [None, 6]


def test_varchar_conditions(ctx, monkeypatch):
    """VARCHAR predicates (=, IN, LIKE) as conditions, numeric results (Q12 and Q14 shapes)"""
    rng = np.random.default_rng(12)
    words = ["1-URGENT", "2-HIGH", "3-MEDIUM", "PROMO BRUSHED TIN", "STANDARD PROMO", "PROMO", "", None]
    n = 1500
    s = [words[int(rng.integers(0, len(words)))] for _ in range(n)]
    x = [int(v) for v in rng.integers(-50, 50, n)]
    f = [float(v) for v in rng.normal(0, 10, n)]
    rows = [(None if w is None else w.encode(), xi, fi) for w, xi, fi in zip(s, x, f)]
    page = Page(Block.varchar(s), Block.bigint(x), Block.double(f))
    V, X, F = ops.Col(0, S), ops.Col(1, B), ops.Col(2, D)
    urgent = call(abi.EX_OR, call(abi.EX_EQ, V, ops.Const("1-URGENT", S)), call(abi.EX_EQ, V, ops.Const("2-HIGH", S)))
    projs = [ops.Case([(urgent, ops.Const(1, B))], ops.Const(0, B)),
             ops.If(call(abi.EX_IN, V, in_list=["1-URGENT", "2-HIGH"]), ops.Const(0, B), ops.Const(1, B)),
             ops.If(call(abi.EX_LIKE, V, pattern="PROMO%"), call(abi.EX_MUL, F, ops.Const(2.0, D)), ops.Const(0.0, D)),
             ops.Coalesce(ops.If(call(abi.EX_EQ, V, ops.Const("", S)), X), ops.Const(-1, B)),
             ops.If(call(abi.EX_LIKE, V, pattern="%PROMO"), call(abi.EX_GT, X, ops.Const(0, B)), ops.Null(BOOL))]
    _check_rows(ctx, monkeypatch, rows, page, call(abi.EX_GT, ops.If(urgent, X, call(abi.EX_NEG, X)), ops.Const(-40, B)), projs)


def _hash_agg(ctx, key, aggs, pages, pre=None, expected=16):
    fac = ops.HashAggregationOperatorFactory(ctx, [key], abi.STEP_SINGLE, [ops.Aggregator(fn, ch, -1) for fn, ch in aggs], expected_groups=expected, pre=pre)
    op = fac.create_operator()
    try:
        return sorted((r for p in ops.drive(op, pages) for r in p.rows()), key=lambda r: (r[0] is None, r[0] if r[0] is not None else 0))
    finally:
        op.close()


def _global_agg(ctx, aggs, pages, pre, input_types):
    fac = ops.AggregationOperatorFactory(ctx, abi.STEP_SINGLE, [ops.Aggregator(fn, ch, -1) for fn, ch in aggs], pre=pre, input_types=input_types)
    op = fac.create_operator()
    try:
        return [r for p in ops.drive(op, pages) for r in p.rows()]
    finally:
        op.close()


@pytest.mark.parametrize("path", ["S", "G", "global"])
@pytest.mark.parametrize("nulls", ["x_non_null", "x_nullable", "both_nullable", "y_nullable"])
def test_count_of_conditionals(ctx, path, nulls):
    """count(IF(c, x, NULL)), count(IF(c, x, y)), count(COALESCE(x, y)) and count(*) in the fused pre-stage: count(e) may share
    count(*)'s accumulator only when e is never NULL, which depends on x's and y's nullability"""
    rng = np.random.default_rng(13)
    n = 300_001
    groups = 6 if path != "G" else 3000
    key = rng.integers(0, groups, n).astype(np.int32)
    x = rng.integers(-100, 100, n)
    y = rng.integers(-100, 100, n)
    c = rng.integers(0, 2, n).astype(np.int8)
    xn = rng.random(n) < 0.3 if nulls in ("x_nullable", "both_nullable") else None
    yn = rng.random(n) < 0.3 if nulls in ("both_nullable", "y_nullable") else None
    page = Page(Block.integer(key), Block.bigint(x, xn), Block.bigint(y, yn), Block.boolean(c))
    X, Y, Cc = ops.Col(1, B), ops.Col(2, B), ops.Col(3, BOOL)
    exprs = [ops.If(Cc, X), ops.If(Cc, X, Y), ops.Coalesce(X, Y), ops.Coalesce(ops.If(Cc, X), Y)]
    xv = np.zeros(n, bool) if xn is None else xn
    yv = np.zeros(n, bool) if yn is None else yn
    cb = c != 0
    nonnull = [cb & ~xv, np.where(cb, ~xv, ~yv), ~xv | ~yv, (cb & ~xv) | ~yv]
    if path == "global":
        pre = ops.PageProcessorProgram(None, exprs)
        got = _global_agg(ctx, [(abi.AGG_COUNT, k) for k in range(4)] + [(abi.AGG_COUNT_STAR, -1)], [page], pre,
                          [abi.INT32, abi.INT64, abi.INT64, abi.INT8])
        assert got == [tuple(int(m.sum()) for m in nonnull) + (n,)]
        return
    pre = ops.PageProcessorProgram(None, [0] + exprs)
    got = _hash_agg(ctx, 0, [(abi.AGG_COUNT, k) for k in range(1, 5)] + [(abi.AGG_COUNT_STAR, -1)], [page], pre,
                    expected=16 if path == "S" else 10_000)
    want = [(g,) + tuple(int(m[key == g].sum()) for m in nonnull) + (int((key == g).sum()),) for g in range(groups) if (key == g).any()]
    assert got == want


def test_q12_pipeline(ctx):
    """Q12's CASE: FilterAndProject (shipmode IN, CASE over the order priority) -> HashAggregationOperator sum, against agg_reference"""
    rng = np.random.default_rng(14)
    modes = ["MAIL", "SHIP", "AIR", "RAIL", "TRUCK"]
    prios = ["1-URGENT", "2-HIGH", "3-MEDIUM", "4-NOT SPECIFIED", "5-LOW"]
    pages, rows = [], []
    for n in (1, 1024, 1025, 200_000):
        m = [modes[i] for i in rng.integers(0, 5, n)]
        p = [prios[i] for i in rng.integers(0, 5, n)]
        k = rng.integers(0, 8, n).astype(np.int8)
        pages.append(Page(Block.varchar(m), Block.varchar(p), Block.tinyint(k)))
        rows += [(a.encode(), b.encode(), int(c)) for a, b, c in zip(m, p, k)]
    M, P, Kc = ops.Col(0, S), ops.Col(1, S), ops.Col(2, B)
    high = call(abi.EX_OR, call(abi.EX_EQ, P, ops.Const("1-URGENT", S)), call(abi.EX_EQ, P, ops.Const("2-HIGH", S)))
    high_line = ops.Case([(high, ops.Const(1, B))], ops.Const(0, B))
    low_line = ops.Case([(call(abi.EX_AND, call(abi.EX_NE, P, ops.Const("1-URGENT", S)), call(abi.EX_NE, P, ops.Const("2-HIGH", S))),
                          ops.Const(1, B))], ops.Const(0, B))
    flt = call(abi.EX_IN, M, in_list=["MAIL", "SHIP"])
    prog = ops.PageProcessorProgram(flt, [2, high_line, low_line])
    op = ops.FilterAndProjectOperatorFactory(ctx, prog).create_operator()
    try:
        mid = ops.drive(op, pages)
    finally:
        op.close()
    got = _hash_agg(ctx, 0, [(abi.AGG_SUM, 1), (abi.AGG_SUM, 2), (abi.AGG_COUNT_STAR, -1)], mid)
    sel = [r for r in rows if cr.evaluate(flt, r)]
    ref_page = Page(Block.tinyint([r[2] for r in sel]), Block.bigint([cr.evaluate(high_line, r) for r in sel]),
                    Block.bigint([cr.evaluate(low_line, r) for r in sel]))
    want = sorted(agg_reference.aggregate([ref_page], [0], [(abi.AGG_SUM, 1, -1), (abi.AGG_SUM, 2, -1), (abi.AGG_COUNT_STAR, -1, -1)]))
    assert got == want


def test_q14_pipeline(ctx):
    """Q14's CASE: sum(CASE WHEN p_type LIKE 'PROMO%' THEN l_extendedprice * (1 - l_discount) ELSE 0 END) as decimal(26, 4), through
    FilterAndProject -> HashAggregationOperator (decimal sum), over dictionary and RLE blocks, against exact integers"""
    rng = np.random.default_rng(15)
    types = ["PROMO BRUSHED COPPER", "STANDARD POLISHED TIN", "PROMO ANODIZED STEEL", "ECONOMY BURNISHED NICKEL"]
    T = (12, 2)
    pages, rows = [], []
    for n, enc in ((1, "flat"), (1023, "dict"), (4097, "rle"), (300_000, "flat")):
        ep = rng.integers(90_000, 10_500_000, n)
        disc = rng.integers(0, 11, n)
        k = rng.integers(0, 4, n).astype(np.int8)
        ty = [types[i] for i in rng.integers(0, 4, n)]
        if enc == "rle":
            ty = [ty[0]] * n
            tblock = RunLengthEncodedBlock(Block.varchar(ty[:1]), n)
        elif enc == "dict":
            idx = rng.integers(0, 4, n)
            ty = [types[i] for i in idx]
            tblock = DictionaryBlock(Block.varchar(types), idx)
        else:
            tblock = Block.varchar(ty)
        pages.append(Page(tblock, Block.bigint(ep), Block.bigint(disc), Block.tinyint(k)))
        rows += [(t.encode(), int(a), int(b), int(c)) for t, a, b, c in zip(ty, ep, disc, k)]
    Ty, EP, DI = ops.Col(0, S), ops.Col(1, DEC, T), ops.Col(2, DEC, T)
    rev = call(abi.EX_MUL, EP, call(abi.EX_SUB, ops.Const(1, DEC, (1, 0)), DI))
    promo = ops.Case([(call(abi.EX_LIKE, Ty, pattern="PROMO%"), rev)], ops.Const(0, DEC, rev.dtype))
    assert promo.dtype == (26, 4)
    prog = ops.PageProcessorProgram(call(abi.EX_GE, EP, ops.Const(100_000, DEC, T)), [3, promo, rev])
    op = ops.FilterAndProjectOperatorFactory(ctx, prog).create_operator()
    try:
        mid = ops.drive(op, pages)
    finally:
        op.close()
    got = _hash_agg(ctx, 0, [(abi.AGG_SUM_DECIMAL, 1), (abi.AGG_SUM_DECIMAL, 2)], mid)
    want = {}
    for t, a, b, k in rows:
        if a < 100_000:
            continue
        r = a * (100 - b)
        s = want.setdefault(k, [0, 0])
        s[0] += r if t.startswith(b"PROMO") else 0
        s[1] += r
    assert got == sorted((k, v[0], v[1]) for k, v in want.items())


def test_interpreter_forms_in_child_process():
    """the interpreter kernels (fp_filter_kernel, fp_project_kernel, the pre-stage of agg_small_kernel and the global kernel's twin)"""
    if NO_JIT:
        pytest.skip("already the child")
    env = dict(os.environ, TGPU_DISABLE_JIT="1")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", "-p", "no:cacheprovider", os.path.abspath(__file__)],
                       cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=2400)
    assert r.returncode == 0, r.stdout[-6000:]
    assert " passed" in r.stdout and "1 skipped" in r.stdout, r.stdout[-2000:]
