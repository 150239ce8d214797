"""DECIMAL arithmetic, comparisons and casts in FilterAndProject on the GPU, compared exactly with decimal_reference.

Each operation runs over short (TGPU_INT64) and long (TGPU_INT128) columns with NULLs, at the edge values of its types (0, +-1,
+-(10^p - 1), HALF_UP ties, 2^53 +- 1, products past 128 bits, zero and +-1 divisors), in the forms
- chunked:          a filter, the chunked two-pass kernels
- selection_vector: the same program with TGPU_FP_SELECTION_VECTOR=1
- no_filter:        the projection alone
A page whose selected rows raise must fail with the reference's status; the same page without those rows gives every value and NULL.
test_interpreter_forms_in_child_process runs the file again with TGPU_DISABLE_JIT=1 (fp_filter_kernel / fp_project_kernel)."""
import os
import random
import subprocess
import sys

import pytest

import decimal_reference as dref
from trino_b200 import abi
from trino_b200 import operators as ops
from trino_b200.page import Block, Page

pytestmark = pytest.mark.gpu
B, D, BOOL, DEC = abi.V_BIGINT, abi.V_DOUBLE, abi.V_BOOLEAN, abi.V_DECIMAL
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NO_JIT = bool(os.environ.get("TGPU_DISABLE_JIT"))
FORMS = ("chunked", "selection_vector", "no_filter")
CMP = (abi.EX_EQ, abi.EX_NE, abi.EX_LT, abi.EX_LE, abi.EX_GT, abi.EX_GE)

# (op, operand vtype, operand types, result type or None for the default rules)
CASES = [
    (abi.EX_ADD, DEC, [(12, 2), (12, 2)], None), (abi.EX_SUB, DEC, [(12, 2), (18, 4)], None), (abi.EX_ADD, DEC, [(26, 4), (12, 2)], None),
    (abi.EX_SUB, DEC, [(38, 6), (38, 0)], None), (abi.EX_ADD, DEC, [(38, 10), (1, 0)], None), (abi.EX_SUB, DEC, [(17, 0), (18, 18)], (18, 18)),
    (abi.EX_ADD, DEC, [(18, 2), (18, 2)], (18, 2)),
    (abi.EX_MUL, DEC, [(12, 2), (5, 2)], None), (abi.EX_MUL, DEC, [(12, 2), (13, 2)], None), (abi.EX_MUL, DEC, [(26, 4), (13, 2)], None),
    (abi.EX_MUL, DEC, [(38, 10), (38, 10)], None), (abi.EX_MUL, DEC, [(20, 10), (5, 5)], None), (abi.EX_MUL, DEC, [(18, 0), (18, 0)], (36, 0)),
    (abi.EX_MUL, DEC, [(10, 0), (9, 0)], (18, 0)),
    (abi.EX_DIV, DEC, [(12, 2), (12, 2)], None), (abi.EX_DIV, DEC, [(5, 2), (3, 1)], None), (abi.EX_DIV, DEC, [(26, 4), (12, 2)], None),
    (abi.EX_DIV, DEC, [(12, 2), (26, 4)], None), (abi.EX_DIV, DEC, [(38, 6), (38, 6)], None), (abi.EX_DIV, DEC, [(12, 2), (12, 2)], (14, 2)),
    (abi.EX_DIV, DEC, [(18, 0), (18, 0)], (18, 0)), (abi.EX_DIV, DEC, [(20, 2), (12, 2)], (18, 2)), (abi.EX_DIV, DEC, [(12, 2), (20, 2)], (18, 2)),
    (abi.EX_NEG, DEC, [(12, 2)], None), (abi.EX_NEG, DEC, [(38, 6)], None),
    (abi.EX_CAST_TO_DECIMAL, B, [None], (12, 2)), (abi.EX_CAST_TO_DECIMAL, B, [None], (18, 0)), (abi.EX_CAST_TO_DECIMAL, B, [None], (38, 6)),
    (abi.EX_CAST_TO_DECIMAL, B, [None], (20, 19)),
    (abi.EX_CAST_TO_DECIMAL, DEC, [(12, 2)], (18, 4)), (abi.EX_CAST_TO_DECIMAL, DEC, [(18, 4)], (12, 2)), (abi.EX_CAST_TO_DECIMAL, DEC, [(12, 2)], (26, 10)),
    (abi.EX_CAST_TO_DECIMAL, DEC, [(38, 6)], (12, 2)), (abi.EX_CAST_TO_DECIMAL, DEC, [(26, 4)], (38, 10)), (abi.EX_CAST_TO_DECIMAL, DEC, [(38, 6)], (20, 2)),
    (abi.EX_CAST_DECIMAL_TO_BIGINT, DEC, [(12, 2)], None), (abi.EX_CAST_DECIMAL_TO_BIGINT, DEC, [(38, 6)], None),
    (abi.EX_CAST_DECIMAL_TO_BIGINT, DEC, [(18, 0)], None), (abi.EX_CAST_DECIMAL_TO_BIGINT, DEC, [(38, 0)], None),
    (abi.EX_CAST_DECIMAL_TO_DOUBLE, DEC, [(18, 4)], None), (abi.EX_CAST_DECIMAL_TO_DOUBLE, DEC, [(16, 0)], None),
    (abi.EX_CAST_DECIMAL_TO_DOUBLE, DEC, [(38, 10)], None), (abi.EX_CAST_DECIMAL_TO_DOUBLE, DEC, [(26, 4)], None),
    (abi.EX_CAST_DECIMAL_TO_DOUBLE, DEC, [(38, 0)], None), (abi.EX_CAST_DECIMAL_TO_DOUBLE, DEC, [(19, 19)], None),
] + [(op, DEC, [t, t], None) for op in CMP for t in ((12, 2), (38, 6))] + [
    (abi.EX_BETWEEN, DEC, [(12, 2)] * 3, None), (abi.EX_BETWEEN, DEC, [(26, 4)] * 3, None),
    (abi.EX_IS_NULL, DEC, [(12, 2)], None), (abi.EX_IS_NOT_NULL, DEC, [(38, 6)], None),
]


def _edge_values(t, rng):
    if t is None:     # BIGINT
        vals = [0, 1, -1, 10, -10, 12345, 2 ** 63 - 1, -2 ** 63, 10 ** 17, -10 ** 17, 10 ** 18, 92233720368547758, -92233720368547759]
        return vals + [rng.randrange(-10 ** 12, 10 ** 12) for _ in range(20)]
    p, s = t
    m = 10 ** p - 1
    vals = [0, 1, -1, m, -m, m // 2, -m // 2, 5, -5, 15, -15, 25, -25]
    if s > 0:
        vals += [10 ** s // 2, -(10 ** s // 2), 10 ** s + 10 ** s // 2, -(10 ** s + 10 ** s // 2), 10 ** s, -10 ** s]
    if p >= 16:
        vals += [2 ** 53 + 1, -(2 ** 53 + 1), 2 ** 53 - 1, 2 ** 53 + 3]
    vals += [rng.randrange(-m, m + 1) for _ in range(24)]
    vals += [rng.randrange(-10 ** (p // 2), 10 ** (p // 2) + 1) for _ in range(12)]
    return [v for v in vals if abs(v) <= m]


def _block(t, values):
    if t is None or t[0] <= 18:
        return Block.bigint([0 if v is None else v for v in values], [v is None for v in values])
    return Block.int128(values)


def _rows(case, rng, n):
    op, vt, types, _ = case
    pools = [_edge_values(t, rng) for t in types]
    rows = []
    for i in range(n):
        row = [rng.choice(pl) if rng.random() > 0.08 else None for pl in pools]
        rows.append(row)
    # pairs of edge values against each other, so that products past 128 bits, +-1 and zero divisors and ties appear
    if len(pools) > 1:
        for x in pools[0][:13]:
            for y in pools[1][:13]:
                rows.append([x, y] + [rng.choice(pl) for pl in pools[2:]])
    else:
        rows += [[x] for x in pools[0]]
    return rows


def _expr(case):
    op, vt, types, rt = case
    args = [ops.Col(k, vt, types[k]) for k in range(len(types))]
    kw = {"result_dtype": rt} if rt is not None else {}
    return ops.Call(op, *args, **kw)


def _expected(case, row, expr):
    """(value or None) of one row, or raise DecimalError"""
    op, vt, types, _ = case
    if op == abi.EX_IS_NULL:
        return row[0] is None
    if op == abi.EX_IS_NOT_NULL:
        return row[0] is not None
    if op == abi.EX_BETWEEN:
        a, b, c = row
        if a is None:
            return None
        f1 = b is not None and a < b
        f2 = c is not None and a > c
        if f1 or f2:
            return False
        return None if (b is None or c is None) else True
    if any(v is None for v in row):
        return None
    sig = (types[0], types[1] if len(types) > 1 else None, None, expr.dtype)
    return dref.apply(op, vt, sig, *row)


_PRIORITY = {abi.ERR_DIVISION_BY_ZERO: 0, abi.ERR_INVALID_CAST_ARGUMENT: 1, abi.ERR_NUMERIC_VALUE_OUT_OF_RANGE: 2}


def _run(ctx, prog, page, monkeypatch, form):
    if form == "selection_vector":
        monkeypatch.setenv("TGPU_FP_SELECTION_VECTOR", "1")
    else:
        monkeypatch.delenv("TGPU_FP_SELECTION_VECTOR", raising=False)
    f = ops.FilterAndProjectOperatorFactory(ctx, prog)
    op = f.create_operator()
    try:
        op.add_input(page)
        out = op.get_output()
    finally:
        op.close()
    return out


def _check_case(ctx, case, form, monkeypatch, seed):
    rng = random.Random(seed)
    op, vt, types, _ = case
    expr = _expr(case)
    rows = _rows(case, rng, 160)
    keep = [i % 5 != 3 for i in range(len(rows))] if form != "no_filter" else [True] * len(rows)
    flt = ops.Call(abi.EX_NE, ops.Col(len(types), B), ops.Const(0, B)) if form != "no_filter" else None
    prog = ops.PageProcessorProgram(flt, [expr, len(types)])
    want, raised = [], []
    for r, k in zip(rows, keep):
        if not k:
            continue
        try:
            want.append(_expected(case, r, expr))
            raised.append(None)
        except dref.DecimalError as e:
            want.append(None)
            raised.append(e.status)

    def page(sel):
        cols = [_block(types[k] if vt == DEC else None, [rows[i][k] for i in sel]) for k in range(len(types))]
        return Page(*cols, Block.bigint([1 if keep[i] else 0 for i in sel]))

    kept = [i for i in range(len(rows)) if keep[i]]
    statuses = [s for s in raised if s is not None]
    if statuses:
        with pytest.raises(abi.TrinoGpuError) as exc:
            _run(ctx, prog, page(range(len(rows))), monkeypatch, form)
        assert exc.value.code == min(statuses, key=lambda s: _PRIORITY[s]), (case, form)
    good = [i for i, s in zip(kept, raised) if s is None]
    wanted = [w for w, s in zip(want, raised) if s is None]
    good_all = [i for i in range(len(rows)) if not keep[i]] + good
    out = _run(ctx, prog, page(sorted(good_all)), monkeypatch, form)
    got = out.get_block(0).to_pylist() if out is not None else []
    order = sorted(good_all)
    want_by_row = dict(zip(good, wanted))
    exp = [want_by_row[i] for i in order if keep[i]]
    if expr.result_vtype == BOOL:
        got = [None if g is None else bool(g) for g in got]
    assert len(got) == len(exp), (case, form)
    for g, w, i in zip(got, exp, [i for i in order if keep[i]]):
        assert g == w, (case, form, rows[i], g, w)


@pytest.fixture(scope="module")
def ctx():
    c = ops.Context(0)
    yield c
    c.close()


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("k", range(len(CASES)))
def test_decimal_operation(ctx, monkeypatch, form, k):
    _check_case(ctx, CASES[k], form, monkeypatch, 1000 + k)


def test_decimal_q1_program_multi_tile(ctx, monkeypatch):
    """Q1's revenue expressions over decimal(12,2) columns, on one page of several chunk tiles, against the reference"""
    rng = random.Random(7)
    n = 300_000
    t = (12, 2)
    ep = [rng.randrange(90_000, 10_500_000) for _ in range(n)]
    disc = [rng.randrange(0, 11) for _ in range(n)]
    tax = [None if i % 97 == 0 else rng.randrange(0, 9) for i in range(n)]
    ship = [rng.randrange(0, 2600) for _ in range(n)]
    one = ops.Const(1, DEC, (1, 0))
    c_ep, c_disc, c_tax = ops.Col(0, DEC, t), ops.Col(1, DEC, t), ops.Col(2, DEC, t)
    disc_price = ops.Call(abi.EX_MUL, c_ep, ops.Call(abi.EX_SUB, one, c_disc))
    charge = ops.Call(abi.EX_MUL, disc_price, ops.Call(abi.EX_ADD, one, c_tax))
    assert disc_price.dtype == (26, 4) and charge.dtype == (38, 6)
    prog = ops.PageProcessorProgram(ops.Call(abi.EX_LE, ops.Col(3, B), ops.Const(2400, B)), [disc_price, charge, 0])
    page = Page(Block.bigint(ep), Block.bigint(disc), Block.bigint([0 if v is None else v for v in tax], [v is None for v in tax]),
                Block.integer(ship))
    for form in ("chunked", "selection_vector"):
        out = _run(ctx, prog, page, monkeypatch, form)
        sel = [i for i in range(n) if ship[i] <= 2400]
        dp = out.get_block(0).to_pylist()
        ch = out.get_block(1).to_pylist()
        assert len(dp) == len(sel)
        for j, i in enumerate(sel):
            w = ep[i] * (100 - disc[i])
            assert dp[j] == w
            assert ch[j] == (None if tax[i] is None else w * (100 + tax[i]))


def test_wrong_channel_type_at_add_input(ctx, monkeypatch):
    prog = ops.PageProcessorProgram(None, [ops.Call(abi.EX_NEG, ops.Col(0, DEC, (38, 2)))])
    with pytest.raises(abi.TrinoGpuError) as exc:
        _run(ctx, prog, Page(Block.bigint([1, 2])), monkeypatch, "no_filter")
    assert exc.value.code == abi.ERR_INVALID_ARGUMENT
    prog = ops.PageProcessorProgram(None, [ops.Call(abi.EX_NEG, ops.Col(0, DEC, (12, 2)))])
    with pytest.raises(abi.TrinoGpuError) as exc:
        _run(ctx, prog, Page(Block.int128([1, 2])), monkeypatch, "no_filter")
    assert exc.value.code == abi.ERR_INVALID_ARGUMENT


@pytest.mark.skipif(NO_JIT, reason="this is the child run")
def test_interpreter_forms_in_child_process():
    env = dict(os.environ, TGPU_DISABLE_JIT="1")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", "-p", "no:cacheprovider", os.path.abspath(__file__)],
                       cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-4000:]
