"""DECIMAL FilterAndProject on the GPU beyond single operations: the reference's own cases on the device, decimal Q1 and Q6 end to end through
the decimal accumulators on one page of 4 M rows, DICT32 / RLE blocks and device pages, a VARCHAR pass-through channel, seeded random
trees that mix DECIMAL with BIGINT, DOUBLE and BOOLEAN operations and a raising one (where the error is raised), and the refusals of the
fused aggregation pre-stage and of filtered join builds through their create entry points."""
import ctypes as C
import random

import numpy as np
import pytest

import decimal_golden as dg
import decimal_reference as dref
from trino_b200 import abi
from trino_b200 import operators as ops
from trino_b200.page import Block, DictionaryBlock, Page, RunLengthEncodedBlock

pytestmark = pytest.mark.gpu
B, D, BOOL, DEC, S = abi.V_BIGINT, abi.V_DOUBLE, abi.V_BOOLEAN, abi.V_DECIMAL, abi.V_VARCHAR
PRIORITY = {abi.ERR_DIVISION_BY_ZERO: 0, abi.ERR_NUMERIC_VALUE_OUT_OF_RANGE: 1, abi.ERR_INVALID_CAST_ARGUMENT: 2}


@pytest.fixture(scope="module")
def ctx():
    c = ops.Context(0)
    yield c
    c.close()


def _run(ctx, prog, pages, device_out=False):
    op = ops.FilterAndProjectOperatorFactory(ctx, prog).create_operator()
    out = []
    try:
        for p in pages:
            op.add_input(p)
            o = op.get_output_device() if device_out else op.get_output()
            if o is not None:
                out.append(o)
    finally:
        op.close()
    return out


def _block(t, values):
    if isinstance(t, str):
        return (Block.bigint if t == "bigint" else Block.integer)([0 if v is None else v for v in values], [v is None for v in values])
    if t[0] <= 18:
        return Block.bigint([0 if v is None else v for v in values], [v is None for v in values])
    return Block.int128(values)


def _same(got, want):
    return got == want if not isinstance(want, bool) or got is None else bool(got) == want


# ---- the reference's cases ---------------------------------------------------------------------------------------------------------
def _signature(case):
    return (case["op"], tuple(dg.arg_type(a) for a in case["args"]), str(case.get("target")))


def test_golden_cases_over_columns(ctx):
    """cases of one signature share a program over one page (error cases one row each)"""
    groups = {}
    for c in dg.CASES:
        groups.setdefault(_signature(c) + (("error", c["source"]) if "error" in c else ()), []).append(c)
    for key, cases in groups.items():
        c0 = cases[0]
        expr = dg.expression(c0, [dg.operand_expr(a, k, True) for k, a in enumerate(c0["args"])])
        prog = ops.PageProcessorProgram(None, [expr])
        page = Page(*[_block(dg.arg_type(a), [None if c["args"][k]["value"] is None else int(c["args"][k]["value"]) for c in cases])
                      for k, a in enumerate(c0["args"])])
        if "error" in c0:
            with pytest.raises(abi.TrinoGpuError) as exc:
                _run(ctx, prog, [page])
            assert exc.value.code == dg.wanted(c0), c0["source"]
            continue
        got = _run(ctx, prog, [page])[0].get_block(0).to_pylist()
        for g, c in zip(got, cases):
            assert _same(g, dg.wanted(c)), (c["source"], g, dg.wanted(c))


def test_golden_cases_over_constants(ctx):
    """up to six cases per program as constant projections (error cases alone)"""
    ok = [c for c in dg.CASES if "error" not in c]
    batches = [ok[k:k + 6] for k in range(0, len(ok), 6)] + [[c] for c in dg.CASES if "error" in c]
    for batch in batches:
        exprs = [dg.expression(c, [dg.operand_expr(a, k, False) for k, a in enumerate(c["args"])]) for c in batch]
        prog = ops.PageProcessorProgram(None, exprs)
        page = Page(Block.bigint([0]))
        if "error" in batch[0]:
            with pytest.raises(abi.TrinoGpuError) as exc:
                _run(ctx, prog, [page])
            assert exc.value.code == dg.wanted(batch[0]), batch[0]["source"]
            continue
        out = _run(ctx, prog, [page])[0]
        for k, c in enumerate(batch):
            g = out.get_block(k).to_pylist()[0]
            assert _same(g, dg.wanted(c)), (c["source"], g, dg.wanted(c))


# ---- decimal Q1 / Q6 end to end ------------------------------------------------------------------------------------------------------
N_BIG = 4 * 1024 * 1024
T = (12, 2)


def _lineitem(n, seed):
    rng = np.random.default_rng(seed)
    return {
        "ship": rng.integers(0, 2600, n).astype(np.int32),
        "flag": rng.integers(0, 3, n).astype(np.int8),
        "status": rng.integers(0, 2, n).astype(np.int8),
        "qty": rng.integers(100, 5001, n).astype(np.int64),             # decimal(12,2): 1.00 .. 50.00
        "ep": rng.integers(90_000, 10_500_000, n).astype(np.int64),
        "disc": rng.integers(0, 11, n).astype(np.int64),
        "tax": rng.integers(0, 9, n).astype(np.int64),
    }


def _li_page(li):
    return Page(Block.integer(li["ship"]), Block.tinyint(li["flag"]), Block.tinyint(li["status"]), Block.bigint(li["qty"]),
                Block.bigint(li["ep"]), Block.bigint(li["disc"]), Block.bigint(li["tax"]))


def _half_up_div(s, n):
    q, r = divmod(abs(s), n)
    q += 1 if 2 * r >= n else 0
    return q if s >= 0 else -q


def test_decimal_q1_end_to_end(ctx):
    """FilterAndProject (l_extendedprice * (1 - l_discount) as decimal(26,4), * (1 + l_tax) as decimal(38,6)) -> HashAggregation with decimal
    sum and avg, over one page of 4 M rows, against exact integer arithmetic"""
    li = _lineitem(N_BIG, 11)
    one = ops.Const(1, DEC, (1, 0))
    qty, ep, disc, tax = (ops.Col(c, DEC, T) for c in (3, 4, 5, 6))
    disc_price = ops.Call(abi.EX_MUL, ep, ops.Call(abi.EX_SUB, one, disc))
    charge = ops.Call(abi.EX_MUL, disc_price, ops.Call(abi.EX_ADD, one, tax))
    prog = ops.PageProcessorProgram(ops.Call(abi.EX_LE, ops.Col(0, B), ops.Const(2400, B)), [1, 2, 3, 4, disc_price, charge, 5])
    out = _run(ctx, prog, [_li_page(li)], device_out=True)
    A = ops.Aggregator
    aggs = [A(abi.AGG_SUM_DECIMAL, 2), A(abi.AGG_SUM_DECIMAL, 3), A(abi.AGG_SUM_DECIMAL, 4), A(abi.AGG_SUM_DECIMAL, 5),
            A(abi.AGG_AVG_DECIMAL, 2), A(abi.AGG_AVG_DECIMAL, 3), A(abi.AGG_AVG_DECIMAL, 6), A(abi.AGG_COUNT_STAR)]
    agg = ops.HashAggregationOperatorFactory(ctx, [0, 1], abi.STEP_SINGLE, aggs, 16).create_operator()
    try:
        res = ops.drive(agg, out)
    finally:
        agg.close()
        for o in out:
            o.release()
    rows = sorted(r for p in res for r in zip(*[p.get_block(c).to_pylist() for c in range(p.channel_count)]))
    sel = li["ship"] <= 2400
    dp = li["ep"] * (100 - li["disc"])
    ch = dp * (100 + li["tax"])
    want = []
    for f in range(3):
        for s in range(2):
            m = sel & (li["flag"] == f) & (li["status"] == s)
            n = int(m.sum())
            if n == 0:
                continue
            sq, se, sd = int(li["qty"][m].sum()), int(li["ep"][m].sum()), int(li["disc"][m].sum())
            want.append((f, s, sq, se, int(dp[m].sum()), int(ch[m].sum()), _half_up_div(sq, n), _half_up_div(se, n), _half_up_div(sd, n), n))
    assert rows == sorted(want)


def test_decimal_q6_end_to_end(ctx):
    """FilterAndProject (l_extendedprice * l_discount as decimal(25,4)) -> AggregationOperator sum, 1.5 M rows over three pages"""
    li = _lineitem(1_500_000, 12)
    ep, disc, qty = ops.Col(4, DEC, T), ops.Col(5, DEC, T), ops.Col(3, DEC, T)
    flt = ops.Call(abi.EX_AND, ops.Call(abi.EX_BETWEEN, ops.Col(0, B), ops.Const(365, B), ops.Const(729, B)),
                   ops.Call(abi.EX_AND, ops.Call(abi.EX_BETWEEN, disc, ops.Const(5, DEC, T), ops.Const(7, DEC, T)),
                            ops.Call(abi.EX_LT, qty, ops.Const(2400, DEC, T))))
    revenue = ops.Call(abi.EX_MUL, ep, disc)
    assert revenue.dtype == (25, 4)
    prog = ops.PageProcessorProgram(flt, [revenue])
    pages = []
    for a in range(0, 1_500_000, 500_000):
        pages.append(_li_page({k: v[a:a + 500_000] for k, v in li.items()}))
    out = _run(ctx, prog, pages, device_out=True)
    agg = ops.AggregationOperatorFactory(ctx, abi.STEP_SINGLE, [ops.Aggregator(abi.AGG_SUM_DECIMAL, 0)], input_types=[abi.INT128]).create_operator()
    try:
        res = ops.drive(agg, out)
    finally:
        agg.close()
        for o in out:
            o.release()
    m = (li["ship"] >= 365) & (li["ship"] <= 729) & (li["disc"] >= 5) & (li["disc"] <= 7) & (li["qty"] < 2400)
    assert res[0].get_block(0).to_pylist() == [int((li["ep"][m] * li["disc"][m]).sum())]


def test_big_page_values(ctx):
    """one page of 4 M rows: every long output cell of a short x short -> long product and a division, checked in bulk"""
    li = _lineitem(N_BIG, 13)
    ep, qty = ops.Col(4, DEC, T), ops.Col(3, DEC, T)
    prog = ops.PageProcessorProgram(ops.Call(abi.EX_GT, ops.Col(0, B), ops.Const(100, B)),
                                    [ops.Call(abi.EX_MUL, ep, qty), ops.Call(abi.EX_DIV, ep, ops.Col(5, DEC, T), result_dtype=(18, 2))])
    li["disc"][li["disc"] == 0] = 1
    out = _run(ctx, prog, [_li_page(li)])[0]
    sel = li["ship"] > 100
    prod = li["ep"][sel] * li["qty"][sel]
    cells = out.get_block(0).values
    assert np.array_equal(cells[:, 1], prod) and np.array_equal(cells[:, 0], prod >> 63)
    e, d = li["ep"][sel], li["disc"][sel]
    q = (e * 100) // d
    q = q + ((e * 100 - q * d) * 2 >= d)
    assert np.array_equal(out.get_block(1).values, q)


# ---- encodings and device pages ----------------------------------------------------------------------------------------------------
def test_dictionary_rle_and_device_pages(ctx):
    rng = random.Random(5)
    n = 5000
    dict_vals = [None, 0, 1, -1, 10 ** 30, -(10 ** 30), 10 ** 37 - 1, 123456789012345678901234]
    ids = [rng.randrange(len(dict_vals)) for _ in range(n)]
    short = [rng.randrange(-10 ** 9, 10 ** 9) for _ in range(n)]
    prog = ops.PageProcessorProgram(ops.Call(abi.EX_IS_NOT_NULL, ops.Col(1, DEC, (12, 2))),
                                    [ops.Call(abi.EX_ADD, ops.Col(0, DEC, (38, 6)), ops.Col(1, DEC, (12, 2))), ops.Call(abi.EX_NEG, ops.Col(2, DEC, (20, 0))), 0])
    sig = ((38, 6), (12, 2), None, ops.decimal_result_type(abi.EX_ADD, (38, 6), (12, 2)))
    rle_v = 10 ** 19 + 7

    def expect(a_vals, b_vals):
        return [None if a is None else dref.apply(abi.EX_ADD, DEC, sig, a, b) for a, b in zip(a_vals, b_vals)]

    a_vals = [dict_vals[i] for i in ids]
    pages = {
        "dict_rle": Page(DictionaryBlock(Block.int128(dict_vals), np.array(ids, np.int32)), Block.bigint(short),
                         RunLengthEncodedBlock(Block.int128([rle_v]), n)),
        "flat": Page(Block.int128(a_vals), Block.bigint(short), Block.int128([rle_v] * n)),
    }
    for name, page in pages.items():
        out = _run(ctx, prog, [page])[0]
        assert out.get_block(0).to_pylist() == expect(a_vals, short), name
        assert out.get_block(1).to_pylist() == [-rle_v] * n, name
    # the flat page from device memory
    flat = pages["flat"]
    cols = []
    for c in range(3):
        b = flat.get_block(c)
        valid = None if b.nulls is None else ctx.to_device(np.packbits(~np.asarray(b.nulls, bool), bitorder="little"))
        cols.append(ops.DeviceColumn(b.type, ctx.to_device(np.ascontiguousarray(b.values)), n, valid))
    out = _run(ctx, prog, [ops.DevicePage(cols, n)])[0]
    assert out.get_block(0).to_pylist() == expect(a_vals, short)


def test_varchar_pass_through(ctx):
    """a VARCHAR channel passed through beside long DECIMAL results (the selection-vector form with a gather of the strings)"""
    n = 3000
    rng = random.Random(8)
    a = [rng.randrange(-10 ** 25, 10 ** 25) for _ in range(n)]
    s = [("row%d" % i) * (i % 4) for i in range(n)]
    keep = [i % 3 != 0 for i in range(n)]
    prog = ops.PageProcessorProgram(ops.Call(abi.EX_NE, ops.Col(2, B), ops.Const(0, B)),
                                    [1, ops.Call(abi.EX_MUL, ops.Col(0, DEC, (26, 4)), ops.Const(3, DEC, (1, 0))), 1])
    out = _run(ctx, prog, [Page(Block.int128(a), Block.varchar(s), Block.bigint([int(k) for k in keep]))])[0]
    sel = [i for i in range(n) if keep[i]]
    assert out.get_block(0).to_pylist() == [s[i].encode() for i in sel]
    assert out.get_block(1).to_pylist() == [a[i] * 3 for i in sel]


# ---- random trees: where the error is raised ------------------------------------------------------------------------------------
class _Err(Exception):
    def __init__(self, status):
        self.status = status


def _eval(e, row):
    """value of expression e on one row in the reference's evaluation order: AND / OR short-circuit, a NULL argument skips the rest; an
    error raises _Err"""
    if isinstance(e, ops.Col):
        return row[e.channel]
    if isinstance(e, ops.Const):
        return e.value
    if isinstance(e, ops.Null):
        return None
    op = e.op
    if op in (abi.EX_AND, abi.EX_OR):
        a = _eval(e.args[0], row)
        if a is not None and bool(a) == (op == abi.EX_OR):
            return op == abi.EX_OR
        b = _eval(e.args[1], row)
        if b is not None and bool(b) == (op == abi.EX_OR):
            return op == abi.EX_OR
        return None if a is None or b is None else op != abi.EX_OR
    if op == abi.EX_NOT:
        a = _eval(e.args[0], row)
        return None if a is None else not a
    vals = []
    for x in e.args:
        v = _eval(x, row)
        if v is None:
            return None
        vals.append(v)
    try:
        if e.operand_vtype == DEC:
            return dref.apply(op, DEC, tuple(e.operand_dtypes + [None] * (3 - len(e.operand_dtypes))) + (e.dtype,), *vals)
        if op == abi.EX_CAST_TO_DECIMAL:
            return dref.bigint_to_decimal(vals[0], e.dtype)
    except dref.DecimalError as x:
        raise _Err(x.status)
    if op == abi.EX_ADD:
        r = vals[0] + vals[1]
        if not -(1 << 63) <= r < 1 << 63:
            raise _Err(abi.ERR_NUMERIC_VALUE_OUT_OF_RANGE)
        return r
    if op == abi.EX_GT:
        return vals[0] > vals[1]
    if op == abi.EX_LT:
        return vals[0] < vals[1]
    if op == abi.EX_CAST_BIGINT_TO_DOUBLE:
        return float(vals[0])
    raise ValueError(op)


def _random_tree(rng, depth):
    """a BOOLEAN tree over c0 decimal(12,2), c1 decimal(30,4), c2 BIGINT, c3 decimal(12,2) (zeros: the raising division)"""
    c0, c1, c2, c3 = ops.Col(0, DEC, (12, 2)), ops.Col(1, DEC, (30, 4)), ops.Col(2, B), ops.Col(3, DEC, (12, 2))
    if depth == 0:
        k = rng.randrange(6)
        if k == 0:
            return ops.Call(abi.EX_GT, ops.Call(abi.EX_DIV, c0, c3, result_dtype=(18, 2)), ops.Const(rng.randrange(-500, 500), DEC, (18, 2)))
        if k == 1:
            lhs = ops.Call(abi.EX_ADD, c1, ops.Call(abi.EX_CAST_TO_DECIMAL, c2, result_dtype=(19, 0)))
            return ops.Call(abi.EX_LT, lhs, ops.Const(rng.randrange(-10 ** 20, 10 ** 20), DEC, lhs.dtype))
        if k == 2:
            return ops.Call(abi.EX_GT, ops.Call(abi.EX_ADD, c2, ops.Const(rng.choice([1, 2 ** 62]), B)), ops.Const(0, B))
        if k == 3:
            return ops.Call(abi.EX_LT, ops.Call(abi.EX_CAST_BIGINT_TO_DOUBLE, c2), ops.Const(float(rng.randrange(-100, 100)), D))
        if k == 4:
            return ops.Call(abi.EX_GT, ops.Call(abi.EX_CAST_TO_DECIMAL, c0, result_dtype=(6, 2)), ops.Const(0, DEC, (6, 2)))
        return ops.Call(abi.EX_GT, ops.Call(abi.EX_MUL, c0, c3), ops.Const(rng.randrange(-10 ** 6, 10 ** 6), DEC, (25, 4)))
    op = rng.choice([abi.EX_AND, abi.EX_OR, abi.EX_AND, abi.EX_NOT])
    if op == abi.EX_NOT:
        return ops.Call(op, _random_tree(rng, depth - 1))
    return ops.Call(op, _random_tree(rng, depth - 1), _random_tree(rng, depth - 1))


def test_random_trees_raise_where_the_reference_evaluates(ctx):
    rng = random.Random(2024)
    n = 400
    rows = []
    for i in range(n):
        rows.append([None if rng.random() < 0.1 else rng.randrange(-10 ** 6, 10 ** 6),
                     None if rng.random() < 0.1 else rng.randrange(-10 ** 25, 10 ** 25),
                     None if rng.random() < 0.1 else rng.choice([0, 5, -7, 2 ** 62, rng.randrange(-1000, 1000)]),
                     None if rng.random() < 0.1 else rng.choice([0, 1, -3, 250, rng.randrange(-10 ** 5, 10 ** 5)])])
    page_of = lambda idx: Page(Block.bigint([0 if rows[i][0] is None else rows[i][0] for i in idx], [rows[i][0] is None for i in idx]),
                               Block.int128([rows[i][1] for i in idx]),
                               Block.bigint([0 if rows[i][2] is None else rows[i][2] for i in idx], [rows[i][2] is None for i in idx]),
                               Block.bigint([0 if rows[i][3] is None else rows[i][3] for i in idx], [rows[i][3] is None for i in idx]))
    raised_any = 0
    for t in range(12):
        tree = _random_tree(rng, 2)
        # up to 3 / 4 / 5 leaves: at most 8 temporaries
        try:
            prog = ops.PageProcessorProgram(tree, [2])
        except ValueError:
            continue
        want, errs = [], []
        for r in rows:
            try:
                v = _eval(tree, r)
                want.append(v)
            except _Err as x:
                errs.append(x.status)
        if errs:
            raised_any += 1
            with pytest.raises(abi.TrinoGpuError) as exc:
                _run(ctx, prog, [page_of(range(n))])
            assert exc.value.code == min(errs, key=lambda s: PRIORITY[s])
            continue
        out = _run(ctx, prog, [page_of(range(n))])
        got = out[0].get_block(0).to_pylist() if out else []
        assert got == [r[2] for r, w in zip(rows, want) if w]
    assert raised_any > 0


# ---- refusals through the create entry points ---------------------------------------------------------------------------------------
def test_pre_stage_and_filtered_build_refuse_decimal(ctx):
    c0 = ops.Col(1, DEC, (12, 2))
    pre = ops.PageProcessorProgram(ops.Call(abi.EX_GT, c0, ops.Const(5, DEC, (12, 2))), [0, 1])
    with pytest.raises(abi.TrinoGpuError) as exc:
        ops.HashAggregationOperatorFactory(ctx, [0], abi.STEP_SINGLE, [ops.Aggregator(abi.AGG_COUNT_STAR)], 16, pre=pre).create_operator()
    assert exc.value.code == abi.ERR_NOT_SUPPORTED
    with pytest.raises(abi.TrinoGpuError) as exc:
        ops.AggregationOperatorFactory(ctx, abi.STEP_SINGLE, [ops.Aggregator(abi.AGG_COUNT_STAR)], pre=pre,
                                       input_types=[abi.INT64, abi.INT64]).create_operator()
    assert exc.value.code == abi.ERR_NOT_SUPPORTED
    jf = ops.PageProcessorProgram(ops.Call(abi.EX_GT, ops.Col(0, DEC, (12, 2)), ops.Col(2, DEC, (12, 2))), [])
    spec = abi.JoinBuildSpec()
    keys = (C.c_int32 * 1)(1)
    outs = (C.c_int32 * 2)(0, 1)
    spec.num_key_channels, spec.key_channels = 1, C.cast(keys, C.POINTER(C.c_int32))
    spec.num_output_channels, spec.output_channels = 2, C.cast(outs, C.POINTER(C.c_int32))
    spec.expected_positions = 16
    h = C.c_void_p()
    st = ctx.lib.tgpu_join_build_create_filtered(ctx.h, C.byref(spec), C.byref(jf.struct), 2, C.byref(h))
    assert st == abi.ERR_NOT_SUPPORTED
