"""AggregationOperator (aggregation without GROUP BY keys) on the GPU: the reference's TestAggregationOperator restated, the one-row
contract over empty input in every step, TPC-H Q6 against the oracle's left fold, every function over every supported argument type,
PARTIAL -> FINAL, errors, seeded pre-stage programs, and the launch count of a page.

test_interpreter_forms_in_child_process runs the file again in a process started with TGPU_DISABLE_JIT=1 (agg_global_kernel)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import expr_cases as ec
import oracle_lib as o
from helpers import oracle_agg_rows, rows_equal
from q1 import q1_host_page
from q6 import INPUT_TYPES, q6_factory, q6_oracle
from trino_b200 import abi
from trino_b200 import operators as ops
from trino_b200.page import Block, Page

pytestmark = pytest.mark.gpu
A = ops.Aggregator
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NO_JIT = bool(os.environ.get("TGPU_DISABLE_JIT"))


def _run(factory, pages):
    """drive one operator through the AggregationOperator protocol; -> its one output Page"""
    op = factory.create_operator()
    for p in pages:
        assert op.needs_input()
        op.add_input(p)
        assert op.get_output() is None            # nothing before finish()
    assert op.needs_input()
    op.finish()
    assert not op.needs_input()
    out = op.get_output()
    assert out is not None and out.position_count == 1
    assert op.is_finished()
    assert op.get_output() is None
    op.close()
    return out


def _row(factory, pages):
    return _run(factory, pages).rows()[0]


def _factory(ctx, step, aggs, types, pre=None, row_typed=False):
    return ops.AggregationOperatorFactory(ctx, step, aggs, pre=pre, input_types=types, row_typed_states=row_typed)


# ---- TestAggregationOperator ------------------------------------------------------------------------------------------------
def test_aggregation_operator_known_answers(ctx):
    """testAggregation (T/operator/TestAggregationOperator.java:148-180), the supported subset: count(*), sum and avg over BIGINT
    0..99, sum over BIGINT 500..599 and over DOUBLE 500..599"""
    seq = np.arange(100, dtype=np.int64)
    page = Page(Block.bigint(seq), Block.bigint(500 + seq), Block.double((500 + seq).astype(np.float64)))
    types = [abi.INT64, abi.INT64, abi.FLOAT64]
    row = _row(_factory(ctx, abi.STEP_SINGLE, [A(abi.AGG_COUNT_STAR), A(abi.AGG_SUM, 0), A(abi.AGG_AVG, 0), A(abi.AGG_SUM, 1), A(abi.AGG_SUM, 2)], types), [page])
    assert row == (100, 4950, 49.5, 54950, 54950.0)


@pytest.mark.parametrize("fn,type_", [(abi.AGG_SUM, abi.FLOAT32), (abi.AGG_MAX, abi.UTF8), (abi.AGG_COUNT, abi.UTF8)])
def test_real_and_varchar_arguments_are_not_supported(ctx, fn, type_):
    # the REAL sum and the VARCHAR max / count of testAggregation stay on the Java operator, as on the keyed operator
    with pytest.raises(abi.TrinoGpuError) as e:
        _factory(ctx, abi.STEP_SINGLE, [A(fn, 0)], [type_]).create_operator()
    assert e.value.code == abi.ERR_NOT_SUPPORTED


def test_long_decimal_min_max_and_fused_wide_pre_stage_are_not_supported(ctx):
    for f, pre in (([A(abi.AGG_MAX, 0)], None), ([A(abi.AGG_SUM, 0)], ops.PageProcessorProgram(None, [1]))):
        with pytest.raises(abi.TrinoGpuError) as e:
            _factory(ctx, abi.STEP_SINGLE, f, [abi.INT128, abi.INT64], pre=pre).create_operator()
        assert e.value.code == abi.ERR_NOT_SUPPORTED


def test_spec_fields_of_the_keyed_operator_are_rejected(ctx):
    lib = ctx.lib
    fns = (abi.AggFn * 1)()
    fns[0].function, fns[0].input_channel, fns[0].mask_channel = abi.AGG_COUNT_STAR, -1, -1
    types = (C.c_int32 * 1)(abi.INT64)
    keys = (C.c_int32 * 1)(0)
    base = dict(num_keys=0, step=abi.STEP_SINGLE, num_aggs=1, aggs=C.cast(fns, C.POINTER(abi.AggFn)), group_id_key=-1, num_input_channels=1,
                input_channel_types=C.cast(types, C.POINTER(C.c_int32)))
    for bad in (dict(num_keys=1, key_channels=C.cast(keys, C.POINTER(C.c_int32))), dict(max_partial_bytes=1 << 20), dict(group_id_key=0),
                dict(num_global_group_ids=1, global_group_ids=C.cast(keys, C.POINTER(C.c_int32)))):
        spec = abi.AggSpec(**{**base, **bad})
        h = C.c_void_p()
        assert lib.tgpu_aggregation_create(ctx.h, C.byref(spec), C.byref(h)) == abi.ERR_INVALID_ARGUMENT
    # HashAggregationOperator is never planned without keys: the keyed entry point keeps answering NOT_SUPPORTED at the first page
    f = ops.HashAggregationOperatorFactory(ctx, [], abi.STEP_SINGLE, [A(abi.AGG_COUNT_STAR)])
    op = f.create_operator()
    with pytest.raises(abi.TrinoGpuError) as e:
        op.add_input(Page(Block.bigint(np.arange(3))))
    assert e.value.code == abi.ERR_NOT_SUPPORTED
    op.close()


def test_mask_with_dirty_nulls(ctx):
    """testMaskWithDirtyNulls (:88-113): a NULL mask position whose value byte is non-zero does not count"""
    mask = Block.boolean(np.array([1, 1], dtype=np.int8), np.array([False, True]))
    page = Page(Block.bigint(np.array([1, 2], dtype=np.int64)), mask)
    assert _row(_factory(ctx, abi.STEP_SINGLE, [A(abi.AGG_COUNT, 0, 1)], [abi.INT64, abi.INT8]), [page]) == (1,)


def test_memory_tracking(ctx):
    """testMemoryTracking (:182-207): the operator reports memory once it holds input, and close() releases it"""
    op = _factory(ctx, abi.STEP_SINGLE, [A(abi.AGG_SUM, 0)], [abi.INT64]).create_operator()
    op.add_input(Page(Block.bigint(np.arange(100, dtype=np.int64))))
    assert op.memory_bytes() > 0
    op.close()
    assert op.h is None


# ---- empty input ----------------------------------------------------------------------------------------------------------------
RAW_TYPES = [abi.INT64, abi.FLOAT64, abi.INT64]          # bigint, double, short decimal
RAW_AGGS = [A(abi.AGG_COUNT_STAR), A(abi.AGG_COUNT, 0), A(abi.AGG_SUM, 0), A(abi.AGG_SUM, 1), A(abi.AGG_AVG, 0), A(abi.AGG_MIN, 0), A(abi.AGG_MAX, 1),
            A(abi.AGG_SUM_DECIMAL, 2)]
# state channels of RAW_AGGS: count(*), count, sum(bigint), sum(double), avg (count, sum), min, max, decimal sum (sum, overflow)
STATE_TYPES = [abi.INT64, abi.INT64, abi.INT64, abi.FLOAT64, abi.INT64, abi.FLOAT64, abi.INT64, abi.FLOAT64, abi.INT128, abi.INT64]
STATE_AGGS = [A(abi.AGG_COUNT_STAR, 0), A(abi.AGG_COUNT, 1), A(abi.AGG_SUM, 2), A(abi.AGG_SUM, 3), A(abi.AGG_AVG, 4), A(abi.AGG_MIN, 6), A(abi.AGG_MAX, 7),
              A(abi.AGG_SUM_DECIMAL, 8)]
FINAL_EMPTY = (0, 0, None, None, None, None, None, None)
STATE_EMPTY = (0, 0, None, None, 0, 0.0, None, None, None, 0)


def _empty_pages(types):
    make = {abi.INT64: lambda: Block.bigint(np.zeros(0, dtype=np.int64)), abi.FLOAT64: lambda: Block.double(np.zeros(0)), abi.INT128: lambda: Block.int128([])}
    blocks = [make[t]() for t in types]
    return [Page(*blocks, position_count=0), Page(*blocks, position_count=0)]


@pytest.mark.parametrize("step,aggs,types,expected", [(abi.STEP_SINGLE, RAW_AGGS, RAW_TYPES, FINAL_EMPTY), (abi.STEP_PARTIAL, RAW_AGGS, RAW_TYPES, STATE_EMPTY),
                                                       (abi.STEP_FINAL, STATE_AGGS, STATE_TYPES, FINAL_EMPTY),
                                                       (abi.STEP_INTERMEDIATE, STATE_AGGS, STATE_TYPES, STATE_EMPTY)])
@pytest.mark.parametrize("zero_row_pages", [False, True])
def test_empty_input_gives_one_row(ctx, step, aggs, types, expected, zero_row_pages):
    pages = _empty_pages(types) if zero_row_pages else []
    assert _row(_factory(ctx, step, aggs, types), pages) == expected


# ---- TPC-H Q6 -------------------------------------------------------------------------------------------------------------------
def _q6_cols(n):
    return o.synth_lineitem_q1(n, 0, 0x7C01)


def _check_q6(got, cols, **kw):
    rev, cnt = q6_oracle(cols, **kw)
    assert got[1] == cnt
    if rev is None:
        assert got[0] is None
    else:
        assert abs(got[0] - rev) <= 1e-6 * abs(rev), (got, rev)


@pytest.mark.parametrize("n", [1_000_000, 2_000_003])
@pytest.mark.parametrize("page_rows", [None, 8192])
def test_q6_matches_the_oracle(ctx, n, page_rows):
    cols = _q6_cols(n)
    page_rows = page_rows or n
    pages = [q1_host_page(cols, lo, min(n, lo + page_rows)) for lo in range(0, n, page_rows)]
    got = _row(q6_factory(ctx), pages)
    _check_q6(got, cols)
    assert _row(q6_factory(ctx), pages) == got             # bit-identical on a second run over the same pages


@pytest.mark.parametrize("n,page_rows", [(50_001, 7), (3_001, 1)])
def test_q6_tiny_pages(ctx, n, page_rows):
    # (the Q6 window holds ~1.8 % of the rows: widen it so that tiny pages select something)
    cols = _q6_cols(n)
    pages = [q1_host_page(cols, lo, min(n, lo + page_rows)) for lo in range(0, n, page_rows)]
    _check_q6(_row(q6_factory(ctx, 0, 20000), pages), cols, ship_lo=0, ship_hi=20000)


def test_q6_selects_nothing_and_everything(ctx):
    cols = _q6_cols(1_000_000)
    page = q1_host_page(cols)
    assert _row(q6_factory(ctx, 9131, 8766), [page]) == (None, 0)
    # a filter every row passes, and the same projection
    D = abi.V_DOUBLE
    prog = ops.PageProcessorProgram(ops.Call(abi.EX_GE, ops.Col(0, abi.V_BIGINT), ops.Const(-(1 << 31), abi.V_BIGINT)),
                                    [ops.Call(abi.EX_MUL, ops.Col(4, D), ops.Col(5, D))])
    got = _row(ops.AggregationOperatorFactory(ctx, abi.STEP_SINGLE, [A(abi.AGG_SUM, 0), A(abi.AGG_COUNT_STAR)], pre=prog, input_types=INPUT_TYPES), [page])
    want = oracle_agg_rows([Page(Block.bigint(np.zeros(1_000_000, dtype=np.int64)), Block.double(cols["extendedprice"] * cols["discount"]))], [0],
                           [(abi.AGG_SUM, 1, -1), (abi.AGG_COUNT_STAR, -1, -1)])[0]
    assert got[1] == 1_000_000 and abs(got[0] - want[1]) <= 1e-6 * abs(want[1])


def _device_q6_page(ctx, cols, offset, keep):
    specs = [("shipdate", abi.INT32), ("returnflag", abi.INT8), ("linestatus", abi.INT8), ("quantity", abi.FLOAT64), ("extendedprice", abi.FLOAT64),
             ("discount", abi.FLOAT64), ("tax", abi.FLOAT64)]
    n = len(cols["shipdate"]) - offset
    dcols = []
    for name, t in specs:
        arr = np.ascontiguousarray(cols[name])
        p = ctx.to_device(arr)
        keep.append(p)
        dcols.append(ops.DeviceColumn(t, p + offset * arr.itemsize, n))
    return ops.DevicePage(dcols, n)


@pytest.mark.parametrize("offset", [0, 1])
def test_q6_device_columns(ctx, offset):
    """device-resident columns; sliced at a 1-row offset they are not 16-byte aligned and take the scalar loader"""
    n = 1_000_003
    cols = _q6_cols(n)
    keep = []
    page = _device_q6_page(ctx, cols, offset, keep)
    got = _row(q6_factory(ctx), [page])
    _check_q6(got, {k: v[offset:] for k, v in cols.items()})
    for p in keep:
        ctx.free(p)


def test_q6_page_costs_the_kernel_and_the_fold(ctx):
    cols = _q6_cols(1 << 20)
    keep = []
    page = _device_q6_page(ctx, cols, 0, keep)
    op = q6_factory(ctx).create_operator()
    op.add_input(page)                    # (the first page compiles the kernel)
    before = ctx.kernel_launches
    op.add_input(page)
    assert ctx.kernel_launches - before == 2
    op.finish()
    got = op.get_output().rows()[0]
    op.close()
    rev, cnt = q6_oracle(cols)
    assert got[1] == 2 * cnt
    for p in keep:
        ctx.free(p)


# ---- every function x argument type x NULLs x mask ---------------------------------------------------------------------------
_TYPED = {abi.INT64: (Block.bigint, np.int64, -(1 << 40), 1 << 40), abi.INT32: (Block.integer, np.int32, -(1 << 30), 1 << 30),
          abi.INT16: (Block.smallint, np.int16, -30000, 30000), abi.INT8: (Block.tinyint, np.int8, -120, 120)}


def _typed_pages(rng, type_, null_mode, n=20_000, pages=3):
    out = []
    for _ in range(pages):
        nulls = {"none": None, "some": rng.random(n) < 0.3, "all": np.ones(n, dtype=bool)}[null_mode]
        if type_ == abi.FLOAT64:
            v = Block.double(np.round(rng.normal(0, 1000, n), 3), nulls)
        else:
            mk, dt, lo, hi = _TYPED[type_]
            v = mk(rng.integers(lo, hi, n).astype(dt), nulls)
        mask = Block.boolean((rng.random(n) < 0.6).astype(np.int8), rng.random(n) < 0.1)
        out.append(Page(v, mask))
    return out


@pytest.mark.parametrize("type_", [abi.INT64, abi.INT32, abi.INT16, abi.INT8, abi.FLOAT64])
@pytest.mark.parametrize("null_mode", ["none", "some", "all"])
def test_every_function_against_the_oracle(ctx, type_, null_mode):
    rng = np.random.default_rng(type_ * 10 + ["none", "some", "all"].index(null_mode))
    pages = _typed_pages(rng, type_, null_mode)
    fns = [abi.AGG_COUNT_STAR, abi.AGG_COUNT, abi.AGG_SUM, abi.AGG_AVG, abi.AGG_MIN, abi.AGG_MAX]
    for mask in (-1, 1):
        aggs = [A(f, -1 if f == abi.AGG_COUNT_STAR else 0, mask) for f in fns]
        got = _row(_factory(ctx, abi.STEP_SINGLE, aggs, [type_, abi.INT8]), pages)
        keyed = [Page(Block.bigint(np.zeros(p.position_count, dtype=np.int64)), *p.blocks) for p in pages]
        want = list(oracle_agg_rows(keyed, [0], [(f, -1 if f == abi.AGG_COUNT_STAR else 1, 2 if mask >= 0 else -1) for f in fns])[0][1:])
        if mask >= 0:
            # (oracle_agg_rows applies no mask to min / max: take them from the masked values directly)
            on = np.concatenate([(p.blocks[1].values != 0) & ~p.blocks[1].nulls & (~p.blocks[0].nulls if p.blocks[0].nulls is not None else True) for p in pages])
            vals = np.concatenate([p.blocks[0].values for p in pages])[on]
            conv = float if type_ == abi.FLOAT64 else int
            want[4] = conv(vals.min()) if len(vals) else None
            want[5] = conv(vals.max()) if len(vals) else None
        assert rows_equal([got], [tuple(want)], rel=1e-6), (mask, got, want)


@pytest.mark.parametrize("wide", [False, True])
@pytest.mark.parametrize("null_mode", ["none", "some", "all"])
def test_decimal_sum_against_the_oracle(ctx, wide, null_mode):
    rng = np.random.default_rng(7 + wide)
    n = 10_000
    vals = [int(x) * (10 ** 20 if wide else 1) for x in rng.integers(-(1 << 50), 1 << 50, n)]
    nulls = {"none": np.zeros(n, bool), "some": rng.random(n) < 0.3, "all": np.ones(n, bool)}[null_mode]
    if wide:
        blk = Block.int128(vals, nulls if nulls.any() else None)
    else:
        blk = Block.bigint(np.array(vals, dtype=np.int64), nulls if nulls.any() else None)
    for mask in (-1, 1):
        sel = ~nulls
        mvals = (rng.random(n) < 0.5).astype(np.int8)
        if mask >= 0:
            sel = sel & (mvals != 0)
        page = Page(blk, Block.boolean(mvals))
        got = _row(_factory(ctx, abi.STEP_SINGLE, [A(abi.AGG_SUM_DECIMAL, 0, mask), A(abi.AGG_COUNT, 0, mask)], [abi.INT128 if wide else abi.INT64, abi.INT8]), [page])
        st = o.DecimalSumState().add([v for v, s in zip(vals, sel) if s], short=not wide)
        assert got[1] == int(sel.sum())
        assert got[0] == (st.value if sel.any() else None), (got, st.value)


# ---- PARTIAL -> FINAL ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("row_typed", [False, True])
def test_partial_then_final_equals_single(ctx, row_typed):
    rng = np.random.default_rng(11)
    chunks = []
    for k in range(5):
        n = 0 if k in (1, 3) else 30_000 + k
        nulls = rng.random(n) < 0.2
        chunks.append([Page(Block.bigint(rng.integers(-1000, 1000, n), nulls), Block.double(np.round(rng.normal(0, 10, n), 2)),
                            Block.bigint(rng.integers(-(1 << 40), 1 << 40, n)), position_count=n)] if n else [])
    single = _row(_factory(ctx, abi.STEP_SINGLE, RAW_AGGS, RAW_TYPES), [p for c in chunks for p in c])
    partial_f = _factory(ctx, abi.STEP_PARTIAL, RAW_AGGS, RAW_TYPES, row_typed=row_typed)
    states = [_run(partial_f.duplicate() if k else partial_f, c) for k, c in enumerate(chunks)]
    if row_typed:
        # the Java plan numbers one channel per state: count(*), count, sum, sum, avg ROW, min, max, decimal VARBINARY
        aggs = [A(abi.AGG_COUNT_STAR, 0), A(abi.AGG_COUNT, 1), A(abi.AGG_SUM, 2), A(abi.AGG_SUM, 3), A(abi.AGG_AVG, 4), A(abi.AGG_MIN, 5), A(abi.AGG_MAX, 6),
                A(abi.AGG_SUM_DECIMAL, 7)]
        assert states[0].channel_count == 8
    else:
        aggs = STATE_AGGS
    final = _row(_factory(ctx, abi.STEP_FINAL, aggs, STATE_TYPES, row_typed=row_typed), states)
    assert rows_equal([final], [single], rel=1e-9), (final, single)


# ---- errors -------------------------------------------------------------------------------------------------------------------
def _code(fn):
    try:
        fn()
    except abi.TrinoGpuError as e:
        return e.code
    return 0


def test_overflow_behaves_as_the_keyed_operator(ctx):
    big = np.full(4, 1 << 62, dtype=np.int64)
    wide = [10 ** 38 - 1, 10 ** 38 - 1]        # DECIMAL(38) maximum twice
    for aggs, types, page in (([A(abi.AGG_SUM, 0)], [abi.INT64], Page(Block.bigint(big))),
                              ([A(abi.AGG_SUM_DECIMAL, 0)], [abi.INT128], Page(Block.int128(wide)))):
        glob = _code(lambda: _row(_factory(ctx, abi.STEP_SINGLE, aggs, types), [page]))
        keyed_page = Page(Block.bigint(np.zeros(page.position_count, dtype=np.int64)), *page.blocks)
        keyed_aggs = [A(a.function, a.input_channel + 1) for a in aggs]
        keyed = _code(lambda: ops.drive(ops.HashAggregationOperatorFactory(ctx, [0], abi.STEP_SINGLE, keyed_aggs, 16).create_operator(), [keyed_page]))
        assert glob == keyed == abi.ERR_NUMERIC_VALUE_OUT_OF_RANGE


def test_division_by_zero_only_where_trino_evaluates(ctx):
    B = abi.V_BIGINT
    x, y = ops.Col(0, B), ops.Col(1, B)
    page = Page(Block.bigint(np.array([0, 2, 0], dtype=np.int64)), Block.bigint(np.array([5, 10, 7], dtype=np.int64)))
    # a projection the aggregation reads raises
    prog = ops.PageProcessorProgram(None, [ops.Call(abi.EX_DIV, y, x)])
    assert _code(lambda: _row(_factory(ctx, abi.STEP_SINGLE, [A(abi.AGG_SUM, 0)], [abi.INT64, abi.INT64], pre=prog), [page])) == abi.ERR_DIVISION_BY_ZERO
    # x <> 0 AND y / x > 2: the division is never evaluated where x = 0
    flt = ops.Call(abi.EX_AND, ops.Call(abi.EX_NE, x, ops.Const(0, B)), ops.Call(abi.EX_GT, ops.Call(abi.EX_DIV, y, x), ops.Const(2, B)))
    prog = ops.PageProcessorProgram(flt, [1])
    assert _row(_factory(ctx, abi.STEP_SINGLE, [A(abi.AGG_SUM, 0), A(abi.AGG_COUNT_STAR)], [abi.INT64, abi.INT64], pre=prog), [page]) == (10, 1)


# ---- seeded pre-stage programs ------------------------------------------------------------------------------------------------
def _case_expected(case, idx, read):
    """(count, {projection: (sum or None, overflow?, count)}, error codes) of one page through the reference evaluator"""
    if case.filt is not None:
        fv, fe = case.evaluate(case.filt)
        errs = {fe[i] for i in idx.tolist() if fe[i] is not None}
        if errs:
            return None, None, errs
        sel = [i for i in idx.tolist() if fv[i] is True]
    else:
        sel = idx.tolist()
    out, errs = {}, set()
    for p in read:
        pv, pe = case.evaluate(case.projs[p])
        errs |= {pe[i] for i in sel if pe[i] is not None}
        vals = [pv[i] for i in sel if pv[i] is not None]
        out[p] = vals
    return len(sel), out, errs


@pytest.mark.parametrize("seed", range(48))
def test_seeded_pre_stage_programs(ctx, seed):
    case = ec.random_case(5000 + seed, {}, sizes=[1025, 7])
    types = [abi.INT8 if c.type == "boolean" else c.type for c in case.columns[:case.varchar]]
    prog = ops.PageProcessorProgram(case.filt, case.projs)
    big = [i for i, p in enumerate(case.projs) if p.vtype == abi.V_BIGINT]
    dbl = [i for i, p in enumerate(case.projs) if p.vtype == abi.V_DOUBLE]
    # sum / min / max of the BIGINT projections, count of the DOUBLE ones, count(*)
    aggs = [A(abi.AGG_COUNT_STAR)] + [A(f, i) for i in big for f in (abi.AGG_SUM, abi.AGG_MIN, abi.AGG_MAX)] + [A(abi.AGG_COUNT, i) for i in dbl]
    count, sums, errs = 0, {i: [] for i in big + dbl}, set()
    for idx in case.pages:
        c, vals, e = _case_expected(case, idx, big + dbl)
        if e:
            errs |= e
            break
        count += c
        for i in vals:
            sums[i] += vals[i]
    pages = [case.page(idx) for idx in case.pages]
    f = _factory(ctx, abi.STEP_SINGLE, aggs, types, pre=prog)
    if errs:
        assert _code(lambda: _row(f, pages)) in errs, case.describe()
        return
    want = [count]
    overflow = False
    for i in big:
        s = sum(sums[i])
        overflow |= not (-(1 << 63) <= s < (1 << 63))
        want += [s if sums[i] else None, min(sums[i]) if sums[i] else None, max(sums[i]) if sums[i] else None]
    want += [len(sums[i]) for i in dbl]
    if overflow:
        assert _code(lambda: _row(f, pages)) == abi.ERR_NUMERIC_VALUE_OUT_OF_RANGE, case.describe()
        return
    assert _row(f, pages) == tuple(want), case.describe()


# ---- the interpreter kernels --------------------------------------------------------------------------------------------------
def test_interpreter_forms_in_child_process():
    """agg_global_kernel runs where NVRTC is missing: no other test reaches it, because the choice is made once per process"""
    if NO_JIT:
        pytest.skip("already the child")
    env = dict(os.environ, TGPU_DISABLE_JIT="1")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", "-p", "no:cacheprovider", "-k", "not seeded_pre_stage",
                        os.path.abspath(__file__)], cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-6000:]
    assert " passed" in r.stdout and "1 skipped" in r.stdout, r.stdout[-2000:]
