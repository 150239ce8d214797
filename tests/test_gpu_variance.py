"""var_samp, var_pop, stddev_samp and stddev_pop in AggregationOperator on the GPU, against the exact variance of the input doubles
(tests/variance_reference.py): every argument type, with and without a NULL-bearing mask, over every data family of
tests/variance_families.py; PARTIAL -> FINAL and PARTIAL -> INTERMEDIATE -> FINAL, flat and ROW-typed states; empty input; a fused
pre-stage; run-to-run bit identity.  HashAggregationOperator: every device form a variance plan reaches (path S at L = 4..32, the
S -> G spill, the multipass path G with table growth, DOUBLE keys), checked against exact per group and with the profiler; PARTIAL
flushes; skipped partial aggregation, whose per-row states are compared bit for bit; grouping-set default rows.

test_interpreter_forms_in_child_process runs the file again with TGPU_DISABLE_JIT=1 (agg_global_kernel)."""
import math
import os
import struct
import subprocess
import sys
import zlib

import numpy as np
import pytest

import variance_families as fam
import variance_reference as vr
from trino_b200 import abi
from trino_b200 import operators as ops
from trino_b200.page import Block, Page

pytestmark = pytest.mark.gpu
A = ops.Aggregator
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NO_JIT = bool(os.environ.get("TGPU_DISABLE_JIT"))
VAR_FNS = (abi.AGG_VAR_SAMP, abi.AGG_VAR_POP, abi.AGG_STDDEV_SAMP, abi.AGG_STDDEV_POP)
MAKE = {abi.INT64: Block.bigint, abi.INT32: Block.integer, abi.INT16: Block.smallint, abi.INT8: Block.tinyint, abi.FLOAT64: Block.double}
NP = {abi.INT64: np.int64, abi.INT32: np.int32, abi.INT16: np.int16, abi.INT8: np.int8, abi.FLOAT64: np.float64}
LIMIT = {abi.INT64: 1 << 40, abi.INT32: 1 << 30, abi.INT16: 1 << 14, abi.INT8: 100}


def _run(factory, pages):
    op = factory.create_operator()
    for p in pages:
        op.add_input(p)
    op.finish()
    out = op.get_output()
    assert out is not None and out.position_count == 1
    op.close()
    return out


def _row(factory, pages):
    return _run(factory, pages).rows()[0]


def _factory(ctx, step, aggs, types, pre=None, row_typed=False):
    return ops.AggregationOperatorFactory(ctx, step, aggs, pre=pre, input_types=types, row_typed_states=row_typed)


def _values_for(type_, vals):
    """a family's values as the argument type sees them: integers are rounded into the type's range (NaN / Inf have no integer form)"""
    if type_ == abi.FLOAT64:
        return vals
    out = []
    for v in vals:
        if v is None or not math.isfinite(v):
            out.append(None if v is None else 0)
        else:
            out.append(int(max(-LIMIT[type_], min(LIMIT[type_], round(v)))))
    return out


def _pages(type_, vals, masked, rng, page_rows=1500):
    """[argument, BOOLEAN mask] pages; the mask drops about a third of the rows and is NULL on some (NULL drops the row too)"""
    pages, kept = [], []
    for s in range(0, max(len(vals), 1), page_rows):
        chunk = vals[s:s + page_rows]
        n = len(chunk)
        nulls = np.array([v is None for v in chunk], dtype=bool)
        data = np.array([0 if v is None else v for v in chunk], dtype=NP[type_])
        m = rng.random(n) < 0.67
        mnull = rng.random(n) < 0.1
        mask = Block.boolean(m.astype(np.int8), mnull if masked else None)
        pages.append(Page(MAKE[type_](data, nulls), mask, position_count=n))
        for i, v in enumerate(chunk):
            if not masked or (m[i] and not mnull[i]):
                kept.append(v)
    return pages, kept


def _check(got, vals):
    want = vr.expected(vals)
    for g, w in zip(got, want):
        assert vr.close(g, w), (got, want)


FAMILY_TYPES = [(name, t) for name in sorted(fam.FAMILIES) for t in (abi.FLOAT64, abi.INT64, abi.INT32, abi.INT16, abi.INT8)
                if t == abi.FLOAT64 or name not in ("large_mean", "nonfinite", "outlier_first")]


@pytest.mark.parametrize("name,type_", FAMILY_TYPES)
@pytest.mark.parametrize("masked", [False, True])
def test_single_step_against_exact(ctx, name, type_, masked):
    rng = np.random.default_rng(7)
    for group in fam.FAMILIES[name](0):
        vals = _values_for(type_, group)
        pages, kept = _pages(type_, vals, masked, rng)
        mask = 1 if masked else -1
        got = _row(_factory(ctx, abi.STEP_SINGLE, [A(f, 0, mask) for f in VAR_FNS], [type_, abi.INT8]), pages)
        _check(got, [None if v is None else float(v) for v in kept])


def test_constant_groups_are_exactly_zero_in_every_split(ctx):
    """a group of identical values: m2 stays +0.0 through every thread, warp, CTA and page merge"""
    for n in (1 << 20, 3 * (1 << 20) + 17):
        page = Page(Block.double(np.full(n, 1e9 + 0.1)), Block.boolean(np.ones(n, dtype=np.int8)))
        got = _row(_factory(ctx, abi.STEP_SINGLE, [A(f, 0) for f in VAR_FNS], [abi.FLOAT64, abi.INT8]), [page, page])
        assert got == (0.0, 0.0, 0.0, 0.0)
        assert all(math.copysign(1.0, g) == 1.0 for g in got)


def test_large_mean_over_many_ctas(ctx):
    """1e9 + k/1024 over 2^22 rows (thousands of CTA partials): the naive sum of squares would be off by orders of magnitude"""
    rng = np.random.default_rng(3)
    k = rng.integers(0, 4096, 1 << 22)
    x = 1e9 + k / 1024
    got = _row(_factory(ctx, abi.STEP_SINGLE, [A(f, 0) for f in VAR_FNS], [abi.FLOAT64]), [Page(Block.double(x))])
    # exact over the integers k: var(x) = var(k) / 1024^2
    from fractions import Fraction
    n = len(k)
    s1, s2 = int(k.sum()), int((k.astype(object) ** 2).sum())
    m2 = Fraction(s2) - Fraction(s1 * s1, n)
    want = (float(m2 / (n - 1) / 1024 ** 2), float(m2 / n / 1024 ** 2))
    assert vr.close(got[0], want[0]) and vr.close(got[1], want[1]), (got, want)
    assert vr.close(got[2], math.sqrt(want[0])) and vr.close(got[3], math.sqrt(want[1]))


@pytest.mark.parametrize("type_", [abi.FLOAT64, abi.INT64])
@pytest.mark.parametrize("row_typed", [False, True])
def test_partial_intermediate_final(ctx, type_, row_typed):
    rng = np.random.default_rng(5)
    vals = _values_for(type_, fam.well_conditioned(40_000, 2))
    vals = [None if rng.random() < 0.1 else v for v in vals]
    chunks = [vals[:10_000], [], vals[10_000:10_001], vals[10_001:]]
    raw = [abi.FLOAT64 if type_ == abi.FLOAT64 else abi.INT64, abi.INT8]
    aggs = [A(f, 0) for f in VAR_FNS]
    partial = _factory(ctx, abi.STEP_PARTIAL, aggs, raw, row_typed=row_typed)
    states = [_run(partial.duplicate(), _pages(type_, c, False, rng)[0] if c else []) for c in chunks]
    st_types = [abi.INT64, abi.FLOAT64, abi.FLOAT64] * 4
    if row_typed:
        assert states[0].channel_count == 4
        st_aggs = [A(f, i) for i, f in enumerate(VAR_FNS)]
    else:
        assert states[0].channel_count == 12
        st_aggs = [A(f, 3 * i) for i, f in enumerate(VAR_FNS)]
    inter = _factory(ctx, abi.STEP_INTERMEDIATE, st_aggs, st_types, row_typed=row_typed)
    mids = [_run(inter.duplicate(), states[:2]), _run(inter.duplicate(), states[2:])]
    final = _row(_factory(ctx, abi.STEP_FINAL, st_aggs, st_types, row_typed=row_typed), mids)
    _check(final, [None if v is None else float(v) for v in vals])


def test_partial_state_layout(ctx):
    """ROW(count, m2, mean): one PARTIAL over 1, 2, 6 gives (3, 14.0, 3.0); over nothing (0, 0.0, 0.0)"""
    f = _factory(ctx, abi.STEP_PARTIAL, [A(abi.AGG_VAR_POP, 0)], [abi.FLOAT64])
    assert _row(f, [Page(Block.double(np.array([1.0, 2.0, 6.0])))]) == (3, 14.0, 3.0)
    assert _row(f, []) == (0, 0.0, 0.0)
    s = _row(f, [Page(Block.double(np.array([5.0, 1.0])))])
    assert s == (2, 8.0, 3.0)


@pytest.mark.parametrize("step", [abi.STEP_SINGLE, abi.STEP_FINAL])
def test_empty_input_is_null(ctx, step):
    types = [abi.FLOAT64] if step == abi.STEP_SINGLE else [abi.INT64, abi.FLOAT64, abi.FLOAT64]
    assert _row(_factory(ctx, step, [A(f, 0) for f in VAR_FNS], types), []) == (None,) * 4


def test_one_row_gives_null_sample_and_zero_population(ctx):
    got = _row(_factory(ctx, abi.STEP_SINGLE, [A(f, 0) for f in VAR_FNS], [abi.INT32]), [Page(Block.integer(np.array([-5], dtype=np.int32)))])
    assert got == (None, 0.0, None, 0.0)


def test_fused_pre_stage(ctx):
    """var_pop(a * b) and stddev_samp(c) over the rows where a < 50, the projection evaluated in the aggregation kernel"""
    rng = np.random.default_rng(9)
    n = 300_000
    a, b, c = rng.uniform(0, 100, n), rng.uniform(-1, 1, n), rng.integers(-1000, 1000, n)
    X = ops
    prog = X.PageProcessorProgram(X.Call(abi.EX_LT, X.Col(0, abi.V_DOUBLE), X.Const(50.0, abi.V_DOUBLE)),
                                  [X.Call(abi.EX_MUL, X.Col(0, abi.V_DOUBLE), X.Col(1, abi.V_DOUBLE)), X.Col(2, abi.V_BIGINT)])
    page = Page(Block.double(a), Block.double(b), Block.bigint(c))
    got = _row(_factory(ctx, abi.STEP_SINGLE, [A(abi.AGG_VAR_POP, 0), A(abi.AGG_STDDEV_SAMP, 1)], [abi.FLOAT64, abi.FLOAT64, abi.INT64], pre=prog), [page])
    keep = a < 50
    assert vr.close(got[0], vr.exact(list(a[keep] * b[keep]))[1])
    assert vr.close(got[1], vr.exact([float(v) for v in c[keep]])[2])


def test_runs_are_bit_identical(ctx):
    rng = np.random.default_rng(1)
    pages = [Page(Block.double(rng.normal(3.0, 2.0, 1 << 21))), Page(Block.double(rng.normal(-1.0, 5.0, 777_777)))]
    f = _factory(ctx, abi.STEP_SINGLE, [A(f, 0) for f in VAR_FNS], [abi.FLOAT64])
    r1, r2 = _row(f, pages), _row(f.duplicate(), pages)
    assert [struct.pack("<d", x) for x in r1] == [struct.pack("<d", x) for x in r2]


@pytest.mark.parametrize("type_", [abi.FLOAT32, abi.UTF8, abi.INT128])
def test_real_varchar_and_long_decimal_are_not_supported(ctx, type_):
    with pytest.raises(abi.TrinoGpuError) as e:
        _factory(ctx, abi.STEP_SINGLE, [A(abi.AGG_STDDEV_SAMP, 0)], [type_]).create_operator()
    assert e.value.code == abi.ERR_NOT_SUPPORTED


def test_interpreter_forms_in_child_process():
    """agg_global_kernel runs where NVRTC is missing: the choice is made once per process"""
    if NO_JIT:
        pytest.skip("already the child")
    env = dict(os.environ, TGPU_DISABLE_JIT="1")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", "-p", "no:cacheprovider", os.path.abspath(__file__)],
                       cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-6000:]
    # (skipped in the child: this test and the profiler checks of the specialised kernels)
    assert " passed" in r.stdout and " failed" not in r.stdout, r.stdout[-2000:]


# ---- HashAggregationOperator ----------------------------------------------------------------------------------------------------
def _drain(op, out):
    while True:
        o = op.get_output()
        if o is None:
            return
        out.append(o)


def _hash_run(f, pages):
    op = f.create_operator()
    outs = []
    for p in pages:
        op.add_input(p)
        _drain(op, outs)
    op.finish()
    while not op.is_finished():
        _drain(op, outs)
    skipped = op.rows_with_partial_aggregation_disabled()
    op.close()
    return outs, skipped


def _grouped_pages(rng, key_sets, type_=abi.FLOAT64, family="well", page_rows=4000):
    """[BIGINT key, argument, BOOLEAN mask with NULLs] pages; key_sets: the distinct keys each page draws from"""
    pages, rows = [], []
    for keys in key_sets:
        n = page_rows
        k = rng.choice(np.array(keys, dtype=np.int64), n)
        if family == "large_mean":
            v = 1e9 + rng.integers(0, 4096, n) / 1024
        else:
            v = rng.normal(50.0, 20.0, n)
        v = v if type_ == abi.FLOAT64 else np.clip(np.round(v), -100, 100)
        vn = rng.random(n) < 0.05
        m, mn = rng.random(n) < 0.7, rng.random(n) < 0.1
        pages.append(Page(Block.bigint(k), MAKE[type_](v.astype(NP[type_]), vn), Block.boolean(m.astype(np.int8), mn)))
        rows += [(int(k[i]), None if vn[i] else float(v[i]), bool(m[i] and not mn[i])) for i in range(n)]
    return pages, rows


def _expect_groups(rows, masked):
    groups = {}
    for k, v, on in rows:
        groups.setdefault(k, [])
        if not masked or on:
            groups[k].append(v)
    return {k: vr.expected(vs) for k, vs in groups.items()}


def _check_groups(outs, want):
    got = {}
    for o in outs:
        for r in o.rows():
            assert r[0] not in got
            got[r[0]] = r[1:]
    assert set(got) == set(want)
    for k, w in want.items():
        for g, e in zip(got[k], w):
            assert vr.close(g, e), (k, got[k], w)


# key sets: 3 / 7 / 15 / 30 keys take path S at L = 4 / 8 / 16 / 32; "spill" adds 200 keys on the third page; "many" is 3000 keys with
# a small expected_groups (multipass path G with table growth)
KEYSETS = {"S_L4": [list(range(3))] * 3, "S_L8": [list(range(7))] * 3, "S_L16": [list(range(15))] * 3, "S_L32": [list(range(30))] * 3,
           "S_spill": [list(range(3)), list(range(3)), list(range(200))], "multipass_growth": [list(range(3000))] * 3}
KERNELS = {"S": ("tg_agg_small_jit", "agg_small_merge_kernel"), "G": ("g_insert_kernel", "g_accumulate_kernel", "var_pass_kernel", "var_page_merge_kernel")}


@pytest.mark.parametrize("form", sorted(KEYSETS))
@pytest.mark.parametrize("type_", [abi.FLOAT64, abi.INT64, abi.INT32, abi.INT16, abi.INT8])
@pytest.mark.parametrize("masked", [False, True])
def test_grouped_forms_against_exact(ctx, form, type_, masked):
    rng = np.random.default_rng(zlib.crc32(repr((form, type_, masked)).encode()))
    pages, rows = _grouped_pages(rng, KEYSETS[form], type_)
    mask = 2 if masked else -1
    f = ops.HashAggregationOperatorFactory(ctx, [0], abi.STEP_SINGLE, [A(fn, 1, mask) for fn in VAR_FNS], 16)
    outs, _ = _hash_run(f, pages)
    _check_groups(outs, _expect_groups(rows, masked))


@pytest.mark.parametrize("form", sorted(KEYSETS))
def test_grouped_forms_launch_their_kernels(ctx, form):
    if NO_JIT:
        pytest.skip("the interpreted kernels are checked by the results")
    from helpers import kernels_launched
    rng = np.random.default_rng(4)
    pages, rows = _grouped_pages(rng, KEYSETS[form], abi.FLOAT64, family="large_mean")
    f = ops.HashAggregationOperatorFactory(ctx, [0], abi.STEP_SINGLE, [A(fn, 1) for fn in VAR_FNS], 16)
    box = {}
    names = kernels_launched(lambda: box.update(outs=_hash_run(f, pages)[0]))
    _check_groups(box["outs"], _expect_groups(rows, False))
    assert names is not None
    joined = " ".join(names)
    want = KERNELS["S"] if form.startswith("S_L") else KERNELS["S"] + KERNELS["G"] if form == "S_spill" else KERNELS["G"]
    for k in want:
        assert k in joined, (form, k, sorted(set(names)))
    assert "tg_agg_general_jit" not in joined and "gf_page_kernel" not in joined      # never the fused record form
    if form.startswith("S_L"):
        assert "var_pass_kernel" not in joined


def test_double_keys_and_constant_groups(ctx):
    """DOUBLE keys take the multipass form by themselves; constant groups are exactly 0 on both paths"""
    for nkeys in (5, 500):
        n = 60_000
        rng = np.random.default_rng(nkeys)
        k = rng.integers(0, nkeys, n).astype(np.float64) / 4
        v = np.where(k < 1.0, 7.25, rng.normal(0, 1, n))
        f = ops.HashAggregationOperatorFactory(ctx, [0], abi.STEP_SINGLE, [A(fn, 1) for fn in VAR_FNS], 16)
        outs, _ = _hash_run(f, [Page(Block.double(k[:30_000]), Block.double(v[:30_000])), Page(Block.double(k[30_000:]), Block.double(v[30_000:]))])
        groups = {}
        for kk, vv in zip(k.tolist(), v.tolist()):
            groups.setdefault(kk, []).append(vv)
        _check_groups(outs, {kk: vr.expected(vs) for kk, vs in groups.items()})
        for o in outs:
            for r in o.rows():
                if r[0] < 1.0:
                    assert r[1:] == (0.0, 0.0, 0.0, 0.0)


@pytest.mark.parametrize("flush", [False, True])
def test_grouped_partial_intermediate_final(ctx, flush):
    """PARTIAL (with forced flushes at max_partial_bytes) -> INTERMEDIATE -> FINAL over 300 keys"""
    rng = np.random.default_rng(8)
    pages, rows = _grouped_pages(rng, [list(range(300))] * 4, abi.FLOAT64, family="large_mean")
    p = ops.HashAggregationOperatorFactory(ctx, [0], abi.STEP_PARTIAL, [A(fn, 1, 2) for fn in VAR_FNS], 16, max_partial_memory=1 if flush else 0)
    states, _ = _hash_run(p, pages)
    if flush:
        assert len(states) >= 2
    st_aggs = [A(fn, 1 + 3 * i) for i, fn in enumerate(VAR_FNS)]
    inter, _ = _hash_run(ops.HashAggregationOperatorFactory(ctx, [0], abi.STEP_INTERMEDIATE, st_aggs, 16), states)
    final, _ = _hash_run(ops.HashAggregationOperatorFactory(ctx, [0], abi.STEP_FINAL, st_aggs, 16), inter)
    _check_groups(final, _expect_groups(rows, True))


def _bits(x):
    if isinstance(x, float) and x != x:
        return "nan"
    return struct.pack("<q", x) if isinstance(x, int) else struct.pack("<d", x)


def _skip_state(v, on, is_double):
    """SkipAggregationBuilder: one Welford step from the empty state, in Python floats"""
    if not on or v is None:
        return (0, 0.0, 0.0)
    n, mean, m2 = vr.update((0, 0.0, 0.0), float(v))
    return (n, m2, mean)


@pytest.mark.parametrize("type_", [abi.FLOAT64, abi.INT32])
def test_skipped_builder_states_are_bit_exact(ctx, type_):
    n = 3000
    rng = np.random.default_rng(12)
    if type_ == abi.FLOAT64:
        v = rng.normal(0, 1e6, n)
        v[:6] = [-0.0, 0.0, float("inf"), float("-inf"), float("nan"), -3.5]
    else:
        v = rng.integers(-1 << 30, 1 << 30, n)
    vn = rng.random(n) < 0.1
    m, mn = rng.random(n) < 0.7, rng.random(n) < 0.1
    page = Page(Block.bigint(rng.integers(0, 50, n)), MAKE[type_](v.astype(NP[type_]), vn), Block.boolean(m.astype(np.int8), mn))
    controller = ops.PartialAggregationController(ctx.lib, 1 << 40, 0.0)
    controller.on_flush(1 << 41, 10, 10)
    assert controller.is_partial_aggregation_disabled()
    f = ops.HashAggregationOperatorFactory(ctx, [0], abi.STEP_PARTIAL, [A(abi.AGG_VAR_SAMP, 1), A(abi.AGG_STDDEV_POP, 1, 2)], 16,
                                           partial_aggregation_controller=controller)
    outs, skipped = _hash_run(f, [page])
    assert skipped == n and len(outs) == 1
    got = outs[0].rows()
    for i, r in enumerate(got):
        val = None if vn[i] else float(v[i])
        want = _skip_state(val, True, True) + _skip_state(val, bool(m[i] and not mn[i]), True)
        # bit for bit (so the mean of -0.0 must be +0.0); a NaN only has to be a NaN (the hardware's default NaN differs)
        assert [_bits(x) for x in r[1:]] == [_bits(x) for x in want], (i, r, want)
    controller.close()


def test_grouping_set_default_rows(ctx):
    """a global grouping set over empty input: one row, the $group_id key, NULL for every variance function"""
    f = ops.HashAggregationOperatorFactory(ctx, [0, 1], abi.STEP_SINGLE, [A(fn, 2) for fn in VAR_FNS], 16, global_aggregation_group_ids=(3,),
                                           group_id_channel=1, input_types=[abi.INT64, abi.INT64, abi.FLOAT64])
    outs, _ = _hash_run(f, [])
    assert [r for o in outs for r in o.rows()] == [(None, 3, None, None, None, None)]


def test_grouped_runs_on_path_s_are_bit_identical(ctx):
    rng = np.random.default_rng(2)
    pages, _ = _grouped_pages(rng, [list(range(7))] * 3, abi.FLOAT64, page_rows=400_000)
    f = ops.HashAggregationOperatorFactory(ctx, [0], abi.STEP_SINGLE, [A(fn, 1, 2) for fn in VAR_FNS], 16)
    a, b = _hash_run(f, pages)[0], _hash_run(f.duplicate(), pages)[0]
    ra, rb = [r for o in a for r in o.rows()], [r for o in b for r in o.rows()]
    assert [[struct.pack("<d", x) if isinstance(x, float) else x for x in r] for r in ra] == \
           [[struct.pack("<d", x) if isinstance(x, float) else x for x in r] for r in rb]
