"""LookupJoinOperator with a join filter function (HashBuilderOperatorFactory's filterFunctionFactory) on the GPU.

The filter reads the join-sources layout: build channels 0 .. nb-1 at the build position, then the probe channels at the probe row
(LocalExecutionPlanner.compileJoinFilterFunction).  A NULL or FALSE result makes a position ineligible (JoinHash.isJoinPositionEligible).
PageJoiner walks each probe row's chain in position-link order, appends the eligible positions, stops at the first eligible one under
outputSingleMatch, and emits the NULL-build row of an outer join when none was eligible; the LOOKUP_OUTER / FULL_OUTER page holds the
build rows never appended.

The exact reference: the oracle's join positions and position links, a chain walk here, and expr_reference.evaluate on
build_row + probe_row.  Probe pages draw their rows from a pool, so the reference evaluates each (pool row, candidate) pair once.
Every output row is identified by a probe row-id channel and a build row-id channel and checked in order, for every join type and
both outputSingleMatch settings.  Errors must be raised exactly where the reference evaluates: every candidate of a chain, or under
outputSingleMatch those up to the first eligible one.

test_interpreter_form_in_child_process runs the file again with TGPU_DISABLE_JIT=1: the interpreter kernels.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import expr_cases as ec
import expr_reference as ref
import oracle_lib as o
from trino_b200 import abi
from trino_b200 import operators as ops
from trino_b200.page import Block, Page

pytestmark = pytest.mark.gpu
B, D, BOOL = abi.V_BIGINT, abi.V_DOUBLE, abi.V_BOOLEAN
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NO_JIT = bool(os.environ.get("TGPU_DISABLE_JIT"))
JOIN_TYPES = (abi.JOIN_INNER, abi.JOIN_PROBE_OUTER, abi.JOIN_LOOKUP_OUTER, abi.JOIN_FULL_OUTER)
OUTER = (abi.JOIN_PROBE_OUTER, abi.JOIN_FULL_OUTER)
TRACKING = (abi.JOIN_LOOKUP_OUTER, abi.JOIN_FULL_OUTER)


# ---- running the operators ----------------------------------------------------------------------------------------------------
def run_join(ctx, build_pages, nb, bk, build_out, probe_pages, pk, probe_out, filt, join_type, single, by_reference=False, outer_types=None):
    """(output pages of the probe, pages of the LookupOuterOperator or None); raises TrinoGpuError from the probe"""
    bridge = ops.JoinBridge()
    bf = ops.HashBuilderOperatorFactory(ctx, bridge, bk, build_out, filter=filt, num_build_channels=nb)
    b = bf.create_operator()
    j = None
    try:
        for p in build_pages:
            b.add_input(p)
        b.finish()
        j = ops.LookupJoinOperatorFactory(ctx, bridge, join_type, single, pk, probe_out).create_operator()
        if by_reference:
            j.set_passthrough_by_reference(True)
        out = ops.drive(j, probe_pages)
        outer = None
        if join_type in TRACKING:
            op = ops.LookupOuterOperatorFactory(ctx, bridge, outer_types).create_operator()
            outer = ops.drive(op, [])
            op.close()
        return out, outer
    finally:
        if j is not None:
            j.close()
        b.close()
        if bridge.lookup_source is not None:
            bridge.lookup_source.close()


def column(pages, c):
    """values (int64, -1 where NULL) of output channel c over all pages"""
    vals = [np.where(p.blocks[c].nulls if p.blocks[c].nulls is not None else np.zeros(p.position_count, bool), -1,
                     p.blocks[c].values.astype(np.int64)) for p in pages]
    return np.concatenate(vals) if vals else np.zeros(0, np.int64)


# ---- the reference ------------------------------------------------------------------------------------------------------------
class Reference:
    """PageJoiner with a JoinFilterFunction over one build side and a pool of probe rows"""

    def __init__(self, build_page, bk, pool_page, pk, filt):
        j = o.Join(build_page, bk)
        self.heads = j.positions(pool_page, pk)
        self.links = j.links()
        j.close()
        self.build_rows = build_page.rows()
        self.pool_rows = pool_page.rows()
        self.filt = filt
        self.memo = {}

    def verdict(self, q, b):
        """(eligible, error code or None) of build position b for pool row q"""
        key = (q, b)
        if key not in self.memo:
            v, err = ref.try_evaluate(self.filt, self.build_rows[b] + self.pool_rows[q])
            self.memo[key] = (v is True, err)
        return self.memo[key]

    def row(self, q, join_type, single):
        """(build positions emitted for pool row q, -1 for the NULL-build row; error codes raised)"""
        out, errs = [], set()
        p = int(self.heads[q])
        while p >= 0:
            ok, err = self.verdict(q, p)
            if err is not None:
                errs.add(err)
            if ok:
                out.append(p)
                if single:
                    break
            p = int(self.links[p])
        if not out and join_type in OUTER:
            out.append(-1)
        return out, errs

    def expect(self, pages_idx, join_type, single):
        """per page: (probe pool rows, build positions) of the output, or the set of error codes of the first failing page"""
        per_q = {}
        result = []
        for idx in pages_idx:
            uq = np.unique(idx)
            errs = set()
            for q in uq.tolist():
                if q not in per_q:
                    per_q[q] = self.row(q, join_type, single)
                errs |= per_q[q][1]
            if errs:
                return result, errs
            lens = np.zeros(len(self.pool_rows), np.int64)
            starts = np.zeros(len(self.pool_rows), np.int64)
            flat = []
            at = 0
            for q in uq.tolist():
                lens[q] = len(per_q[q][0])
                starts[q] = at
                flat.extend(per_q[q][0])
                at += lens[q]
            flat = np.asarray(flat, np.int64)
            counts = lens[idx]
            total = int(counts.sum())
            first = np.repeat(np.cumsum(counts) - counts, counts)
            within = np.arange(total) - first
            b = flat[np.repeat(starts[idx], counts) + within] if total else np.zeros(0, np.int64)
            result.append((np.repeat(idx, counts), b))
        return result, None


# ---- cases ----------------------------------------------------------------------------------------------------------------------
# build layout: [key..., id INTEGER, a BIGINT, x DOUBLE, s SMALLINT, f BOOLEAN]; probe layout the same, the ids numbering pool rows
VALUE_TYPES = (abi.INT64, abi.FLOAT64, abi.INT16, "boolean")


def _values(rng, t, k, null_frac):
    if t == "boolean":
        v = rng.integers(0, 2, k)
    elif t == abi.FLOAT64:
        v = np.where(rng.random(k) < 0.1, rng.choice(np.array(ec.DOUBLE_EDGES), k), np.round(rng.normal(0, 40, k), 2))
    elif t == abi.INT16:
        v = rng.integers(-300, 300, k)
    else:
        v = np.where(rng.random(k) < 0.05, rng.choice(np.array(ec.BIGINT_EDGES, dtype=np.int64), k), rng.integers(-100, 100, k))
    return ec.Column(t, v, rng.random(k) < null_frac)


def _key_blocks(kind, keys, nulls):
    keys = np.asarray(keys, np.int64)
    if kind == "bigint":
        return [Block.bigint(keys, nulls)]
    if kind == "varchar":
        return [Block.varchar([None if n else f"k{k:06d}" for k, n in zip(keys.tolist(), nulls.tolist())])]
    # two channels: (k // 7, k % 7 as INTEGER); a NULL key is NULL in the first channel
    return [Block.bigint(keys // 7, nulls), Block.integer((keys % 7).astype(np.int32))]


class JoinCase:
    def __init__(self, name, seed, key_kind="bigint", build_rows=3000, dup=1, key_null=0.05, pay_null=0.2, skew=0, pool=2048,
                 sizes=(1, 1023, 1025, 4097)):
        rng = np.random.default_rng(seed)
        self.name, self.seed, self.key_kind = name, seed, key_kind
        domain = max(1, build_rows // dup)
        if dup == 1:
            bkeys = rng.permutation(domain)[:build_rows]
        else:
            bkeys = rng.integers(0, domain, build_rows)
        if skew:
            bkeys = np.concatenate([bkeys, np.full(skew, 7)])
            rng.shuffle(bkeys)
        nbuild = len(bkeys)
        bnull = rng.random(nbuild) < key_null
        pkeys = rng.integers(0, int(domain * 1.3) + 1, pool)
        if skew:
            pkeys[:4] = 7                      # four pool rows meet the >= 10 000-row chain
            pkeys[4:][pkeys[4:] == 7] = 8
        pnull = rng.random(pool) < key_null
        pnull[:4] = False
        self.nk = 1 if key_kind != "multi" else 2
        bvals = [_values(rng, t, nbuild, pay_null) for t in VALUE_TYPES]
        pvals = [_values(rng, t, pool, pay_null) for t in VALUE_TYPES]
        bblocks = _key_blocks(key_kind, bkeys, bnull) + [Block.integer(np.arange(nbuild, dtype=np.int32))] + [c.block(np.arange(nbuild)) for c in bvals]
        pblocks = _key_blocks(key_kind, pkeys, pnull) + [Block.integer(np.arange(pool, dtype=np.int32))] + [c.block(np.arange(pool)) for c in pvals]
        self.build = Page(*bblocks)
        self.pool = Page(*pblocks)
        self.nb = self.build.channel_count
        self.bk = self.pk = list(range(self.nk))
        self.id = self.nk                     # the id channel on both sides
        half = nbuild // 2                     # two build pages
        self.build_pages = [Page(*[b.get_positions(np.arange(0, half)) for b in bblocks]),
                            Page(*[b.get_positions(np.arange(half, nbuild)) for b in bblocks])]
        self.pages_idx = [rng.integers(0, pool, n) for n in sizes]
        by_vt = {B: [], D: [], BOOL: []}
        for side in (0, self.nb):
            for i, t in enumerate(VALUE_TYPES):
                by_vt[ec.VTYPE_OF[t]].append(side + self.id + 1 + i)
            by_vt[B].append(side + self.id)
        self.by_vt = by_vt
        self.rng = rng

    def probe_pages(self):
        return [Page(*[b.get_positions(idx) for b in self.pool.blocks]) for idx in self.pages_idx]

    def filters(self, n):
        """n seeded filter trees over the join-sources layout, each reading a build and a probe channel"""
        gen = ec.ProgramGen(self.rng, self.by_vt, {}, [self.id + 1, self.nb + self.id + 1])
        a_b, a_p = self.id + 1, self.nb + self.id + 1            # the BIGINT `a` of each side
        x_b, x_p = self.id + 2, self.nb + self.id + 2            # the DOUBLE `x` of each side
        s_b, s_p = self.id + 3, self.nb + self.id + 3            # the SMALLINT `s` of each side
        # three shapes that never raise (the fixed conjunct of the random trees), then random trees AND / OR one of them
        shapes = [
            ops.Call(abi.EX_LT, ops.Col(a_p, B), ops.Col(a_b, B)),
            ops.Call(abi.EX_BETWEEN, ops.Call(abi.EX_SUB, ops.Col(s_p, B), ops.Col(s_b, B)), ops.Const(-100, B), ops.Const(150, B)),
            ops.Call(abi.EX_OR, ops.Call(abi.EX_GT, ops.Col(x_p, D), ops.Call(abi.EX_MUL, ops.Const(0.2, D), ops.Col(x_b, D))),
                     ops.Call(abi.EX_IS_NULL, ops.Col(a_b, B))),
        ]
        out = []
        for i in range(n):
            base = shapes[i % len(shapes)]
            if i < len(shapes):
                out.append(base)
                continue
            while True:
                extra = gen.expr(BOOL, int(self.rng.integers(2, 5)))
                f = ops.Call(abi.EX_AND if i % 2 else abi.EX_OR, base, extra)
                try:
                    p = ops.PageProcessorProgram(f, [])
                except ValueError:
                    continue
                if len(p.insns) <= 64:
                    out.append(f)
                    break
        return out


def reference(case, filt):
    return Reference(case.build, case.bk, case.pool, case.pk, filt)


def check_case(ctx, case, r, join_type, single, by_reference=False):
    """one join of the case's probe pages against the reference r; returns "rows" or "error" (the reference raised)"""
    filt = r.filt
    pages = case.probe_pages()
    want, errs = r.expect(case.pages_idx, join_type, single)
    probe_out, build_out = [case.id, case.id + 2], [case.id, case.id + 1]
    what = f"{case.name} seed {case.seed} join {join_type} single {single}: {ec.show(filt)}"
    if errs:
        with pytest.raises(abi.TrinoGpuError) as exc:
            run_join(ctx, case.build_pages, case.nb, case.bk, build_out, pages, case.pk, probe_out, filt, join_type, single, by_reference,
                     [abi.INT32, abi.FLOAT64])
        assert exc.value.code in errs, (what, exc.value, errs)
        return "error"
    out, outer = run_join(ctx, case.build_pages, case.nb, case.bk, build_out, pages, case.pk, probe_out, filt, join_type, single, by_reference,
                          [abi.INT32, abi.FLOAT64])
    got_q, got_b = column(out, 0), column(out, 2)
    want_q = np.concatenate([w[0] for w in want]) if want else np.zeros(0, np.int64)
    want_b = np.concatenate([w[1] for w in want]) if want else np.zeros(0, np.int64)
    assert len(got_q) == len(want_q), (what, len(got_q), len(want_q))
    assert np.array_equal(got_q, want_q), what
    assert np.array_equal(got_b, want_b), what
    # the build payload of each row (a nullable BIGINT), and the probe DOUBLE that travels with it
    bpay = case.build.blocks[case.id + 1]
    bvals = np.where(bpay.nulls if bpay.nulls is not None else False, -1, bpay.values.astype(np.int64))
    assert np.array_equal(column(out, 3), np.where(want_b >= 0, bvals[np.maximum(want_b, 0)], -1)), what
    px = case.pool.blocks[case.id + 2]
    got_x = np.concatenate([p.blocks[1].values for p in out]) if out else np.zeros(0)
    xnull = np.concatenate([p.blocks[1].nulls if p.blocks[1].nulls is not None else np.zeros(p.position_count, bool) for p in out]) if out else np.zeros(0, bool)
    want_xnull = px.nulls[want_q] if px.nulls is not None else np.zeros(len(want_q), bool)
    assert np.array_equal(xnull, want_xnull), what
    assert np.array_equal(got_x[~xnull].view(np.int64), px.values[want_q][~want_xnull].view(np.int64)), what
    if join_type in TRACKING:
        visited = set(want_b[want_b >= 0].tolist())
        want_outer = [b for b in range(case.build.position_count) if b not in visited]
        got_outer = column(outer, 2).tolist()
        assert got_outer == want_outer, what
        assert all(v == -1 for v in column(outer, 0).tolist()), what
    return "rows"


CASES = [
    dict(name="unique bigint", seed=11, dup=1),
    dict(name="duplicate bigint", seed=12, dup=4),
    dict(name="duplicate varchar", seed=13, key_kind="varchar", dup=3),
    dict(name="unique multi-channel", seed=14, key_kind="multi", dup=1),
    dict(name="duplicate multi-channel", seed=15, key_kind="multi", dup=2),
    dict(name="skewed bigint", seed=16, dup=2, build_rows=2000, skew=10_000, sizes=(1025, 4097)),
]


@pytest.mark.parametrize("spec", CASES, ids=[c["name"] for c in CASES])
def test_against_exact_reference(ctx, spec):
    case = JoinCase(**spec)
    outcomes = {"rows": 0, "error": 0}
    for filt in case.filters(6):
        r = reference(case, filt)
        for join_type in JOIN_TYPES:
            for single in (False, True):
                outcomes[check_case(ctx, case, r, join_type, single)] += 1
    assert outcomes["rows"] >= 24, outcomes          # the three fixed shapes never raise


def test_one_million_row_page(ctx):
    case = JoinCase("big page", 21, dup=3, sizes=(1_000_003, 1000))
    r = reference(case, case.filters(2)[1])
    for join_type in JOIN_TYPES:
        assert check_case(ctx, case, r, join_type, False) == "rows"
    assert check_case(ctx, case, r, abi.JOIN_PROBE_OUTER, True) == "rows"


@pytest.mark.parametrize("dup", [1, 3])
def test_by_reference_probe_filters_on_a_non_key_channel(ctx, dup):
    case = JoinCase("by reference", 31 + dup, dup=dup)
    r = reference(case, case.filters(2)[1])          # reads the probe's `s`, which is neither key nor output channel
    for join_type in (abi.JOIN_INNER, abi.JOIN_PROBE_OUTER):
        for single in (False, True):
            assert check_case(ctx, case, r, join_type, single, by_reference=True) == "rows"


# ---- known answers (T/operator/join/unspilled/TestHashJoinOperator.java) -------------------------------------------------------
def _rows(pages):
    out = []
    for p in pages:
        out.extend(p.rows())
    return out


# probeOuterJoin(false): outputSingleMatch is false in all four
def test_probe_outer_join_with_filter_function(ctx):
    """testProbeOuterJoinWithFilterFunction (:533-586): probe channel 1 >= 1025; build (VARCHAR key, BIGINT, BIGINT)"""
    build = Page(Block.varchar([str(20 + i) for i in range(10)]), Block.bigint(np.arange(30, 40)), Block.bigint(np.arange(40, 50)))
    probe = Page(Block.varchar([str(20 + i) for i in range(15)]), Block.bigint(np.arange(1020, 1035)), Block.bigint(np.arange(2020, 2035)))
    filt = ops.Call(abi.EX_GE, ops.Col(3 + 1, B), ops.Const(1025, B))
    out, _ = run_join(ctx, [build], 3, [0], [0, 1, 2], [probe], [0], [0, 1, 2], filt, abi.JOIN_PROBE_OUTER, False)
    want = []
    for i in range(15):
        b = (str(20 + i).encode(), 30 + i, 40 + i) if 25 <= 20 + i <= 29 else (None, None, None)
        want.append((str(20 + i).encode(), 1020 + i, 2020 + i) + b)
    assert _rows(out) == want


def test_outer_join_with_null_probe_and_filter_function(ctx):
    """testOuterJoinWithNullProbeAndFilterFunction (:638-689): probe key = 1"""
    build = Page(Block.bigint([1, 2, 3]))
    probe = Page(Block.bigint([1, None, None, 1, 2]))
    filt = ops.Call(abi.EX_EQ, ops.Col(1, B), ops.Const(1, B))
    out, _ = run_join(ctx, [build], 1, [0], [0], [probe], [0], [0], filt, abi.JOIN_PROBE_OUTER, False)
    assert _rows(out) == [(1, 1), (None, None), (None, None), (1, 1), (2, None)]


def test_outer_join_with_null_build_and_filter_function(ctx):
    """testOuterJoinWithNullBuildAndFilterFunction (:740-791): probe key IN (1, 3)"""
    build = Page(Block.bigint([1, None, None, 1, 2]))
    probe = Page(Block.bigint([1, 2, 3]))
    filt = ops.Call(abi.EX_IN, ops.Col(1, B), in_list=[1, 3])
    out, _ = run_join(ctx, [build], 1, [0], [0], [probe], [0], [0], filt, abi.JOIN_PROBE_OUTER, False)
    assert _rows(out) == [(1, 1), (1, 1), (2, None), (3, None)]


def test_outer_join_with_null_on_both_sides_and_filter_function(ctx):
    """testOuterJoinWithNullOnBothSidesAndFilterFunction (:843-895)"""
    build = Page(Block.bigint([1, None, None, 1, 2]))
    probe = Page(Block.bigint([1, 2, None, 3]))
    filt = ops.Call(abi.EX_IN, ops.Col(1, B), in_list=[1, 3])
    out, _ = run_join(ctx, [build], 1, [0], [0], [probe], [0], [0], filt, abi.JOIN_PROBE_OUTER, False)
    assert _rows(out) == [(1, 1), (1, 1), (2, None), (None, None), (3, None)]


# ---- errors -----------------------------------------------------------------------------------------------------------------------
# build (key BIGINT, d BIGINT), probe (key BIGINT, v BIGINT); filter: v / d > 0, which raises DIVISION_BY_ZERO where d = 0
DIV = ops.Call(abi.EX_GT, ops.Call(abi.EX_DIV, ops.Col(3, B), ops.Col(1, B)), ops.Const(0, B))


def _div_join(ctx, build_keys, build_d, probe_keys, probe_v, join_type=abi.JOIN_INNER, single=False):
    build = Page(Block.bigint(build_keys), Block.bigint(build_d))
    probe = Page(Block.bigint(probe_keys), Block.bigint(probe_v))
    out, _ = run_join(ctx, [build], 2, [0], [1], [probe], [0], [1], DIV, join_type, single, outer_types=[abi.INT64])
    return _rows(out)


@pytest.mark.parametrize("join_type", JOIN_TYPES)
def test_errors_only_where_the_reference_evaluates(ctx, join_type):
    outer = join_type in OUTER
    # chain of key 1 in position-link order: row 1 (d = 5, eligible for v = 10), then row 0 (d = 0, raises)
    assert _div_join(ctx, [1, 1], [0, 5], [1], [10], join_type, single=True) == [(10, 5)]
    with pytest.raises(abi.TrinoGpuError) as exc:
        _div_join(ctx, [1, 1], [0, 5], [1], [10], join_type, single=False)
    assert exc.value.code == abi.ERR_DIVISION_BY_ZERO
    # the first candidate is not eligible (10 / 50 = 0): the second one is evaluated and raises, even under outputSingleMatch
    with pytest.raises(abi.TrinoGpuError) as exc:
        _div_join(ctx, [1, 1], [0, 50], [1], [10], join_type, single=True)
    assert exc.value.code == abi.ERR_DIVISION_BY_ZERO
    # a NULL probe key has no candidates; a build row with a NULL key is nobody's candidate
    assert _div_join(ctx, [1, None, 1], [0, 0, 5], [None], [10], join_type) == ([(10, None)] if outer else [])
    # no position links: the one candidate raises, a probe key without a match evaluates nothing
    with pytest.raises(abi.TrinoGpuError) as exc:
        _div_join(ctx, [1, 2], [0, 5], [1], [10], join_type)
    assert exc.value.code == abi.ERR_DIVISION_BY_ZERO
    assert _div_join(ctx, [1, 2], [0, 5], [3, 2], [10, 10], join_type) == ([(10, None), (10, 5)] if outer else [(10, 5)])


def test_overflow_in_a_long_chain(ctx):
    """one of 5000 candidates overflows (v * d): raised with NUMERIC_VALUE_OUT_OF_RANGE, and not under outputSingleMatch when an
    eligible candidate comes first"""
    n = 5000
    d = np.full(n, 2, np.int64)
    d[0] = 1 << 62                    # last in position-link order
    filt = ops.Call(abi.EX_GT, ops.Call(abi.EX_MUL, ops.Col(3, B), ops.Col(1, B)), ops.Const(0, B))
    build = Page(Block.bigint(np.ones(n, np.int64)), Block.bigint(d))
    probe = Page(Block.bigint([1]), Block.bigint([4]))
    with pytest.raises(abi.TrinoGpuError) as exc:
        run_join(ctx, [build], 2, [0], [1], [probe], [0], [1], filt, abi.JOIN_INNER, False)
    assert exc.value.code == abi.ERR_NUMERIC_VALUE_OUT_OF_RANGE
    out, _ = run_join(ctx, [build], 2, [0], [1], [probe], [0], [1], filt, abi.JOIN_INNER, True)
    assert _rows(out) == [(4, 2)]


# ---- arguments ----------------------------------------------------------------------------------------------------------------------
def _create(ctx, prog, nb, keys=(0,), outs=(1,)):
    kc, oc = (C.c_int32 * len(keys))(*keys), (C.c_int32 * max(1, len(outs)))(*outs)
    spec = abi.JoinBuildSpec(len(keys), C.cast(kc, C.POINTER(C.c_int32)), len(outs), C.cast(oc, C.POINTER(C.c_int32)), 100)
    h = C.c_void_p()
    st = ctx.lib.tgpu_join_build_create_filtered(ctx.h, C.byref(spec), C.byref(prog.struct), nb, C.byref(h))
    if st == 0:
        ctx.lib.tgpu_op_close(h)
    return st


def test_invalid_arguments(ctx):
    good = ops.PageProcessorProgram(ops.Call(abi.EX_LT, ops.Col(1, B), ops.Col(3, B)), [])
    assert _create(ctx, good, 2) == 0
    assert _create(ctx, good, -1) == abi.ERR_INVALID_ARGUMENT
    assert _create(ctx, ops.PageProcessorProgram(ops.Call(abi.EX_LT, ops.Col(1, B), ops.Col(3, B)), [0]), 2) == abi.ERR_INVALID_ARGUMENT
    no_filter = ops.PageProcessorProgram(None, [ops.Call(abi.EX_ADD, ops.Col(1, B), ops.Const(1, B))])
    no_filter.struct.num_projections = 0
    assert _create(ctx, no_filter, 2) == abi.ERR_INVALID_ARGUMENT
    build = Page(Block.bigint([1, 2]), Block.bigint([3, 4]))
    probe = Page(Block.bigint([1, 2]), Block.bigint([3, 4]))
    # the build page is not the layout the filter was given
    with pytest.raises(abi.TrinoGpuError) as exc:
        run_join(ctx, [build], 3, [0], [1], [probe], [0], [1], ops.Call(abi.EX_LT, ops.Col(1, B), ops.Col(3, B)), abi.JOIN_INNER, False)
    assert exc.value.code == abi.ERR_INVALID_ARGUMENT
    # a probe channel the probe page does not have
    with pytest.raises(abi.TrinoGpuError) as exc:
        run_join(ctx, [build], 2, [0], [1], [probe], [0], [1], ops.Call(abi.EX_LT, ops.Col(1, B), ops.Col(5, B)), abi.JOIN_INNER, False)
    assert exc.value.code == abi.ERR_INVALID_ARGUMENT


@pytest.mark.parametrize("side", ["build", "probe"])
@pytest.mark.parametrize("kind", ["varchar", "real", "int128"])
def test_not_supported_channel_types(ctx, side, kind):
    odd = {"varchar": Block.varchar(["a", "b"]), "real": Block.real(np.array([1.0, 2.0], np.float32)), "int128": Block.int128([1, 2])}[kind]
    build = Page(Block.bigint([1, 2]), odd if side == "build" else Block.bigint([3, 4]))
    probe = Page(Block.bigint([1, 2]), odd if side == "probe" else Block.bigint([3, 4]))
    ch = 1 if side == "build" else 3
    filt = ops.Call(abi.EX_IS_NOT_NULL, ops.Col(ch, B))
    with pytest.raises(abi.TrinoGpuError) as exc:
        run_join(ctx, [build], 2, [0], [0], [probe], [0], [0], filt, abi.JOIN_INNER, False)
    assert exc.value.code == abi.ERR_NOT_SUPPORTED


def test_filtered_lookup_keeps_positions_and_refuses_a_semi_join(ctx):
    keys = np.array([5, 1, 5, 9, None], dtype=object)
    build = Page(Block.bigint(list(keys)), Block.bigint([1, 2, 3, 4, 5]))
    bridge = ops.JoinBridge()
    b = ops.HashBuilderOperatorFactory(ctx, bridge, [0], [1], filter=ops.Call(abi.EX_LT, ops.Col(1, B), ops.Col(3, B)),
                                       num_build_channels=2).create_operator()
    b.add_input(build)
    b.finish()
    lk = bridge.lookup_source
    try:
        probe_keys = Page(Block.bigint([5, 1, 2, 9, None]))
        j = o.Join(build, [0])
        assert lk.get_join_positions(probe_keys).tolist() == j.positions(probe_keys, [0]).tolist()
        assert lk.position_links().tolist() == j.links().tolist()
        j.close()
        lo, hi, cnt, values, has_null = lk.key_domain(16)
        assert (lo, hi, cnt, values.tolist(), has_null) == (1, 9, 3, [1, 5, 9], True)
        with pytest.raises(abi.TrinoGpuError) as exc:
            ops.HashSemiJoinOperatorFactory(ctx, bridge, 0).create_operator()
        assert exc.value.code == abi.ERR_INVALID_ARGUMENT
    finally:
        b.close()
        lk.close()


def test_unfiltered_factory_is_unchanged(ctx):
    """no filter: the plain entry point, and the same rows as the oracle"""
    from helpers import oracle_join_rows
    build = Page(Block.bigint([1, 2, 2, 3]), Block.bigint([10, 20, 21, 30]))
    probe = Page(Block.bigint([2, 3, 4]), Block.bigint([7, 8, 9]))
    assert ops.HashBuilderOperatorFactory(ctx, ops.JoinBridge(), [0], [1]).filter_program is None
    out, _ = run_join(ctx, [build], 2, [0], [1], [probe], [0], [1], None, abi.JOIN_INNER, False)
    assert _rows(out) == oracle_join_rows(build, probe, 0, 0, [1], [1], abi.JOIN_INNER, False)


# ---- the interpreter kernels --------------------------------------------------------------------------------------------------------
def test_interpreter_form_in_child_process():
    """join_filter_positions_kernel / join_filter_pairs_kernel run where NVRTC is missing; the choice is made once per process"""
    if NO_JIT:
        pytest.skip("already the child")
    env = dict(os.environ, TGPU_DISABLE_JIT="1")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", "-p", "no:cacheprovider", os.path.abspath(__file__)],
                       cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-6000:]
    assert " passed" in r.stdout and "1 skipped" in r.stdout, r.stdout[-2000:]

