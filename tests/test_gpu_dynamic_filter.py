"""GPU parity of the DynamicPageFilter operator (csrc/dynfilter.cu) against the oracle and the reference's own cases
(T/sql/gen/TestDynamicPageFilter.java), including the EffectiveFilterProfiler switching filters off."""
import numpy as np
import pytest

import oracle_lib as o
from test_oracle_dynamic_filter import df, golden_cases
from trino_b200 import operators as ops
from trino_b200.page import Block, Page

pytestmark = pytest.mark.gpu


def _gpu_domain(d):
    return ops.ColumnDomain(d.channel, d.kind, d.null_allowed, d.lo, d.hi, None if d.values is None else d.values.tolist())


def _page(columns):
    return Page(*[Block.bigint(v, n) for v, n in columns])


def _selected_rows(op, page):
    op.add_input(page)
    out = op.get_output()
    return [] if out is None else out.rows()


def test_reference_cases(ctx):
    for name, domains, threshold, pages, expected in golden_cases():
        op = ops.DynamicFilterOperatorFactory(ctx, [_gpu_domain(d) for d in domains], threshold).create_operator()
        ev = df.DynamicFilterEvaluator(domains, threshold)
        for columns, want in zip(pages, expected):
            page = _page(columns)
            rows = _selected_rows(op, page)
            sel = ev.evaluate(columns)
            all_rows = page.rows()
            assert rows == [all_rows[i] for i in sel], name
            assert len(rows) == (want if isinstance(want, int) else len(want)), name
        op.close()


def test_random_pages_and_updates_match_oracle(ctx):
    rng = np.random.default_rng(3)
    domains = [df.Domain(0, df.DISCRETE, True, values=rng.integers(0, 2000, 300).tolist()), df.Domain(2, df.RANGE, False, lo=-100, hi=700),
               df.Domain(1, df.ALL, True)]
    op = ops.DynamicFilterOperatorFactory(ctx, [_gpu_domain(d) for d in domains], 0.8).create_operator()
    ev = df.DynamicFilterEvaluator(domains, 0.8)
    for n in (5000, 1, 70000, 3000):
        columns = [(rng.integers(0, 2000, n), rng.random(n) < 0.05), (rng.integers(-5, 5, n), None), (rng.integers(-500, 1500, n), rng.random(n) < 0.02)]
        page = Page(Block.bigint(*columns[0]), Block.integer(columns[1][0].astype(np.int32)), Block.smallint(columns[2][0].astype(np.int16), columns[2][1]))
        rows = _selected_rows(op, page)
        sel = ev.evaluate(columns)
        all_rows = page.rows()
        assert rows == [all_rows[i] for i in sel]
        assert [op.is_effective(i) for i in range(3)] == [not x for x in ev.ineffective]
    # the dynamic filter narrows (testDynamicFilterUpdates :263-305): a new predicate, a fresh profiler
    narrowed = [df.Domain(0, df.DISCRETE, False, values=[7, 8, 9])]
    op.update([_gpu_domain(d) for d in narrowed])
    ev = df.DynamicFilterEvaluator(narrowed, 0.8)
    columns = [(rng.integers(0, 20, 4000), None), (np.zeros(4000, dtype=np.int64), None), (np.zeros(4000, dtype=np.int64), None)]
    page = _page(columns)
    assert _selected_rows(op, page) == [page.rows()[i] for i in ev.evaluate(columns)]
    op.close()


def test_all_none_and_build_side_domain(ctx):
    page = Page(Block.bigint([1, None, 3]), Block.double([0.5, 1.5, None]))
    op = ops.DynamicFilterOperatorFactory(ctx, []).create_operator()           # TupleDomain.all(): testAllPageFilter :85-93
    assert _selected_rows(op, page) == page.rows()
    op.close()
    op = ops.DynamicFilterOperatorFactory(ctx, [ops.ColumnDomain.none(0)]).create_operator()    # TupleDomain.none(): testNonePageFilter :95-103
    assert _selected_rows(op, page) == []
    op.close()
    op = ops.DynamicFilterOperatorFactory(ctx, [ops.ColumnDomain.double_range(1, 0.0, 1.0)]).create_operator()
    assert _selected_rows(op, page) == [(1, 0.5)]                              # DOUBLE range by value, NULL rejected
    op.close()
    # end to end: the build side's key domain (tgpu_lookup_key_domain) prunes the probe page before the join
    bridge = ops.JoinBridge()
    b = ops.HashBuilderOperatorFactory(ctx, bridge, [0], []).create_operator()
    keys = np.array([10, 20, 30, 40], dtype=np.int64)
    b.add_input(Page(Block.bigint(keys)))
    b.finish()
    lo, hi, distinct, values, has_null = bridge.lookup_source.key_domain(16)
    assert (lo, hi, distinct, sorted(values.tolist())) == (10, 40, 4, [10, 20, 30, 40])
    op = ops.DynamicFilterOperatorFactory(ctx, [ops.ColumnDomain.multiple_values(0, values.tolist())]).create_operator()
    probe = Page(Block.bigint(np.arange(0, 50)))
    assert [r[0] for r in _selected_rows(op, probe)] == [10, 20, 30, 40]
    op.close(); b.close(); bridge.lookup_source.close()
