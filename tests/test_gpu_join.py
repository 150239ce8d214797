"""GPU parity: HashBuilderOperator / LookupJoinOperator through the C ABI vs the CPU oracle (bit-exact rows and order)."""
import numpy as np
import pytest

import oracle_lib as o
from helpers import join_type_of, oracle_outer_rows, gpu_join_rows, oracle_join_rows, reference_cases, rows_equal
from trino_b200 import abi
from trino_b200 import operators as ops
from trino_b200.page import Block, DictionaryBlock, Page, RunLengthEncodedBlock

pytestmark = pytest.mark.gpu


def _build_lookup(ctx, build_pages, key=0, out=()):
    bridge = ops.JoinBridge()
    b = ops.HashBuilderOperatorFactory(ctx, bridge, [key], list(out)).create_operator()
    for p in build_pages:
        b.add_input(p)
    b.finish()
    return b, bridge.lookup_source


def test_reference_join_cases(ctx):
    for case in reference_cases()["join"]:
        build = Page(Block.bigint(case["build"])) if case["build"] else Page(Block.bigint([]), position_count=0)
        probe = Page(Block.bigint(case["probe"]))
        jt = join_type_of(case)
        rows = gpu_join_rows(ctx, [build], [probe], 0, 0, [0], [0], jt, case["single_match"])
        assert rows == [tuple(r) for r in case["expected"]], case["source"]


def test_probe_outer_sequence_case(ctx):
    c = reference_cases()["probe_outer_sequence"]
    b0, b1, b2 = c["build_initial"]
    p0, p1, p2 = c["probe_initial"]
    nb, npr = c["build_rows"], c["probe_rows"]
    build = Page(*[Block.bigint([x + i for i in range(nb)]) for x in (b0, b1, b2)])
    probe = Page(*[Block.bigint([x + i for i in range(npr)]) for x in (p0, p1, p2)])
    rows = gpu_join_rows(ctx, [build], [probe], 0, 0, [0, 1, 2], [0, 1, 2], abi.JOIN_PROBE_OUTER, False)
    want = oracle_join_rows(build, probe, 0, 0, [0, 1, 2], [0, 1, 2], abi.JOIN_PROBE_OUTER, False)
    assert rows == want
    assert rows[0] == (20, 1020, 2020, 20, 30, 40) and rows[-1] == (34, 1034, 2034, None, None, None)


@pytest.mark.parametrize("join_type,single", [(abi.JOIN_INNER, False), (abi.JOIN_PROBE_OUTER, False), (abi.JOIN_INNER, True), (abi.JOIN_PROBE_OUTER, True)])
def test_random_duplicates_and_nulls(ctx, join_type, single):
    rng = np.random.default_rng(42)
    nb, npr = 5000, 20000
    bk = rng.integers(0, 1500, nb)
    build = Page(Block.bigint(bk, rng.random(nb) < 0.05), Block.double(rng.normal(size=nb), rng.random(nb) < 0.1), Block.integer(rng.integers(-9, 9, nb)))
    pk = rng.integers(0, 2000, npr)
    probe = Page(Block.double(rng.normal(size=npr)), Block.bigint(pk, rng.random(npr) < 0.05), Block.varchar(["s%d" % (i % 13) if i % 11 else None for i in range(npr)]))
    got = gpu_join_rows(ctx, [build], [probe], 0, 1, [0, 1, 2], [1, 2], join_type, single)
    want = oracle_join_rows(build, probe, 0, 1, [0, 1, 2], [1, 2], join_type, single)
    assert rows_equal(got, want)


def test_multi_page_build_and_probe_pages(ctx):
    rng = np.random.default_rng(7)
    chunks = [rng.integers(0, 3000, n) for n in (1000, 1, 4096, 777)]
    build_pages = [Page(Block.bigint(c), Block.bigint(c * 10)) for c in chunks]
    whole = np.concatenate(chunks)
    build = Page(Block.bigint(whole), Block.bigint(whole * 10))
    probes = [Page(Block.bigint(rng.integers(0, 3500, n))) for n in (8192, 100, 1)]
    got = gpu_join_rows(ctx, build_pages, probes, 0, 0, [0], [0, 1], abi.JOIN_INNER, False)
    want = []
    for p in probes:
        want += oracle_join_rows(build, p, 0, 0, [0], [0, 1], abi.JOIN_INNER, False)
    assert got == want


def test_other_key_types_and_encodings(ctx):
    rng = np.random.default_rng(9)
    # INTEGER keys
    build = Page(Block.integer(rng.integers(-50, 50, 300)))
    probe = Page(Block.integer(rng.integers(-60, 60, 1000), rng.random(1000) < 0.1))
    assert gpu_join_rows(ctx, [build], [probe], 0, 0, [0], [0], abi.JOIN_INNER, False) == oracle_join_rows(build, probe, 0, 0, [0], [0], abi.JOIN_INNER, False)
    # DOUBLE keys: -0.0 == +0.0, NaN never matches
    build = Page(Block.double([0.0, 1.5, float("nan"), 2.5]))
    probe = Page(Block.double([-0.0, float("nan"), 1.5, 3.0]))
    got = gpu_join_rows(ctx, [build], [probe], 0, 0, [0], [0], abi.JOIN_PROBE_OUTER, False)
    want = oracle_join_rows(build, probe, 0, 0, [0], [0], abi.JOIN_PROBE_OUTER, False)
    assert rows_equal(got, want) and got[0][1] == 0.0 and got[1][1] is None
    # dictionary / RLE probe keys are values, not encodings (SURVEY Appendix B.5)
    build = Page(Block.bigint([10, 20, 30]))
    probe = Page(DictionaryBlock(Block.bigint([20, 99, 10]), [0, 1, 2, 2, 0]))
    assert gpu_join_rows(ctx, [build], [probe], 0, 0, [0], [0], abi.JOIN_INNER, False) == [(20, 20), (10, 10), (10, 10), (20, 20)]
    probe = Page(RunLengthEncodedBlock(Block.bigint([30]), 4))
    assert gpu_join_rows(ctx, [build], [probe], 0, 0, [0], [0], abi.JOIN_INNER, False) == [(30, 30)] * 4
    # the INT64_MIN key lives outside the table
    mn = -2**63
    build = Page(Block.bigint([mn, 5, mn]))
    probe = Page(Block.bigint([5, mn, 7]))
    assert gpu_join_rows(ctx, [build], [probe], 0, 0, [0], [0], abi.JOIN_INNER, False) == oracle_join_rows(build, probe, 0, 0, [0], [0], abi.JOIN_INNER, False)


def test_positions_and_links_match_oracle(ctx):
    rng = np.random.default_rng(3)
    bk = rng.integers(0, 40000, 100000)
    build = Page(Block.bigint(bk, rng.random(100000) < 0.01))
    b, lk = _build_lookup(ctx, [build])
    oj = o.Join(build, [0])
    probe = Page(Block.bigint(rng.integers(0, 50000, 300000), rng.random(300000) < 0.01))
    assert (lk.get_join_positions(probe) == oj.positions(probe, [0])).all()
    assert lk.has_position_links() and oj.has_links()
    assert (lk.position_links() == oj.links()).all()
    assert lk.get_join_position_count() == 100000
    oj.close(); b.close(); lk.close()


def test_synthetic_lineitem_orders_full_match(ctx):
    # configs[1] shape at 1/100 scale: every probe row finds its order; positions equal the oracle's
    n_orders = 1_500_000
    okeys = o.synth_orders_keys(n_orders, 0, n_orders, 0x7C02, True)
    rows = o.synth_lineitem_rows(n_orders)
    lkeys = o.synth_lineitem_keys(n_orders, 0, rows, 0x7C01, False)
    build = Page(Block.bigint(okeys))
    b, lk = _build_lookup(ctx, [build])
    pos = lk.get_join_positions(Page(Block.bigint(lkeys)))
    assert not lk.has_position_links()
    assert (pos >= 0).all()
    assert (okeys[pos] == lkeys).all()                      # size-independent property: matched build key == probe key
    oj = o.Join(build, [0], force_default=True)             # DefaultPagesHash is what the reference uses above 2^20 rows
    assert (pos[:2_000_000] == oj.positions(Page(Block.bigint(lkeys[:2_000_000])), [0])).all()
    oj.close(); b.close(); lk.close()


def test_operator_protocol(ctx):
    bridge = ops.JoinBridge()
    b = ops.HashBuilderOperatorFactory(ctx, bridge, [0], []).create_operator()
    assert b.needs_input() and not b.is_finished()
    b.add_input(Page(Block.bigint([1, 2])))
    b.finish(); b.finish()                                  # finish() is re-entrant (Driver.java:380-388)
    assert not b.needs_input() and b.is_finished()
    with pytest.raises(abi.TrinoGpuError) as e:
        b.add_input(Page(Block.bigint([3])))
    assert e.value.code == abi.ERR_ILLEGAL_STATE
    j = ops.LookupJoinOperatorFactory(ctx, bridge, abi.JOIN_INNER, False, [0], [0]).create_operator()
    assert j.needs_input() and j.get_output() is None
    j.add_input(Page(Block.bigint([2, 2, 9])))
    assert not j.needs_input()
    out = j.get_output()
    assert out.rows() == [(2,), (2,)]
    assert j.needs_input()
    j.finish()
    assert j.is_finished()
    j.close(); b.close(); bridge.lookup_source.close()


# ---------------------------------------------------------------- generic join keys (DefaultPagesHash shape)
def test_probe_outer_join_with_varchar_key_reference_case(ctx):
    # TestHashJoinOperator.testProbeOuterJoin :481-530 exactly as written there: VARCHAR join channel
    c = reference_cases()["probe_outer_sequence"]
    b0, b1, b2 = c["build_initial"]
    p0, p1, p2 = c["probe_initial"]
    nb, npr = c["build_rows"], c["probe_rows"]
    build = Page(Block.varchar([str(b0 + i) for i in range(nb)]), Block.bigint([b1 + i for i in range(nb)]), Block.bigint([b2 + i for i in range(nb)]))
    probe = Page(Block.varchar([str(p0 + i) for i in range(npr)]), Block.bigint([p1 + i for i in range(npr)]), Block.bigint([p2 + i for i in range(npr)]))
    rows = gpu_join_rows(ctx, [build], [probe], 0, 0, [0, 1, 2], [0, 1, 2], abi.JOIN_PROBE_OUTER, False)
    assert rows == oracle_join_rows(build, probe, 0, 0, [0, 1, 2], [0, 1, 2], abi.JOIN_PROBE_OUTER, False)
    assert rows[0] == (b"20", 1020, 2020, b"20", 30, 40) and rows[-1] == (b"34", 1034, 2034, None, None, None)


@pytest.mark.parametrize("join_type,single", [(abi.JOIN_INNER, False), (abi.JOIN_PROBE_OUTER, False), (abi.JOIN_INNER, True)])
def test_multi_channel_keys_with_nulls_nan_and_duplicates(ctx, join_type, single):
    rng = np.random.default_rng(77)
    nb, npr = 4000, 15000

    def side(n, hi):
        d = rng.integers(0, 4, n).astype(np.float64)
        d[rng.random(n) < 0.05] = np.nan
        d[rng.random(n) < 0.05] = -0.0
        return Page(Block.bigint(rng.integers(0, hi, n), rng.random(n) < 0.03), Block.varchar([None if x < 0.03 else "k%d" % int(x * 5) for x in rng.random(n)]),
                    Block.double(d, rng.random(n) < 0.03), Block.integer(rng.integers(0, 1000, n)))
    build, probe = side(nb, 40), side(npr, 50)
    got = gpu_join_rows(ctx, [build], [probe], [0, 1, 2], [0, 1, 2], [3, 0], [3, 1], join_type, single)
    want = oracle_join_rows(build, probe, [0, 1, 2], [0, 1, 2], [3, 0], [3, 1], join_type, single)
    assert rows_equal(got, want)
    assert len(got) > npr // 10


def test_multi_page_build_with_nullable_and_varchar_columns(ctx):
    rng = np.random.default_rng(5)
    pages, all_keys, all_pay, all_str = [], [], [], []
    for n in (700, 1, 64, 5000, 9):
        k = rng.integers(0, 3000, n)
        pay = [None if x < 0.1 else float(v) for x, v in zip(rng.random(n), k)]
        st = [None if x < 0.1 else "s%d" % v for x, v in zip(rng.random(n), k)]
        pages.append(Page(Block.bigint(k), Block.double(pay), Block.varchar(st)))
        all_keys += list(k); all_pay += pay; all_str += st
    whole = Page(Block.bigint(all_keys), Block.double(all_pay), Block.varchar(all_str))
    probe = Page(Block.bigint(rng.integers(0, 3500, 20000)))
    got = gpu_join_rows(ctx, pages, [probe], 0, 0, [0], [1, 2], abi.JOIN_INNER, False)
    assert rows_equal(got, oracle_join_rows(whole, probe, 0, 0, [0], [1, 2], abi.JOIN_INNER, False))


def test_generic_lookup_positions_api(ctx):
    build = Page(Block.bigint([1, 2, 1, 3]), Block.bigint([10, 20, 10, 30]))
    bridge = ops.JoinBridge()
    b = ops.HashBuilderOperatorFactory(ctx, bridge, [0, 1], []).create_operator()
    b.add_input(build)
    b.finish()
    lk = bridge.lookup_source
    pos = lk.get_join_positions(Page(Block.bigint([1, 1, 3, 2, None]), Block.bigint([10, 11, 30, 20, 5])))
    assert list(pos) == [2, -1, 3, 1, -1]
    assert lk.has_position_links() and list(lk.position_links()) == [-1, -1, 0, -1]
    b.close(); lk.close()


@pytest.mark.parametrize("join_type", [abi.JOIN_INNER, abi.JOIN_PROBE_OUTER])
@pytest.mark.parametrize("shape", ["all_match", "misses", "null_keys", "duplicates"])
def test_probe_blocks_by_reference(ctx, join_type, shape):
    """LookupJoinPageBuilder.java:144-150: a 1:1 output returns the probe blocks themselves.  With by-reference on, only the join
    key of a host probe page is uploaded; outputs must be identical to the materialising default in every shape (rows dropped,
    NULL keys, duplicate build keys force the remaining channels to be uploaded after all)."""
    rng = np.random.default_rng(len(shape) + join_type)
    nb, npr = 5000, 20000
    bkeys = rng.permutation(nb * 2)[:nb].astype(np.int64)
    if shape == "duplicates":
        bkeys[: nb // 10] = bkeys[nb // 10: 2 * (nb // 10)]
    build = Page(Block.bigint(bkeys), Block.bigint(bkeys * 7), Block.double(bkeys * 0.5))
    pkeys = rng.choice(bkeys, npr) if shape in ("all_match", "duplicates") else rng.integers(0, nb * 2, npr)
    knull = rng.random(npr) < 0.05 if shape == "null_keys" else None
    probes = [Page(Block.double(rng.normal(size=m), rng.random(m) < 0.1), Block.bigint(pkeys[a:a + m], None if knull is None else knull[a:a + m]),
                   Block.varchar(["s%d" % i if i % 7 else None for i in range(m)]))
              for a, m in ((0, 12000), (12000, 8000))]
    want = []
    for p in probes:
        want.extend(oracle_join_rows(build, p, 0, 1, [2, 0, 1], [1, 2], join_type, False))
    got = gpu_join_rows(ctx, [build], probes, 0, 1, [2, 0, 1], [1, 2], join_type, False, by_reference=True)
    assert got == want
    assert got == gpu_join_rows(ctx, [build], probes, 0, 1, [2, 0, 1], [1, 2], join_type, False)


def _types_of(page, channels):
    return [page.get_block(c).flatten().type for c in channels]


@pytest.mark.parametrize("join_type", [abi.JOIN_LOOKUP_OUTER, abi.JOIN_FULL_OUTER])
@pytest.mark.parametrize("single", [False, True])
def test_lookup_outer_and_full_outer(ctx, join_type, single):
    """JoinOperatorType.lookupOuterJoin / fullOuterJoin: the probe side behaves like INNER / PROBE_OUTER and marks the build
    positions it emits (OuterLookupSource.java:95-100); the LookupOuterOperator then returns the unvisited build rows in position
    order with NULL probe channels (LookupOuterOperator.java:170-206).  Several probe pages and two probe operators share the marks."""
    rng = np.random.default_rng(11 + join_type + int(single))
    nb = 6000
    bkeys = rng.integers(0, 4000, nb)
    build = Page(Block.bigint(bkeys, rng.random(nb) < 0.03), Block.double(rng.normal(size=nb)), Block.varchar(["b%d" % i if i % 11 else None for i in range(nb)]))
    probes = []
    for m in (7000, 1, 5000):
        probes.append(Page(Block.varchar(["p%d" % i for i in range(m)]), Block.bigint(rng.integers(1000, 6000, m), rng.random(m) < 0.05)))
    probe_out, build_out = [1, 0], [0, 2, 1]
    bridge = ops.JoinBridge()
    b = ops.HashBuilderOperatorFactory(ctx, bridge, [0], build_out).create_operator()
    b.add_input(build)
    b.finish()
    pf = ops.LookupJoinOperatorFactory(ctx, bridge, join_type, single, [1], probe_out)
    j1, j2 = pf.create_operator(), pf.create_operator()
    got = []
    want = []
    for i, p in enumerate(probes):
        op = j1 if i % 2 == 0 else j2
        op.add_input(p)
        out = op.get_output()
        got.extend(out.rows() if out is not None else [])
        want.extend(oracle_join_rows(build, p, 0, 1, probe_out, build_out, join_type, single))
    assert got == want
    j1.finish()
    j2.finish()
    outer = ops.LookupOuterOperatorFactory(ctx, bridge, _types_of(probes[0], probe_out)).create_operator()
    assert not outer.needs_input()
    page = outer.get_output()
    rows = page.rows() if page is not None else []
    assert rows == oracle_outer_rows(build, probes, 0, 1, len(probe_out), build_out, join_type, single)
    assert outer.get_output() is None and outer.is_finished()
    for op in (outer, j1, j2, b):
        op.close()
    bridge.lookup_source.close()


def test_outer_reference_cases_and_untouched_lookup(ctx):
    # empty lookup sources (TestHashJoinOperator :961-1000, :1052-1103) are in the golden file; a lookup no probe touched
    # returns every build row from the outer operator
    build = Page(Block.bigint([5, 6, None, 5]), Block.bigint([50, 60, 70, 80]))
    bridge = ops.JoinBridge()
    b = ops.HashBuilderOperatorFactory(ctx, bridge, [0], [1, 0]).create_operator()
    b.add_input(build)
    b.finish()
    ops.LookupJoinOperatorFactory(ctx, bridge, abi.JOIN_FULL_OUTER, False, [0], [0]).create_operator().close()
    outer = ops.LookupOuterOperatorFactory(ctx, bridge, [abi.INT64]).create_operator()
    assert outer.get_output().rows() == [(None, 50, 5), (None, 60, 6), (None, 70, None), (None, 80, 5)]
    outer.close()
    b.close()
    bridge.lookup_source.close()


def test_semi_join_reference_cases_and_random(ctx):
    def run(set_block, probe_page, channel):
        bridge = ops.JoinBridge()
        sb = ops.SetBuilderOperatorFactory(ctx, bridge, 0).create_operator()
        sb.add_input(Page(set_block))
        sb.finish()
        sj = ops.HashSemiJoinOperatorFactory(ctx, bridge, channel).create_operator()
        sj.add_input(probe_page)
        out = sj.get_output()
        sj.close()
        sb.close()
        bridge.lookup_source.close()
        return out
    for case in reference_cases()["semi_join"]:
        probe = Page(Block.bigint(case["probe"]))
        out = run(Block.bigint(case["set"]), probe, 0)
        assert out.rows() == [(p, e) for p, e in zip(case["probe"], case["expected"])], case["source"]
    rng = np.random.default_rng(3)
    for set_nulls, probe_nulls in ((False, False), (True, False), (False, True), (True, True)):
        sv = Block.bigint(rng.integers(0, 5000, 3000), rng.random(3000) < 0.01 if set_nulls else None)
        pk = Block.bigint(rng.integers(0, 8000, 20000), rng.random(20000) < 0.05 if probe_nulls else None)
        probe = Page(Block.double(rng.normal(size=20000)), pk, Block.varchar(["x%d" % (i % 13) for i in range(20000)]))
        out = run(sv, probe, 1)
        assert [r[3] for r in out.rows()] == o.semi_join_bigint(sv, pk)
        assert [r[:3] for r in out.rows()] == probe.rows()
    # empty set: NULL probe keys answer false
    out = run(Block.bigint([]), Page(Block.bigint([1, None])), 0)
    assert out.rows() == [(1, False), (None, False)]


@pytest.mark.parametrize("kind", ["double", "real"])
@pytest.mark.parametrize("set_has_nan", [False, True])
def test_semi_join_over_floating_point_keys(ctx, kind, set_has_nan):
    """The semi-join's ChannelSet compares with IDENTICAL (M/operator/FlatSet.java:54,374): a NaN probe key is a member iff the set holds a NaN
    (any encoding), -0.0 and +0.0 are one member; NULLs as for BIGINT keys (HashSemiJoinOperator.java:181-199)."""
    rng = np.random.default_rng(31 + set_has_nan)
    ns, npr = 2000, 30000
    def column(n, with_nan, p_null):
        v = rng.integers(-300, 300, n) * 0.5
        v[rng.random(n) < 0.03] = -0.0
        if kind == "double":
            bits = v.astype(np.float64).view(np.uint64).copy()
            if with_nan:
                bits[rng.random(n) < 0.02] = rng.choice(np.array([0x7FF8000000000000, 0xFFF8000000000001, 0x7FF0000000000001], dtype=np.uint64))
            return Block.double(bits.view(np.float64), rng.random(n) < p_null if p_null else None)
        bits = v.astype(np.float32).view(np.uint32).copy()
        if with_nan:
            bits[rng.random(n) < 0.02] = rng.choice(np.array([0x7FC00000, 0xFFC00001, 0x7F800001], dtype=np.uint32))
        return Block.real(bits.view(np.float32), rng.random(n) < p_null if p_null else None)
    for set_nulls in (0.0, 0.01):
        sv = column(ns, set_has_nan, set_nulls)
        pk = column(npr, True, 0.05)
        bridge = ops.JoinBridge()
        sb = ops.SetBuilderOperatorFactory(ctx, bridge, 0).create_operator()
        sb.add_input(Page(sv))
        sb.finish()
        sj = ops.HashSemiJoinOperatorFactory(ctx, bridge, 1).create_operator()
        sj.add_input(Page(Block.bigint(np.arange(npr)), pk))
        out = sj.get_output()
        sj.close(); sb.close(); bridge.lookup_source.close()
        got = [r[2] for r in out.rows()]
        want = o.semi_join_float(sv, pk)
        assert got == want, (kind, set_has_nan, set_nulls)
        nan_rows = [i for i in range(npr) if not pk.is_null(i) and pk.get(i) != pk.get(i)]
        assert nan_rows and all(got[i] == (True if set_has_nan else (None if set_nulls else False)) for i in nan_rows)


def test_build_side_key_domain(ctx):
    """DynamicFilterSourceOperator / JoinDomainBuilder collect the build-side key domain: the distinct values while they are few,
    else min/max.  Here it is read off the finished table."""
    rng = np.random.default_rng(17)
    keys = rng.integers(-50, 50, 5000)
    nulls = rng.random(5000) < 0.02
    b, lookup = _build_lookup(ctx, [Page(Block.bigint(keys[:3000], nulls[:3000])), Page(Block.bigint(keys[3000:], nulls[3000:]))])
    want = np.unique(keys[~nulls])
    lo, hi, cnt, values, has_null = lookup.key_domain(1000)
    assert (lo, hi, cnt, has_null) == (int(want.min()), int(want.max()), len(want), True)
    assert (values == want).all()
    lo, hi, cnt, values, _ = lookup.key_domain(10)           # too many distinct values: the range is the filter
    assert (lo, hi, cnt) == (int(want.min()), int(want.max()), len(want)) and values is None
    lookup.close()
    b.close()
    b, lookup = _build_lookup(ctx, [Page(Block.bigint([7, -2**63, 7, 3]))])    # INT64_MIN lives beside the table
    lo, hi, cnt, values, has_null = lookup.key_domain(8)
    assert (lo, hi, cnt, has_null) == (-2**63, 7, 3, False) and list(values) == [-2**63, 3, 7]
    lookup.close()
    b.close()


@pytest.mark.parametrize("mode", ["0", "1", "2", None, "span", "roomy", "narrow", "wide"])
@pytest.mark.parametrize("shape", ["tpch", "every_8th", "clustered", "extremes", "shuffled_probe"])
def test_table_layout_modes_agree_with_oracle(ctx, monkeypatch, mode, shape):
    """Slot placement is not observable: mix(key) (mode 0, M/operator/join/PagesHash.java:35-51), line-local (1) and order-preserving
    lines (2, the default for integer keys; falls back to 1 when the keys pile up in a few lines) give the oracle's positions for dense,
    strided (what a hash exchange leaves on one rank), clustered and extreme key sets."""
    monkeypatch.delenv("TGPU_JOIN_HASH", raising=False)
    if mode == "span":
        monkeypatch.setenv("TGPU_JOIN_SPAN", "1")          # the TMA-staged (cp.async.bulk + mbarrier) probe kernel
    elif mode == "roomy":
        monkeypatch.setenv("TGPU_JOIN_NO_DENSE", "1")      # skip the dense geometry attempt
    elif mode == "narrow":
        monkeypatch.setenv("TGPU_JOIN_NO_WIDE", "1")       # 16-byte slots + slot-ordered payload arrays, whatever the page's key locality
    elif mode == "wide":
        monkeypatch.setenv("TGPU_JOIN_WIDE", "always")     # 32-byte wide slots, whatever the page's key locality (default: sampled per page)
    elif mode is not None:
        monkeypatch.setenv("TGPU_JOIN_HASH", mode)
    rng = np.random.default_rng(11)
    n_orders = 100_000
    okeys = o.synth_orders_keys(n_orders, 0, n_orders, 0x7C02, True)
    rows = o.synth_lineitem_rows(n_orders)
    lkeys = o.synth_lineitem_keys(n_orders, 0, rows, 0x7C01, shape == "shuffled_probe")
    if shape == "every_8th":
        okeys = okeys[o.partition_ids(Page(Block.bigint(okeys)), [0], 8) == 3]
    elif shape == "clustered":      # two dense islands and a far outlier: most rows cannot stay in their home line
        okeys = np.concatenate([np.arange(0, 100_000), np.arange(10**12, 10**12 + 100_000), [2**61]]).astype(np.int64)
        lkeys = np.concatenate([rng.integers(-5, 100_010, 150_000), rng.integers(10**12 - 5, 10**12 + 100_010, 150_000), [2**61, 2**61 - 1]]).astype(np.int64)
    elif shape == "extremes":       # span of almost 2^64, INT64_MIN (kept beside the table), negative keys
        okeys = np.concatenate([[-2**63, 2**63 - 1, -1, 0, 1], rng.integers(-2**62, 2**62, 50_000)]).astype(np.int64)
        lkeys = np.concatenate([okeys[::3], rng.integers(-2**63, 2**63 - 1, 100_000)]).astype(np.int64)
    build = Page(Block.bigint(okeys), Block.bigint(okeys % 2557))
    probe = Page(Block.bigint(lkeys), Block.double(lkeys * 0.5))
    b, lk = _build_lookup(ctx, [build], out=[1])
    oj = o.Join(build, [0])
    want = oj.positions(Page(Block.bigint(lkeys)), [0])
    assert (lk.get_join_positions(Page(Block.bigint(lkeys))) == want).all()
    oj.close(); b.close(); lk.close()
    # the operator (fused probe + payload gather, whole tiles + ragged tail) emits the oracle's rows
    got = gpu_join_rows(ctx, [build], [probe], 0, 0, [0, 1], [1], abi.JOIN_INNER, False)
    assert got == oracle_join_rows(build, probe, 0, 0, [0, 1], [1], abi.JOIN_INNER, False)


@pytest.mark.parametrize("join_type", [abi.JOIN_INNER, abi.JOIN_PROBE_OUTER])
@pytest.mark.parametrize("payload", ["bigint+double", "integer+smallint", "tinyint", "double+integer"])
@pytest.mark.parametrize("variant", ["auto", "always", "always-45", "always-18"])
def test_wide_slots_carry_every_payload_width(ctx, monkeypatch, join_type, payload, variant):
    """The fused probe reads key, head and up to two build output cells from one 32-byte wide slot (join.cu WideSlot): 8 / 4 / 2 / 1-byte
    payloads, misses (PROBE_OUTER emits NULLs, INNER drops the row), the INT64_MIN key beside the table, shuffled probe keys, whole tiles
    and the ragged tail give the oracle's rows; so do the other rows-in-flight x CTAs-per-SM shapes of the kernel."""
    if variant != "auto":           # auto: the probe page below has no key locality, so the sampler picks the wide slots as well
        monkeypatch.setenv("TGPU_JOIN_WIDE", "always")
    if "-" in variant:
        monkeypatch.setenv("TGPU_JOIN_WIDE_SHAPE", variant.split("-")[1])
    rng = np.random.default_rng(5)
    okeys = np.concatenate([[-2**63], rng.permutation(np.arange(-3000, 60_000)) * 3]).astype(np.int64)
    cols = {"bigint": Block.bigint(okeys * 7 - 1), "double": Block.double(okeys * 0.25), "integer": Block.integer((okeys % 100_003).astype(np.int32)),
            "smallint": Block.smallint((okeys % 30_011).astype(np.int16)), "tinyint": Block.tinyint((okeys % 113).astype(np.int8))}
    names = payload.split("+")
    build = Page(Block.bigint(okeys), *[cols[n] for n in names])
    lkeys = np.concatenate([rng.integers(-10_000, 190_000, 70_000), [-2**63, 2**63 - 1, -2**63]]).astype(np.int64)     # about two thirds miss
    probe = Page(Block.bigint(lkeys), Block.double(lkeys * 0.5))
    build_out = list(range(1, 1 + len(names)))
    got = gpu_join_rows(ctx, [build], [probe], 0, 0, [0, 1], build_out, join_type, False)
    assert got == oracle_join_rows(build, probe, 0, 0, [0, 1], build_out, join_type, False)


def test_build_over_a_random_half_of_a_dense_domain_stays_fast(ctx):
    # what a 2-way hash exchange leaves on a rank: a hash-selected half of the order keys.  The dense trial geometry does not suit it
    # (lines of 32 key values expect exactly 8 keys) and used to degenerate into chains thousands of lines long; trial geometries are
    # bounded now and the build falls through to the roomy / scattered layouts in milliseconds.
    import time
    n_orders = 12_000_000
    okeys = o.synth_orders_keys(n_orders, 0, n_orders, 0x7C02, True)
    mine = okeys[o.partition_ids(Page(Block.bigint(okeys)), [0], 2) == 1]
    build = Page(Block.bigint(mine))
    t0 = time.time()
    b, lk = _build_lookup(ctx, [build])
    ctx.synchronize()
    elapsed = time.time() - t0
    assert elapsed < 5.0, f"build of {len(mine)} rows took {elapsed:.1f} s"
    probe_keys = np.concatenate([mine[::7], okeys[:100_000]])
    oj = o.Join(build, [0])
    assert (lk.get_join_positions(Page(Block.bigint(probe_keys))) == oj.positions(Page(Block.bigint(probe_keys)), [0])).all()
    oj.close(); b.close(); lk.close()


def test_join_keys_sharing_a_64_bit_row_hash_are_kept_apart(ctx):
    # round 1 answered NOT_SUPPORTED when two different key tuples shared one row hash; now the build moves one of them to its next hash
    # function and the probe follows (DefaultPagesHash compares the values on every hash hit: M/operator/join/DefaultPagesHash.java:246-260)
    from helpers import colliding_bigint_pairs
    rng = np.random.default_rng(5)
    t1 = (11, 22)
    t2 = (33, colliding_bigint_pairs(11, 22, 33))
    t3 = (44, colliding_bigint_pairs(11, 22, 44))            # same hash again, never built
    base_a, base_b = rng.integers(0, 1000, 5000), rng.integers(0, 1000, 5000)
    ba = np.concatenate([[t1[0], t2[0], t1[0]], base_a]).astype(np.int64)
    bb = np.concatenate([[t1[1], t2[1], t1[1]], base_b]).astype(np.int64)
    build = Page(Block.bigint(ba), Block.bigint(bb), Block.bigint(np.arange(len(ba))))
    pa = np.concatenate([[t2[0], t3[0], t1[0], t2[0]], rng.integers(0, 1000, 20000)]).astype(np.int64)
    pb = np.concatenate([[t2[1], t3[1], t1[1], t2[1]], rng.integers(0, 1000, 20000)]).astype(np.int64)
    probe = Page(Block.bigint(pa), Block.bigint(pb), Block.double(np.arange(len(pa)) * 0.5))
    for jt in (abi.JOIN_INNER, abi.JOIN_PROBE_OUTER):
        got = gpu_join_rows(ctx, [build], [probe], [0, 1], [0, 1], [0, 1, 2], [2], jt, False)
        want = oracle_join_rows(build, probe, [0, 1], [0, 1], [0, 1, 2], [2], jt, False)
        assert got == want
    inner = [r for r in want if r[3] is not None][:5]
    assert [r[3] for r in inner[:1]] == [1] and inner[1][3] in (0, 2)       # t2 finds its own row, t1 its own chain; t3 finds nothing
