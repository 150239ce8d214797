"""Shared helpers: run a case through the CPU oracle and through the GPU operators, as materialised rows."""
import json
import os

import numpy as np

from trino_b200 import abi
from trino_b200.page import Block, Page

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def reference_cases():
    with open(os.path.join(GOLDEN, "reference_cases.json")) as f:
        return json.load(f)


def oracle_join_rows(build_page, probe_page, build_key, probe_key, probe_out, build_out, join_type, single_match, force_default=False):
    """Rows the reference's LookupJoinOperator emits (probe output channels then build output channels)."""
    import oracle_lib as o
    bk = list(build_key) if isinstance(build_key, (list, tuple)) else [build_key]
    pk = list(probe_key) if isinstance(probe_key, (list, tuple)) else [probe_key]
    j = o.Join(build_page, bk, force_default=force_default)
    pos = j.positions(probe_page, pk)
    pi, bi = j.expand(pos, join_type, single_match)
    pcols = [probe_page.get_block(c).flatten().to_pylist() for c in probe_out]
    bcols = [build_page.get_block(c).flatten().to_pylist() for c in build_out]
    rows = []
    for p, b in zip(pi, bi):
        rows.append(tuple(c[p] for c in pcols) + tuple((c[b] if b >= 0 else None) for c in bcols))
    j.close()
    return rows


def join_type_of(case):
    from trino_b200 import abi
    return {"inner": abi.JOIN_INNER, "lookup_outer": abi.JOIN_LOOKUP_OUTER, "full_outer": abi.JOIN_FULL_OUTER}.get(case["join_type"], abi.JOIN_PROBE_OUTER)


def oracle_outer_rows(build_page, probe_pages, build_key, probe_key, num_probe_out, build_out, join_type, single_match):
    """Rows of the LookupOuterOperator after all probe pages: unvisited build positions in order (OuterLookupSource.java:109-139)"""
    import oracle_lib as o
    bk = list(build_key) if isinstance(build_key, (list, tuple)) else [build_key]
    pk = list(probe_key) if isinstance(probe_key, (list, tuple)) else [probe_key]
    j = o.Join(build_page, bk)
    visited = set()
    for p in probe_pages:
        pos = j.positions(p, pk)
        _, bi = j.expand(pos, join_type, single_match)
        visited.update(int(b) for b in bi if b >= 0)
    j.close()
    bcols = [build_page.get_block(c).flatten().to_pylist() for c in build_out]
    return [tuple([None] * num_probe_out) + tuple(c[b] for c in bcols) for b in range(build_page.position_count) if b not in visited]


def gpu_join_rows(ctx, build_pages, probe_pages, build_key, probe_key, probe_out, build_out, join_type, single_match, by_reference=False):
    from trino_b200 import operators as ops
    bridge = ops.JoinBridge()
    bk = list(build_key) if isinstance(build_key, (list, tuple)) else [build_key]
    pk = list(probe_key) if isinstance(probe_key, (list, tuple)) else [probe_key]
    bf = ops.HashBuilderOperatorFactory(ctx, bridge, bk, build_out)
    b = bf.create_operator()
    for p in build_pages:
        assert b.needs_input()
        b.add_input(p)
    b.finish()
    assert b.is_finished()
    pf = ops.LookupJoinOperatorFactory(ctx, bridge, join_type, single_match, pk, probe_out)
    j = pf.create_operator()
    if by_reference:
        j.set_passthrough_by_reference(True)
    out = ops.drive(j, probe_pages)
    rows = []
    for page in out:
        rows.extend(page.rows())
    j.close()
    b.close()
    bridge.lookup_source.close()
    return rows


def rows_equal(a, b, rel=0.0):
    if len(a) != len(b):
        return False
    for ra, rb in zip(a, b):
        if len(ra) != len(rb):
            return False
        for x, y in zip(ra, rb):
            if x is None or y is None:
                if x is not y:
                    return False
            elif isinstance(x, float) or isinstance(y, float):
                if x != x and y != y:
                    continue
                if rel == 0.0:
                    if x != y:
                        return False
                elif abs(x - y) > rel * max(abs(x), abs(y), 1e-300):
                    return False
            elif x != y:
                return False
    return True


def random_bigint_block(rng, n, lo, hi, null_frac=0.0):
    v = rng.integers(lo, hi, size=n, dtype=np.int64)
    nulls = rng.random(n) < null_frac if null_frac > 0 else None
    return Block.bigint(v, nulls)


def oracle_agg_rows(pages, key_channels, aggs):
    """group-id order rows: keys then aggregate values (None = NULL), sequential left fold like the reference"""
    import numpy as np
    import oracle_lib as o
    from trino_b200 import abi
    lib = o.load()
    og = o.GroupByHash(0, 16)
    state = []
    keyrows = {}
    for page in pages:
        ids = og.get_group_ids(page, key_channels)
        G = og.group_count()
        for i, gid in enumerate(ids):
            if gid not in keyrows:
                keyrows[int(gid)] = tuple(page.get_block(c).flatten().get(i) for c in key_channels)
        for ai, (fn, ch, mask) in enumerate(aggs):
            if len(state) <= ai:
                state.append({"sum": np.zeros(0), "cnt": np.zeros(0, np.int64), "isum": np.zeros(0, np.int64), "nn": np.zeros(0, np.uint8), "acc": np.zeros(0), "iacc": np.zeros(0, np.int64)})
            st = state[ai]
            for k in [k for k in st if k != "dbl"]:
                if len(st[k]) < G:
                    st[k] = np.concatenate([st[k], np.zeros(G - len(st[k]), st[k].dtype)])
            blk = page.get_block(ch).flatten() if ch >= 0 else None
            valid = None
            if blk is not None and blk.nulls is not None:
                valid = np.packbits(~blk.nulls, bitorder="little")
            sel = None
            if mask >= 0:
                mb = page.get_block(mask).flatten()
                sel = ((mb.values != 0) & (~mb.nulls if mb.nulls is not None else True)).astype(np.uint8)
            n = page.position_count
            P = o._p
            ids32 = np.ascontiguousarray(ids, np.int32)
            is_dbl = blk is not None and blk.type == abi.FLOAT64
            vals = None if blk is None else np.ascontiguousarray(blk.values.astype(np.float64 if is_dbl else np.int64))
            if fn == abi.AGG_COUNT_STAR:
                lib.orc_agg_count(P(ids32), n, None, P(sel), P(st["cnt"]))
            elif fn == abi.AGG_COUNT:
                lib.orc_agg_count(P(ids32), n, P(valid), P(sel), P(st["cnt"]))
            elif fn == abi.AGG_SUM and is_dbl:
                lib.orc_agg_sum_double(P(ids32), n, P(vals), P(valid), P(sel), P(st["sum"]), P(st["nn"]))
            elif fn == abi.AGG_SUM:
                assert lib.orc_agg_sum_bigint(P(ids32), n, P(vals), P(valid), P(sel), P(st["isum"]), P(st["nn"])) == 0
            elif fn == abi.AGG_AVG:
                fvals = np.ascontiguousarray(vals.astype(np.float64))   # keep alive across the call
                lib.orc_agg_avg_double(P(ids32), n, P(fvals), P(valid), P(sel), P(st["sum"]), P(st["cnt"]))
            elif is_dbl:
                lib.orc_agg_minmax_double(P(ids32), n, P(vals), P(valid), int(fn == abi.AGG_MAX), P(st["acc"]), P(st["nn"]))
            else:
                lib.orc_agg_minmax_bigint(P(ids32), n, P(vals), P(valid), int(fn == abi.AGG_MAX), P(st["iacc"]), P(st["nn"]))
            st["dbl"] = is_dbl
    G = og.group_count()
    rows = []
    for g in range(G):
        r = list(keyrows[g])
        for ai, (fn, ch, mask) in enumerate(aggs):
            st = state[ai]
            if fn in (abi.AGG_COUNT_STAR, abi.AGG_COUNT):
                r.append(int(st["cnt"][g]))
            elif fn == abi.AGG_SUM:
                r.append(None if not st["nn"][g] else (float(st["sum"][g]) if st["dbl"] else int(st["isum"][g])))
            elif fn == abi.AGG_AVG:
                r.append(None if st["cnt"][g] == 0 else float(st["sum"][g]) / float(st["cnt"][g]))
            else:
                r.append(None if not st["nn"][g] else (float(st["acc"][g]) if st["dbl"] else int(st["iacc"][g])))
        rows.append(tuple(r))
    og.close()
    return rows




def kernels_launched(fn, attempts=5):
    """Names of the kernels `fn` launches, from a profiler session (CUDA activity) in which `fn` runs between two marker kernels
    (torch's spin_kernel, with device synchronisations around `fn`).  Only kernels that start between this session's own markers count,
    so a record delivered late from another session cannot be attributed to `fn`.  The profiler can lose the records of a short session;
    a session without both markers is incomplete and `fn` is observed again.  None: no complete session in `attempts`."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    for _ in range(attempts):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            torch.cuda._sleep(1000)
            torch.cuda.synchronize()
            fn()
            torch.cuda.synchronize()
            torch.cuda._sleep(1000)
            torch.cuda.synchronize()
        events = [(e.time_range.start, e.name.replace(" ", "")) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        marks = sorted(t for t, name in events if "spin_kernel" in name)
        if len(marks) == 2:
            return sorted({name for t, name in events if marks[0] < t < marks[1]})
    return None


def aggregation_known_answer_cases():
    """The sequences of the reference's AbstractTestAggregationFunction (:70-127: testNoPositions is omitted - a grouped aggregation
    without rows has no group -, testSinglePosition, testMultiplePositions, testAllPositionsNull, testMixedNullAndNonNullPositions,
    testNegativeOnlyValues, testPositiveOnlyValues) with the expected values of TestDoubleSumAggregation.java:38-50,
    TestDoubleAverageAggregation.java:38-50, TestCountAggregation / TestLongSumAggregation (same formulas over BIGINT)."""
    import numpy as np
    cases = []
    for name, start, length, total, pattern in (("single", 0, 1, 1, "none"), ("multiple", 0, 5, 5, "none"), ("all_null", 0, 0, 10, "all"),
                                                ("alternating", 0, 10, 20, "alternate"), ("negative", -10, 5, 5, "none"), ("positive", 2, 4, 4, "none")):
        if pattern == "none":
            values = np.arange(start, start + length)
            nulls = None
        elif pattern == "all":
            values = np.zeros(total, dtype=np.int64)
            nulls = np.ones(total, dtype=bool)
        else:       # AbstractTestAggregationFunction.createAlternatingNullsBlock: null, v0, null, v1, ...
            values = np.repeat(np.arange(start, start + length), 2)
            nulls = np.tile(np.array([True, False]), length)
        seq = [float(i) for i in range(start, start + length)]
        s = 0.0
        for v in seq:
            s += v
        cases.append({"name": name, "values": values, "nulls": nulls, "count_star": total, "count": length, "sum_double": s if length else None,
                      "avg_double": (s / length) if length else None, "sum_bigint": int(sum(range(start, start + length))) if length else None,
                      "min": float(start) if length else None, "max": float(start + length - 1) if length else None})
    return cases


def hash_aggregation_operator_case(number_of_rows=40_000):
    """TestHashAggregationOperator.testHashAggregation (:138-188) restated over BIGINT channels (the GPU path takes dictionary codes
    where the reference test uses VARCHAR; max(varchar) is left out): three sequence pages, group key = channel 1 starting at 0,
    aggregates count(*), sum(ch3), avg(ch3), count(ch0), count(ch4 boolean).  Expected row i: (i, 3, 3*i, float(i), 3, 3)."""
    import numpy as np
    from trino_b200 import abi
    from trino_b200.page import Block, Page
    pages = []
    for start2 in (100_000, 200_000, 300_000):
        seq = np.arange(number_of_rows, dtype=np.int64)
        pages.append(Page(Block.bigint(100 + seq), Block.bigint(seq), Block.bigint(start2 + seq), Block.bigint(seq), Block.boolean((500 + seq) % 2 == 0)))
    aggs = [(abi.AGG_COUNT_STAR, -1, -1), (abi.AGG_SUM, 3, -1), (abi.AGG_AVG, 3, -1), (abi.AGG_COUNT, 0, -1), (abi.AGG_COUNT, 4, -1)]
    expected = [(i, 3, 3 * i, float(i), 3, 3) for i in range(number_of_rows)]
    return pages, [1], aggs, expected


def _oracle_inner_probe(build_keys, build_payload, probe_keys, probe_valid):
    """INNER join of probe rows (NULL keys never match, JoinProbe.java:154-171) against unique build keys through the oracle:
    (selected probe rows, their build payload)"""
    import oracle_lib as o
    j = o.Join(Page(Block.bigint(build_keys)), [0])
    pos = j.positions(Page(Block.bigint(probe_keys, None if probe_valid is None else ~probe_valid)), [0])
    j.close()
    sel = np.nonzero(pos >= 0)[0]
    return sel, build_payload[pos[sel]]


def oracle_star_rows(n, first, seed=0xD501):
    """store_sales rows [first, first + n) through the star join of bench_workloads.py as a chain of oracle joins:
    rows (ss_customer_sk, ss_net_paid, d_year, i_brand_id, s_val, c_birth_year) in fact order, and the generator's count of rows with
    both nullable keys present"""
    import oracle_lib as o
    date0 = 2415022
    cols, both = o.synth_store_sales(n, first, seed)
    cv = np.unpackbits(cols["customer_valid"], bitorder="little")[:n].astype(bool)
    sv = np.unpackbits(cols["store_valid"], bitorder="little")[:n].astype(bool)
    date_k, item_k, store_k, cust_k = np.arange(date0, date0 + 73049), np.arange(1, 300001), np.arange(1, 1003), np.arange(1, 12_000_001)
    idx = np.arange(n)
    sel, d_year = _oracle_inner_probe(date_k, 1900 + (date_k - date0) // 365, cols["date_sk"], None)
    idx = idx[sel]
    sel, i_brand = _oracle_inner_probe(item_k, item_k % 1000 + 1, cols["item_sk"][idx], None)
    idx, d_year = idx[sel], d_year[sel]
    sel, s_val = _oracle_inner_probe(store_k, store_k * 7 % 100, cols["store_sk"][idx], sv[idx])
    idx, d_year, i_brand = idx[sel], d_year[sel], i_brand[sel]
    sel, c_birth = _oracle_inner_probe(cust_k, 1920 + cust_k % 70, cols["customer_sk"][idx], cv[idx])
    idx, d_year, i_brand, s_val = idx[sel], d_year[sel], i_brand[sel], s_val[sel]
    rows = list(zip(cols["customer_sk"][idx].tolist(), cols["net_paid"][idx].tolist(), d_year.tolist(), i_brand.tolist(), s_val.tolist(), c_birth.tolist()))
    return rows, both


# ---- constructing 64-bit hash collisions (to drive the full-key-compare-and-rehash paths that replace the round-1 "abort on collision")
_M = (1 << 64) - 1
_P1, _P2 = 0x9E3779B185EBCA87, 0xC2B2AE3D27D4EB4F


def _rotl(x, r):
    return ((x << r) | (x >> (64 - r))) & _M


def _rotr(x, r):
    return ((x >> r) | (x << (64 - r))) & _M


def _hash_long(v):
    return (_rotl((v * _P2) & _M, 31) * _P1) & _M


def _unhash_long(h):
    v = (_rotr((h * pow(_P1, -1, 1 << 64)) & _M, 31) * pow(_P2, -1, 1 << 64)) & _M
    return v - (1 << 64) if v >= (1 << 63) else v


def colliding_bigint_pairs(a1, b1, a2):
    """b2 such that the reference row hash 31 * H(a) + H(b) (InterpretedHashGenerator.java:102-110) of (a2, b2) equals that of (a1, b1)"""
    target = (31 * _hash_long(a1 & _M) + _hash_long(b1 & _M) - 31 * _hash_long(a2 & _M)) & _M
    return _unhash_long(target)


def _fmix(x):
    x ^= x >> 33; x = (x * 0xff51afd7ed558ccd) & _M; x ^= x >> 33; x = (x * 0xc4ceb9fe1a85ec53) & _M; x ^= x >> 33
    return x


def _unfmix(x):
    x ^= x >> 33; x = (x * pow(0xc4ceb9fe1a85ec53, -1, 1 << 64)) & _M; x ^= x >> 33; x = (x * pow(0xff51afd7ed558ccd, -1, 1 << 64)) & _M; x ^= x >> 33
    return x


def colliding_groupby_pairs(a1, b1, a2):
    """b2 such that the composite-key fingerprint of the general group-by path (csrc/groupby.cu pack_key, two non-NULL BIGINT keys,
    attempt 0) of (a2, b2) equals that of (a1, b1)"""
    seed = 0x9E3779B97F4A7C15

    def step(h, u):
        return (_fmix(h ^ (u & _M)) * 31) & _M

    target = step(step(seed, a1), b1)
    h1 = step(seed, a2)
    x = (target * pow(31, -1, 1 << 64)) & _M
    b2 = _unfmix(x) ^ h1
    return b2 - (1 << 64) if b2 >= (1 << 63) else b2
