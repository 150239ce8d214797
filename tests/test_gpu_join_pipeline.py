"""The key-ordered probe over a one-column (keyed) build with order-preserving lines is a pipeline: a producer warp bulk-copies the
probe keys of each 1024-row tile into a shared-memory ring, and the table lines the tile needs into a line buffer, while the consumer
warps resolve the tile before it from shared memory.  These cases cover ring wrap-around and partial rounds, every payload width, and
every way out of the staged path: tiles whose line span is too wide, line walks that leave the staged span, INT64_MIN, and a key column
that is not 16-byte aligned (the earlier kernel then runs).  Every case is compared row for row, in order, with the oracle, including which
build cells are NULL under PROBE_OUTER."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as o
from helpers import gpu_join_rows, oracle_join_rows
from test_gpu_join_match_bits import _device_join_rows, _payload_blocks, _set_layout
from trino_b200 import abi
from trino_b200 import operators as ops
from trino_b200.page import Block, Page

pytestmark = pytest.mark.gpu

RATES = ["all", "none", "half", "last_miss"]
JOIN_TYPES = [abi.JOIN_INNER, abi.JOIN_PROBE_OUTER]
INT64_MIN = -2**63


def _clustered_case(n, rate, seed=0):
    """build keys: even numbers 2, 4, ...; probe keys in key order, about 8 rows per build key, so that a 1024-row tile needs a few dozen
    table lines (lineitem against orders needs about 33): hits, odd misses between them, about half of each, or hits and one miss in the
    last row"""
    rng = np.random.default_rng(3000 + n + 7 * seed + len(rate))
    nb = n // 8 + 16
    bkeys = np.arange(nb, dtype=np.int64) * 2 + 2
    hits = rng.choice(bkeys, n)
    misses = rng.integers(0, nb + 1, n) * 2 + 1
    if rate == "all":
        pkeys = hits
    elif rate == "none":
        pkeys = misses
    elif rate == "half":
        pkeys = np.where(rng.random(n) < 0.5, hits, misses)
    else:
        pkeys = hits.copy()
    pkeys = np.sort(pkeys)
    if rate == "last_miss":
        pkeys[-1] = bkeys[-1] + 1
    return bkeys, pkeys.astype(np.int64)


def _pages(bkeys, pkeys, payload="bigint"):
    build = Page(Block.bigint(bkeys), *_payload_blocks(bkeys, [payload]))
    probe = Page(Block.bigint(pkeys), Block.double(pkeys.astype(np.float64) * 0.5))
    return build, probe


def _check(ctx, build, probe, join_type):
    want = oracle_join_rows(build, probe, 0, 0, [0, 1], [1], join_type, False)
    assert gpu_join_rows(ctx, [build], [probe], 0, 0, [0, 1], [1], join_type, False) == want
    assert _device_join_rows(ctx, build, probe, [abi.INT64, abi.FLOAT64], [1], join_type) == want


@pytest.fixture(autouse=True)
def _auto_layout(monkeypatch):
    _set_layout(monkeypatch, "auto")


@pytest.mark.parametrize("join_type", JOIN_TYPES)
@pytest.mark.parametrize("rate", RATES)
@pytest.mark.parametrize("n", [1024, 1025, 8 * 1024 + 5])
def test_page_sizes_and_match_rates(ctx, n, rate, join_type):
    """One tile, one tile and a ragged tail, and fewer tiles than CTAs, with every row, no row, about half and all but the last row matching."""
    _check(ctx, *_pages(*_clustered_case(n, rate)), join_type)


def _oracle_arrays(build, probe, join_type):
    j = o.Join(build, [0])
    pi, bi = j.expand(j.positions(probe, [0]), join_type, False)
    j.close()
    pk, pp, bp = (b.flatten().values for b in (probe.get_block(0), probe.get_block(1), build.get_block(1)))
    return pk[pi], pp[pi], np.where(bi >= 0, bp[np.maximum(bi, 0)], 0), bi < 0


def _gpu_arrays(ctx, build, probe, join_type):
    bridge = ops.JoinBridge()
    b = ops.HashBuilderOperatorFactory(ctx, bridge, [0], [1]).create_operator()
    b.add_input(build)
    b.finish()
    j = ops.LookupJoinOperatorFactory(ctx, bridge, join_type, False, [0], [0, 1]).create_operator()
    out = ops.drive(j, [probe])
    j.close(); b.close(); bridge.lookup_source.close()
    cols = [np.concatenate([p.get_block(c).flatten().values for p in out]) for c in range(3)]
    nulls = np.concatenate([p.get_block(2).flatten().nulls if p.get_block(2).flatten().nulls is not None
                            else np.zeros(p.position_count, np.bool_) for p in out])
    return cols[0], cols[1], np.where(nulls, 0, cols[2]), nulls


@pytest.mark.parametrize("join_type", JOIN_TYPES)
def test_many_tiles_per_cta(ctx, join_type):
    """4 M rows are about 3900 tiles, several times as many as the CTAs of the grid hold in their rings: the key ring and the line buffers
    wrap around many times, and the last round of tiles leaves some CTAs without a tile."""
    build, probe = _pages(*_clustered_case(4_000_000 + 77, "half"))
    got = _gpu_arrays(ctx, build, probe, join_type)
    want = _oracle_arrays(build, probe, join_type)
    for g, w in zip(got, want):
        assert np.array_equal(g, w)


@pytest.mark.parametrize("join_type", JOIN_TYPES)
@pytest.mark.parametrize("payload", ["tinyint", "smallint", "integer", "bigint"])
def test_payload_widths(ctx, payload, join_type):
    """One payload column of 1, 2, 4 or 8 bytes."""
    _check(ctx, *_pages(*_clustered_case(70_001, "half", seed=1), payload=payload), join_type)


@pytest.mark.parametrize("join_type", JOIN_TYPES)
def test_tiles_with_a_wide_span(ctx, join_type):
    """A far outlier in every 7th tile (a hit at the other end of the build range) makes the tile's line span too wide to stage: those tiles
    read their slots from global memory.  The outlier sits at row 500 of its tile, away from the row pairs the locality vote samples
    (rows 32 m and 32 m + 1), so the page still votes key-ordered."""
    bkeys, pkeys = _clustered_case(64 * 1024 + 3, "half", seed=2)
    pkeys = pkeys.copy()
    for t in range(0, len(pkeys) // 1024, 7):
        pkeys[t * 1024 + 500] = bkeys[-1] if t < len(pkeys) // 2048 else bkeys[0]
    _check(ctx, *_pages(bkeys, pkeys), join_type)


@pytest.mark.parametrize("join_type", JOIN_TYPES)
def test_line_walks_leave_the_staged_span(ctx, join_type):
    """Build keys 16 apart (order-preserving lines of 32 key values, two keys per line), except that six lines hold all 32 of their values:
    24 of those keys overflow into the next four lines.  Each probe tile covers 40 lines and ends with such a line, so the staged span
    (its lines plus the one behind) ends before the walks to the overflowed keys do, and those walks continue in global memory."""
    rng = np.random.default_rng(11)
    lines, per_tile = 10_000, 40
    full = {per_tile * t + per_tile - 1 for t in (10, 50, 90, 130, 170, 210)}
    base = np.arange(1, 2 * lines + 1, dtype=np.int64) * 16          # key 16 + 32 L and 32 + 32 L in line L (kmin = 16)
    extra = np.array([16 + 32 * line + v for line in sorted(full) for v in range(32) if v not in (0, 16)], dtype=np.int64)
    bkeys = np.sort(np.concatenate([base, extra]))
    tiles = []
    for t in range(lines // per_tile):
        lo, hi = 16 + 32 * per_tile * t, 16 + 32 * per_tile * (t + 1)
        own = bkeys[(bkeys >= lo) & (bkeys < hi)]
        tile = np.where(rng.random(1024) < 0.6, rng.choice(own, 1024), rng.integers(lo, hi, 1024))
        tiles.append(np.sort(tile))
    pkeys = np.concatenate(tiles).astype(np.int64)
    _check(ctx, *_pages(bkeys, pkeys), join_type)


@pytest.mark.parametrize("join_type", JOIN_TYPES)
@pytest.mark.parametrize("build_has_min", [True, False])
def test_int64_min_probe_key(ctx, build_has_min, join_type):
    """INT64_MIN in the first rows of every third tile (its cell is in slot mask + 1, beside the table); the other tiles are staged."""
    bkeys, pkeys = _clustered_case(32 * 1024 + 9, "half", seed=3)
    if build_has_min:
        bkeys = np.concatenate([[INT64_MIN], bkeys]).astype(np.int64)
    pkeys = pkeys.copy()
    for t in range(0, len(pkeys) // 1024, 3):
        pkeys[t * 1024:t * 1024 + 3] = INT64_MIN
    _check(ctx, *_pages(bkeys, pkeys), join_type)


def _kernels_launched(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
    return {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}


@pytest.mark.parametrize("join_type", JOIN_TYPES)
def test_key_column_not_16_byte_aligned(ctx, join_type):
    """A key column that starts one row into its buffer (8- but not 16-byte aligned) cannot be bulk-copied: the earlier key-ordered kernel
    runs instead, with the same rows.  The aligned page launches the pipelined kernel."""
    bkeys, pkeys = _clustered_case(16 * 1024 + 3, "half", seed=4)
    build, probe = _pages(bkeys, pkeys)
    want = oracle_join_rows(build, probe, 0, 0, [0, 1], [1], join_type, False)
    n = len(pkeys)
    d_keys = ctx.to_device(np.concatenate([[0], pkeys]).astype(np.int64))
    d_price = ctx.to_device(pkeys.astype(np.float64) * 0.5)
    rows = {}

    def run(shifted):
        bridge = ops.JoinBridge()
        b = ops.HashBuilderOperatorFactory(ctx, bridge, [0], [1]).create_operator()
        b.add_input(build)
        b.finish()
        j = ops.LookupJoinOperatorFactory(ctx, bridge, join_type, False, [0], [0, 1]).create_operator()
        key = d_keys + 8 if shifted else ctx.to_device(pkeys)
        out = ops.drive(j, [ops.DevicePage([ops.DeviceColumn(abi.INT64, key, n), ops.DeviceColumn(abi.FLOAT64, d_price, n)], n)])
        rows[shifted] = [r for page in out for r in page.rows()]
        j.close(); b.close(); bridge.lookup_source.close()
        if not shifted:
            ctx.free(key)

    try:
        shifted = _kernels_launched(lambda: run(True))
        aligned = _kernels_launched(lambda: run(False))
    finally:
        ctx.free(d_keys)
        ctx.free(d_price)
    assert (d_keys + 8) % 16 == 8
    assert rows[True] == want and rows[False] == want
    assert not any("join_probe_keyed_pipe_kernel" in k for k in shifted) and any("join_probe_wide_kernel" in k for k in shifted), shifted
    assert any("join_probe_keyed_pipe_kernel" in k for k in aligned), aligned


def test_bench_shape(ctx):
    """Synthetic lineitem JOIN orders at SF1 (1.5 M orders, about 6 M lineitem rows in order-key order), generated on the device as the
    benchmark does: every probe row matches, its payload is its key % 2557 on every row, and two runs give identical output pages."""
    lib = ctx.lib
    n_orders = 1_500_000
    n = lib.tgpu_synth_lineitem_rows(n_orders)
    d_okeys = ctx.malloc(n_orders * 8)
    ctx.check(lib.tgpu_synth_orders_keys(ctx.h, n_orders, 0, n_orders, 0x7C02, 1, C.c_void_p(d_okeys)))
    d_lkeys = ctx.malloc(n * 8)
    ctx.check(lib.tgpu_synth_lineitem_keys(ctx.h, n_orders, 0, n, 0x7C01, 0, C.c_void_p(d_lkeys)))
    okeys = ctx.to_host(d_okeys, np.int64, n_orders)
    lkeys = ctx.to_host(d_lkeys, np.int64, n)
    d_date = ctx.to_device(okeys % 2557)
    d_price = ctx.to_device(lkeys.astype(np.float64) * 0.5)

    def column_sum(col, mod=0):
        c = abi.Column()
        c.type, c.flags, c.length, c.data, c.offsets, c.validity = col.type, 0, col.length, col.ptr, col.offsets, col.validity
        v = C.c_int64()
        ctx.check(lib.tgpu_column_sum(ctx.h, C.byref(c), mod, C.byref(v)))
        return v.value

    bridge = ops.JoinBridge()
    b = ops.HashBuilderOperatorFactory(ctx, bridge, [0], [1], n_orders).create_operator()
    b.add_input(ops.DevicePage([ops.DeviceColumn(abi.INT64, d_okeys, n_orders), ops.DeviceColumn(abi.INT64, d_date, n_orders)], n_orders))
    b.finish()
    j = ops.LookupJoinOperatorFactory(ctx, bridge, abi.JOIN_INNER, False, [0], [0, 1]).create_operator()
    probe = ops.DevicePage([ops.DeviceColumn(abi.INT64, d_lkeys, n), ops.DeviceColumn(abi.FLOAT64, d_price, n)], n)
    runs = []
    try:
        for _ in range(2):
            j.add_input(probe)
            out = j.get_output_device()
            assert out is not None and out.rows == n
            assert column_sum(out.column(2)) == column_sum(out.column(0), 2557)
            runs.append([ctx.to_host(out.column(c).ptr, dt, n) for c, dt in ((0, np.int64), (1, np.float64), (2, np.int64))])
            out.release()
    finally:
        j.close(); b.close(); bridge.lookup_source.close()
        for p in (d_okeys, d_lkeys, d_date, d_price):
            ctx.free(p)
    assert np.array_equal(runs[0][0], lkeys)
    assert np.array_equal(runs[0][2], lkeys % 2557)
    for a, b_ in zip(runs[0], runs[1]):
        assert np.array_equal(a, b_)
