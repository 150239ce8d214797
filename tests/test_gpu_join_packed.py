"""A one-column build with order-preserving lines (mode 2) packs its keyed table into 4-byte {int16 krel, uint16 cell} or 8-byte
{int32 krel, uint32 cell} slots when the data allow: krel is the key relative to its slot's line, key - kmin - ((slot >> 3) << shift), and
the cell is the payload relative to the smallest payload of the table.  Otherwise the table keeps 16-byte {key, cell} slots.  The tier is
seen through the lookup's memory size.  Every case is compared row for row, in order, with the oracle, for INNER and PROBE_OUTER, over a
key-ordered page (the pipelined kernel), a shuffled page (the random-access shape) and a key column that is not 16-byte aligned."""
import ctypes as C

import numpy as np
import pytest

from helpers import oracle_join_rows
from test_gpu_join_match_bits import _lookup_bytes, _set_layout
from trino_b200 import abi
from trino_b200 import operators as ops
from trino_b200.page import Block, Page

pytestmark = pytest.mark.gpu

JOIN_TYPES = [abi.JOIN_INNER, abi.JOIN_PROBE_OUTER]
INT64_MIN, INT64_MAX = -2**63, 2**63 - 1


@pytest.fixture(autouse=True)
def _auto_layout(monkeypatch):
    _set_layout(monkeypatch, "auto")


def _width(sizes):
    """bytes per slot of the keyed table: its size (auto minus no_wide, one build column) against the 32-byte wide table that a
    two-column build of the same keys carries (allocations are rounded up to a few hundred bytes)"""
    keyed = sizes["auto"][0] - sizes["no_wide"][0]
    wide = sizes["auto"][1] - sizes["no_wide"][1]
    width = round(32 * keyed / wide)
    assert width in (4, 8, 16), sizes
    return width


def _slot_bytes(ctx, monkeypatch, bkeys, payload):
    one = Page(Block.bigint(bkeys), payload)
    two = Page(Block.bigint(bkeys), payload, payload)
    sizes = {}
    for layout in ("no_wide", "auto"):
        _set_layout(monkeypatch, layout)
        sizes[layout] = (_lookup_bytes(ctx, one, [1]), _lookup_bytes(ctx, two, [1, 2]))
    return _width(sizes)


def _device_rows(ctx, build, probe, join_type, shifted):
    """the join of a probe page resident on the device; shifted: its key column starts one row into its buffer (8- but not 16-byte
    aligned), which the bulk copies of the pipelined kernel cannot read"""
    pk = probe.get_block(0).flatten().values
    n = len(pk)
    d_keys = ctx.to_device(np.concatenate([[0], pk]).astype(np.int64) if shifted else pk)
    d_price = ctx.to_device(probe.get_block(1).flatten().values)
    key = d_keys + 8 if shifted else d_keys
    assert key % 16 == (8 if shifted else 0)
    bridge = ops.JoinBridge()
    b = ops.HashBuilderOperatorFactory(ctx, bridge, [0], [1]).create_operator()
    b.add_input(build)
    b.finish()
    j = ops.LookupJoinOperatorFactory(ctx, bridge, join_type, False, [0], [0, 1]).create_operator()
    try:
        out = ops.drive(j, [ops.DevicePage([ops.DeviceColumn(abi.INT64, key, n), ops.DeviceColumn(abi.FLOAT64, d_price, n)], n)])
        return [r for page in out for r in page.rows()]
    finally:
        j.close(); b.close(); bridge.lookup_source.close()
        ctx.free(d_keys)
        ctx.free(d_price)


def _check(ctx, bkeys, payload, pkeys, join_type, seed=0):
    build = Page(Block.bigint(bkeys), payload)
    ordered = np.sort(pkeys).astype(np.int64)
    shuffled = np.random.default_rng(seed).permutation(pkeys).astype(np.int64)
    for keys, shifted in ((ordered, False), (shuffled, False), (ordered, True)):
        probe = Page(Block.bigint(keys), Block.double(keys.astype(np.float64) * 0.5))
        want = oracle_join_rows(build, probe, 0, 0, [0, 1], [1], join_type, False)
        got = _device_rows(ctx, build, probe, join_type, shifted)
        assert got == want, ("shuffled" if keys is shuffled else "ordered", shifted)


def _hits_and_misses(bkeys, n, seed):
    """about half build keys, half keys next to them that the build does not hold"""
    rng = np.random.default_rng(seed)
    hits = rng.choice(bkeys, n)
    misses = rng.choice(bkeys, n) + 1
    misses = misses[~np.isin(misses, bkeys)]
    return np.concatenate([hits, misses[:n // 2]]).astype(np.int64)


DENSE = np.arange(70_001, dtype=np.int64) * 2 + 2           # order-key-like: a line of 8 key values holds 4 keys

TIER_PAYLOADS = {
    "tinyint": (4, lambda k: Block.tinyint((k % 113).astype(np.int8))),
    "smallint": (4, lambda k: Block.smallint((k % 30_011).astype(np.int16))),
    "bigint_mod_2557": (4, lambda k: Block.bigint(k % 2557)),
    "integer_range_2e5": (8, lambda k: Block.integer((k % 100_003 * 2).astype(np.int32))),
    "bigint_range_1e6": (8, lambda k: Block.bigint(k * 7 - 1)),
    "bigint_range_1e11": (16, lambda k: Block.bigint(k << 20)),
    "double_wide_bits": (16, lambda k: Block.double(k * 0.25)),
}


@pytest.mark.parametrize("join_type", JOIN_TYPES)
@pytest.mark.parametrize("payload", list(TIER_PAYLOADS))
def test_tier_by_payload_range(ctx, monkeypatch, payload, join_type):
    """Over the same keys, a payload whose range is below 2^16 gets 4-byte slots, one below 2^32 8-byte slots, and a wider one keeps
    the 16-byte slots."""
    width, make = TIER_PAYLOADS[payload]
    assert _slot_bytes(ctx, monkeypatch, DENSE, make(DENSE)) == width
    _set_layout(monkeypatch, "auto")
    _check(ctx, DENSE, make(DENSE), _hits_and_misses(DENSE, 40_000, 1), join_type)


OFFSET_PAYLOADS = {
    "negative_bigint": lambda k: Block.bigint(-(k % 1000) - 5),
    "negative_integer": lambda k: Block.integer((k % 5000 - 10_000).astype(np.int32)),
    "negative_smallint": lambda k: Block.smallint((k % 300 - 150).astype(np.int16)),
    "negative_tinyint": lambda k: Block.tinyint((k % 200 - 100).astype(np.int8)),
    "integer_around_zero": lambda k: Block.integer((k % 60_000 - 30_000).astype(np.int32)),
    "near_int64_min": lambda k: Block.bigint(INT64_MIN + k % 1000),
    "near_int64_max": lambda k: Block.bigint(INT64_MAX - k % 1000),
    "double_near_one": lambda k: Block.double((np.float64(1.0).view(np.int64) + k % 100).view(np.float64)),
    "double_negative": lambda k: Block.double((np.float64(-3.5).view(np.int64) + k % 5000).view(np.float64)),
}


@pytest.mark.parametrize("join_type", JOIN_TYPES)
@pytest.mark.parametrize("payload", list(OFFSET_PAYLOADS))
def test_payload_offset(ctx, monkeypatch, payload, join_type):
    """Small payload ranges anywhere in their type, as cells relative to the smallest: negative values of every integer width, values
    next to INT64_MIN and INT64_MAX, and DOUBLEs whose bits lie close together.  All of them get 4-byte slots."""
    make = OFFSET_PAYLOADS[payload]
    assert _slot_bytes(ctx, monkeypatch, DENSE, make(DENSE)) == 4
    _set_layout(monkeypatch, "auto")
    _check(ctx, DENSE, make(DENSE), _hits_and_misses(DENSE, 40_000, 2), join_type)


@pytest.mark.parametrize("join_type", JOIN_TYPES)
@pytest.mark.parametrize("payload", ["bigint_mod_2557", "bigint_range_1e6", "bigint_range_1e11"])
def test_keys_that_defeat_a_truncated_compare(ctx, monkeypatch, payload, join_type):
    """Keys 1 .. 30000 give 16384 lines of 2 key values (shift 1), so (cap / 8) << shift is 2^15: a probe key 2^15, 2^16 or 2^32 above a
    build key starts its walk in that key's slot and meets it, with a krel that is equal in its low 16 (or 32) bits.  All of them miss,
    in every tier."""
    width, make = TIER_PAYLOADS[payload]
    bkeys = np.arange(1, 30_001, dtype=np.int64)
    assert _slot_bytes(ctx, monkeypatch, bkeys, make(bkeys)) == width
    _set_layout(monkeypatch, "auto")
    sample = np.random.default_rng(3).choice(bkeys, 6000)
    pkeys = np.concatenate([sample, sample + 2**15, sample + 2**16, sample + 2**32])
    _check(ctx, bkeys, make(bkeys), pkeys, join_type)


@pytest.mark.parametrize("join_type", JOIN_TYPES)
@pytest.mark.parametrize("payload", ["bigint_mod_2557", "bigint_range_1e6", "bigint_range_1e11"])
def test_probe_rel_equal_to_the_empty_marker(ctx, monkeypatch, payload, join_type):
    """Keys 1 .. 30000 (kmin 1, 16384 lines of 2 key values, shift 1): a probe key kmin - 2^15 + j or kmin - 2^31 + j lands in line j >> 1
    with rel = -2^15 or -2^31 when j is even, the empty marker of the 4- or 8-byte slot, and its walk meets the empty slots of that line.
    All of them miss, in every tier.  Each key comes 8 times, so that a key-ordered tile spans 64 lines and is staged."""
    width, make = TIER_PAYLOADS[payload]
    bkeys = np.arange(1, 30_001, dtype=np.int64)
    assert _slot_bytes(ctx, monkeypatch, bkeys, make(bkeys)) == width
    _set_layout(monkeypatch, "auto")
    j = np.arange(2**15, dtype=np.int64)
    marker = np.repeat(np.concatenate([bkeys[0] - 2**15 + j, bkeys[0] - 2**31 + j]), 8)
    sample = np.random.default_rng(7).choice(bkeys, 6000)
    _check(ctx, bkeys, make(bkeys), np.concatenate([sample, marker]), join_type)


def _overflowing_lines():
    """keys 16 apart (lines of 32 key values, two keys per line) except that six lines hold all 32 of their values: 24 keys of each
    overflow into the next lines, with negative krel, and walks to them leave a 40-line probe tile's staged span"""
    lines = 10_000
    full = [40 * t + 39 for t in (10, 50, 90, 130, 170, 210)]
    base = np.arange(1, 2 * lines + 1, dtype=np.int64) * 16
    extra = np.array([16 + 32 * line + v for line in full for v in range(32) if v not in (0, 16)], dtype=np.int64)
    return np.sort(np.concatenate([base, extra]))


def _wrapping_build():
    """one key at the start of each of 2047 lines of 32 key values, and all 32 values of the last line: 24 of those walk past the last
    line into lines 0, 1 and 2 (capacity 16384, shift 5), where their krel is about 2^16"""
    return np.concatenate([np.arange(2047, dtype=np.int64) * 32, 2047 * 32 + np.arange(32, dtype=np.int64)]) + 1000


def _spaced_build(spacing):
    """4000 keys `spacing` apart, each at a random offset below spacing / 2: lines of 2^21 (or 2^41) key values, so krel overflows 16
    (or 32) bits from the key side"""
    rng = np.random.default_rng(spacing.bit_length())
    return np.arange(4000, dtype=np.int64) * spacing + rng.integers(0, spacing // 2, 4000) + 5


DISPLACED = {
    "clustered_lines": (4, _overflowing_lines),
    "wrap_to_line_0": (None, _wrapping_build),
    "krel_over_16_bits": (8, lambda: _spaced_build(2**20)),
    "krel_over_32_bits": (16, lambda: _spaced_build(2**40)),
}


@pytest.mark.parametrize("join_type", JOIN_TYPES)
@pytest.mark.parametrize("case", list(DISPLACED))
def test_keys_off_their_home_line(ctx, monkeypatch, case, join_type):
    """Keys displaced to later lines (negative krel, walks that leave the staged span), a walk that wraps from the last line to line 0
    (correct whichever tier it picks), and keys whose krel needs 32 or 64 bits.  The payload alone would fit 4-byte slots."""
    width, make = DISPLACED[case]
    bkeys = make()
    payload = lambda k: Block.bigint(k % 2557)
    got = _slot_bytes(ctx, monkeypatch, bkeys, payload(bkeys))
    assert width is None or got == width
    _set_layout(monkeypatch, "auto")
    pkeys = np.concatenate([_hits_and_misses(bkeys, 30_000, 4), np.random.default_rng(5).integers(bkeys[0], bkeys[-1], 10_000)])
    _check(ctx, bkeys, payload(bkeys), pkeys, join_type)


@pytest.mark.parametrize("join_type", JOIN_TYPES)
@pytest.mark.parametrize("build_min", ["none", "in_range", "far_cell"])
def test_int64_min(ctx, monkeypatch, build_min, join_type):
    """INT64_MIN as a probe key, with and without it in the build.  Its cell sits beside the table (slot mask + 1) and counts towards
    the payload range: a far cell moves the table to 8-byte slots."""
    bkeys = DENSE
    cells = DENSE % 2557
    if build_min != "none":
        bkeys = np.concatenate([[INT64_MIN], DENSE]).astype(np.int64)
        cells = np.concatenate([[1_000_000 if build_min == "far_cell" else 17], cells]).astype(np.int64)
    assert _slot_bytes(ctx, monkeypatch, bkeys, Block.bigint(cells)) == (8 if build_min == "far_cell" else 4)
    _set_layout(monkeypatch, "auto")
    pkeys = _hits_and_misses(DENSE, 30_000, 6)
    pkeys[::97] = INT64_MIN
    _check(ctx, bkeys, Block.bigint(cells), pkeys, join_type)


def test_bench_shape(ctx, monkeypatch):
    """Synthetic lineitem JOIN orders at SF1, generated on the device as the benchmark does: the build picks 4-byte slots, every probe
    row matches with payload key % 2557, and two runs give identical output pages."""
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
    date = ops.DeviceColumn(abi.INT64, d_date, n_orders)
    okey_col = ops.DeviceColumn(abi.INT64, d_okeys, n_orders)

    def lookup_bytes(cols):
        bridge = ops.JoinBridge()
        b = ops.HashBuilderOperatorFactory(ctx, bridge, [0], list(range(1, len(cols))), n_orders).create_operator()
        b.add_input(ops.DevicePage(cols, n_orders))
        b.finish()
        v = bridge.lookup_source.get_in_memory_size_in_bytes()
        b.close(); bridge.lookup_source.close()
        return v

    runs = []
    try:
        sizes = {}
        for layout in ("no_wide", "auto"):
            _set_layout(monkeypatch, layout)
            sizes[layout] = (lookup_bytes([okey_col, date]), lookup_bytes([okey_col, date, date]))
        assert _width(sizes) == 4, sizes
        _set_layout(monkeypatch, "auto")
        bridge = ops.JoinBridge()
        b = ops.HashBuilderOperatorFactory(ctx, bridge, [0], [1], n_orders).create_operator()
        b.add_input(ops.DevicePage([okey_col, date], n_orders))
        b.finish()
        j = ops.LookupJoinOperatorFactory(ctx, bridge, abi.JOIN_INNER, False, [0], [0, 1]).create_operator()
        probe = ops.DevicePage([ops.DeviceColumn(abi.INT64, d_lkeys, n), ops.DeviceColumn(abi.FLOAT64, d_price, n)], n)
        try:
            for _ in range(2):
                j.add_input(probe)
                out = j.get_output_device()
                assert out is not None and out.rows == n
                runs.append([ctx.to_host(out.column(c).ptr, dt, n) for c, dt in ((0, np.int64), (1, np.float64), (2, np.int64))])
                out.release()
        finally:
            j.close(); b.close(); bridge.lookup_source.close()
    finally:
        for p in (d_okeys, d_lkeys, d_date, d_price):
            ctx.free(p)
    assert np.array_equal(runs[0][0], lkeys)
    assert np.array_equal(runs[0][2], lkeys % 2557)
    for a, b_ in zip(runs[0], runs[1]):
        assert np.array_equal(a, b_)
