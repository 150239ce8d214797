"""The fused join probe records which probe rows matched as a bitmap (one bit per row, Arrow LSB order), and a build with one
payload column reads key and payload from one 16-byte keyed slot.  Every case is compared row for row, in order, with the oracle,
including which build cells are NULL under PROBE_OUTER (the bitmap is then those columns' validity)."""
import numpy as np
import pytest

from helpers import gpu_join_rows, oracle_join_rows, rows_equal
from trino_b200 import abi
from trino_b200 import operators as ops
from trino_b200.page import Block, Page

pytestmark = pytest.mark.gpu

SIZES = [1, 31, 32, 33, 1023, 1024, 1025, 4097, 300_001]
RATES = ["all", "none", "half", "last_miss"]
JOIN_TYPES = [abi.JOIN_INNER, abi.JOIN_PROBE_OUTER]
LAYOUTS = {"auto": {}, "no_wide": {"TGPU_JOIN_NO_WIDE": "1"}, "wide_always": {"TGPU_JOIN_WIDE": "always"}, "span": {"TGPU_JOIN_SPAN": "1"}}
PAYLOADS = ["tinyint", "smallint", "integer", "bigint", "bigint+integer", "double+smallint"]


def _payload_blocks(keys, names):
    cols = {"bigint": lambda: Block.bigint(keys * 7 - 1), "double": lambda: Block.double(keys * 0.25),
            "integer": lambda: Block.integer((keys % 100_003).astype(np.int32)), "smallint": lambda: Block.smallint((keys % 30_011).astype(np.int16)),
            "tinyint": lambda: Block.tinyint((keys % 113).astype(np.int8))}
    return [cols[n]() for n in names]


def _case(n, rate, order, seed=0):
    """build keys: even numbers of an order-key-like dense range; probe keys: build keys (hits) or odd numbers (misses)"""
    rng = np.random.default_rng(1000 + n + 7 * seed + len(rate))
    nb = 5000 + n // 4
    bkeys = (np.arange(nb, dtype=np.int64) * 2 + 2)
    hits = rng.choice(bkeys, n)
    misses = rng.integers(0, nb + 2, n) * 2 + 1
    if rate == "all":
        pkeys = hits
    elif rate == "none":
        pkeys = misses
    elif rate == "half":
        pkeys = np.where(rng.random(n) < 0.5, hits, misses)
    else:
        pkeys = hits.copy()
    if order == "ordered":
        pkeys = np.sort(pkeys)
    if rate == "last_miss":
        pkeys[-1] = bkeys[-1] + 1          # a single miss in the last word of the ragged tail, after every hit in key order
    return bkeys, pkeys.astype(np.int64)


def _device_page(ctx, page, types):
    cols = []
    for c, t in enumerate(types):
        arr = page.get_block(c).flatten().values
        cols.append(ops.DeviceColumn(t, ctx.to_device(arr), len(arr)))
    return ops.DevicePage(cols, page.position_count), cols


def _device_join_rows(ctx, build, probe, types, build_out, join_type):
    """like gpu_join_rows, with the probe page already resident on the device"""
    bridge = ops.JoinBridge()
    b = ops.HashBuilderOperatorFactory(ctx, bridge, [0], build_out).create_operator()
    b.add_input(build)
    b.finish()
    j = ops.LookupJoinOperatorFactory(ctx, bridge, join_type, False, [0], [0, 1]).create_operator()
    dp, cols = _device_page(ctx, probe, types)
    out = ops.drive(j, [dp])
    rows = []
    for page in out:
        rows.extend(page.rows())
    j.close(); b.close(); bridge.lookup_source.close()
    for c in cols:
        ctx.free(c.ptr)
    return rows


def _set_layout(monkeypatch, layout):
    for k in ("TGPU_JOIN_NO_WIDE", "TGPU_JOIN_WIDE", "TGPU_JOIN_SPAN", "TGPU_JOIN_WIDE_SHAPE"):
        monkeypatch.delenv(k, raising=False)
    for k, v in LAYOUTS[layout].items():
        monkeypatch.setenv(k, v)


@pytest.mark.parametrize("join_type", JOIN_TYPES)
@pytest.mark.parametrize("rate", RATES)
@pytest.mark.parametrize("n", SIZES)
def test_page_sizes_and_match_rates(ctx, monkeypatch, n, rate, join_type):
    """Warp (32), tile (1024) and ragged-tail boundaries, with every row, no row, about half and all but the last row matching."""
    _set_layout(monkeypatch, "auto")
    bkeys, pkeys = _case(n, rate, "ordered")
    build = Page(Block.bigint(bkeys), *_payload_blocks(bkeys, ["bigint"]))
    probe = Page(Block.bigint(pkeys), Block.double(pkeys * 0.5))
    want = oracle_join_rows(build, probe, 0, 0, [0, 1], [1], join_type, False)
    assert gpu_join_rows(ctx, [build], [probe], 0, 0, [0, 1], [1], join_type, False) == want
    assert _device_join_rows(ctx, build, probe, [abi.INT64, abi.FLOAT64], [1], join_type) == want
    assert gpu_join_rows(ctx, [build], [probe], 0, 0, [0, 1], [1], join_type, False, by_reference=True) == want


@pytest.mark.parametrize("join_type", JOIN_TYPES)
@pytest.mark.parametrize("payload", PAYLOADS)
@pytest.mark.parametrize("order", ["ordered", "shuffled"])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_layouts_and_payload_widths(ctx, monkeypatch, layout, order, payload, join_type):
    """One payload column of 1, 2, 4 or 8 bytes (the keyed table) and two columns (the wide table, or the narrow slots under NO_WIDE),
    key-ordered and shuffled probe pages, through every layout switch."""
    _set_layout(monkeypatch, layout)
    names = payload.split("+")
    build_out = list(range(1, 1 + len(names)))
    for n in (4097, 70_001):
        bkeys, pkeys = _case(n, "half", order, seed=len(payload))
        build = Page(Block.bigint(bkeys), *_payload_blocks(bkeys, names))
        probe = Page(Block.bigint(pkeys), Block.double(pkeys * 0.5))
        got = gpu_join_rows(ctx, [build], [probe], 0, 0, [0, 1], build_out, join_type, False)
        assert rows_equal(got, oracle_join_rows(build, probe, 0, 0, [0, 1], build_out, join_type, False)), (n, layout, order, payload)


@pytest.mark.parametrize("join_type", JOIN_TYPES)
@pytest.mark.parametrize("key", ["nullable_bigint", "integer"])
@pytest.mark.parametrize("n", [33, 1025, 300_001])
def test_whole_page_through_the_gather_kernel(ctx, key, n, join_type):
    """A nullable or INTEGER probe key sends the whole page through join_probe_gather_kernel (no lean tiles before it)."""
    bkeys, pkeys = _case(n, "half", "ordered", seed=3)
    rng = np.random.default_rng(n)
    if key == "integer":
        build = Page(Block.integer(bkeys.astype(np.int32)), *_payload_blocks(bkeys, ["bigint"]))
        probe = Page(Block.integer(pkeys.astype(np.int32)), Block.double(pkeys * 0.5))
    else:
        build = Page(Block.bigint(bkeys), *_payload_blocks(bkeys, ["bigint"]))
        probe = Page(Block.bigint(pkeys, rng.random(n) < 0.1), Block.double(pkeys * 0.5))
    want = oracle_join_rows(build, probe, 0, 0, [0, 1], [1], join_type, False)
    assert gpu_join_rows(ctx, [build], [probe], 0, 0, [0, 1], [1], join_type, False) == want


@pytest.mark.parametrize("join_type", JOIN_TYPES)
@pytest.mark.parametrize("build_has_min", [True, False])
@pytest.mark.parametrize("layout", ["auto", "no_wide", "wide_always"])
def test_int64_min_probe_key(ctx, monkeypatch, layout, build_has_min, join_type):
    """INT64_MIN lives beside the table (the keyed and wide tables keep its cell in slot mask + 1)."""
    _set_layout(monkeypatch, layout)
    bkeys, pkeys = _case(4097, "half", "ordered", seed=5)
    if build_has_min:
        bkeys = np.concatenate([[-2**63], bkeys]).astype(np.int64)
    pkeys = pkeys.copy()
    pkeys[::97] = -2**63
    build = Page(Block.bigint(bkeys), *_payload_blocks(bkeys, ["bigint"]))
    probe = Page(Block.bigint(pkeys), Block.double(pkeys.astype(np.float64)))
    want = oracle_join_rows(build, probe, 0, 0, [0, 1], [1], join_type, False)
    assert gpu_join_rows(ctx, [build], [probe], 0, 0, [0, 1], [1], join_type, False) == want


def test_shared_validity_outlives_the_next_page(ctx):
    """A PROBE_OUTER output page whose build-column validity IS the match bitmap keeps it after the next add_input."""
    bkeys, p1 = _case(4097, "half", "ordered", seed=7)
    _, p2 = _case(4097, "all", "ordered", seed=8)
    build = Page(Block.bigint(bkeys), *_payload_blocks(bkeys, ["bigint"]))
    probes = [Page(Block.bigint(p), Block.double(p * 0.5)) for p in (p1, p2)]
    bridge = ops.JoinBridge()
    b = ops.HashBuilderOperatorFactory(ctx, bridge, [0], [1]).create_operator()
    b.add_input(build)
    b.finish()
    j = ops.LookupJoinOperatorFactory(ctx, bridge, abi.JOIN_PROBE_OUTER, False, [0], [0, 1]).create_operator()
    j.add_input(probes[0])
    first = j.get_output_device()
    assert first is not None and first.column(2).validity
    j.add_input(probes[1])
    second = j.get_output_device()
    got_first = first.to_host().rows()
    first.release()
    second.release()
    j.close(); b.close(); bridge.lookup_source.close()
    assert got_first == oracle_join_rows(build, probes[0], 0, 0, [0, 1], [1], abi.JOIN_PROBE_OUTER, False)


def _lookup_bytes(ctx, build, build_out):
    bridge = ops.JoinBridge()
    b = ops.HashBuilderOperatorFactory(ctx, bridge, [0], build_out).create_operator()
    b.add_input(build)
    b.finish()
    v = bridge.lookup_source.get_in_memory_size_in_bytes()
    b.close(); bridge.lookup_source.close()
    return v


def test_one_column_build_carries_no_wide_table(ctx, monkeypatch):
    """A one-column build's table with payload is the 16-byte keyed table, half the 32-byte wide table that it carried before and
    that a two-column build of the same keys still carries (same keys, same capacity)."""
    bkeys, _ = _case(300_001, "all", "ordered")
    one = Page(Block.bigint(bkeys), *_payload_blocks(bkeys, ["bigint"]))
    two = Page(Block.bigint(bkeys), *_payload_blocks(bkeys, ["bigint", "integer"]))
    sizes = {}
    for layout in ("auto", "no_wide"):
        _set_layout(monkeypatch, layout)
        sizes[layout] = (_lookup_bytes(ctx, one, [1]), _lookup_bytes(ctx, two, [1, 2]))
    keyed = sizes["auto"][0] - sizes["no_wide"][0]
    wide = sizes["auto"][1] - sizes["no_wide"][1]
    assert 0 < keyed < wide, sizes
    assert sizes["auto"][0] < sizes["no_wide"][0] + wide, sizes      # the one-column build with a 32-byte wide table, as before
