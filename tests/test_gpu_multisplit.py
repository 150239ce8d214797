"""GPU parity of the PagePartitioner's stable multi-split (csrc/multisplit.cuh) against an exact host reference, form by form.

A fixed-width page with at most 64 partitions is split by a histogram pass, xchg_offsets_kernel and one scatter pass, and
xchg_launch_scatter picks the scatter's form from the page's shape.  FORMS below names every form, the page shape (or switch) that
reaches it and the kernels it launches; test_every_form_launches_its_kernels checks that mapping with the profiler.

Reference: the keys of a page are drawn from a pool of candidate keys whose partition ids the CPU oracle computes once, so a row's
expected partition is pool_ids[idx].  Partition q's page must hold every column's rows with id q, in input order, moved bit for bit
(DOUBLE / REAL compared as integers: NaN payloads, -0.0 and denormals must survive), with the NULL mask exact and values compared where
they are not NULL.  Skewed pages draw their keys from the candidates of one partition only.

The chunk geometry of the kernels depends on the SM count: `geometry` restates xchg_geom, and every multi-tile case asserts the shape
it was sized for before it runs, so that a card with another SM count cannot quietly turn it into a one-tile case.
"""
import ctypes as C
import functools
import json
import os
import subprocess
import sys
import zlib
from dataclasses import dataclass

import numpy as np
import pytest

import oracle_lib as o
from helpers import kernels_launched as _kernels_launched
from trino_b200 import abi
from trino_b200 import operators as ops
from trino_b200.page import Block, Page

pytestmark = pytest.mark.gpu

INT64_MIN, INT64_MAX = np.iinfo(np.int64).min, np.iinfo(np.int64).max
SWITCHES = ("TGPU_XCHG_CTA", "TGPU_XCHG_NO_LEAN", "TGPU_XCHG_LEAN_MINB", "TGPU_XCHG_PID_ARRAY", "TGPU_PARTITION_SORT")
PATTERNS = ("uniform", "all_first", "all_last", "runs256", "lanes8")
INT_VIEW = {8: np.int64, 4: np.int32, 2: np.int16, 1: np.int8}
VALUE_TYPES = {"B": abi.INT64, "D": abi.FLOAT64, "I": abi.INT32, "S": abi.INT16, "T": abi.INT8, "R": abi.FLOAT32}
DOUBLE_SPECIALS = [0x8000000000000000, 0x7FF8000000000001, 0xFFF0000000000001, 0x7FF4000000000000, 0x0000000000000001, 0x800FFFFFFFFFFFFF,
                   0x7FF0000000000000, 0xFFF0000000000000, 0x7FFFFFFFFFFFFFFF]
REAL_SPECIALS = [0x80000000, 0x7FC00001, 0xFF800001, 0x7FA00000, 0x00000001, 0x807FFFFF, 0x7F800000, 0xFFFFFFFF]


# ---- launch geometry (xchg_geom and tg_grid in csrc/) --------------------------------------------------------------------------
@functools.lru_cache(None)
def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _cdiv(a, b):
    return -(-a // b)


@dataclass(frozen=True)
class Geometry:
    warp_mode: bool
    warps: int            # warp mode: warps of the grid (sm_count x 12 CTAs x 8 warps); CTA mode: the grid
    chunk: int            # rows per warp (CTA) chunk
    nchunks: int
    tile: int             # rows per tile: 256 per warp, 2048 per CTA
    tiles: int            # tiles per full chunk
    last_chunk_rows: int
    hist_trips: int       # trips of 256 rows per chunk in xchg_hist_warp_kernel (its byte counters are flushed after 31)


def geometry(n, P, cta=False):
    sm = sm_count()
    n = max(n, 1)
    if P <= 8 and not cta:
        warps = sm * 12 * 8
        chunk = _cdiv(_cdiv(n, warps), 256) * 256
        tile = 256
    else:
        warps = min(_cdiv(n, 256 * 16), sm * 8)
        chunk = _cdiv(_cdiv(n, warps), 256) * 256
        tile = 2048
    nchunks = max(1, _cdiv(n, chunk))
    return Geometry(P <= 8 and not cta, warps, chunk, nchunks, tile, _cdiv(chunk, tile), n - (nchunks - 1) * chunk, chunk // 256)


def size_of(label):
    """Page sizes named after the geometry they are meant to produce (asserted by check_geometry)."""
    sm = sm_count()
    warps = sm * 12 * 8
    return {"two_tiles": 512 * (warps - 3) - 77,          # 2 tiles per warp chunk, nchunks % 8 != 0, a ragged last tile
            "w256": warps * 256,                           # exactly one full tile per warp
            "w256p1": warps * 256 + 1,                     # the chunk doubles; the last chunk holds one row
            "cta_tiles": 3 * 2048 * 8 * sm + 4999,         # CTA chunks of 3 full 2048-row tiles and a ragged fourth
            "large": 32 * warps * 256 + 4097}[label]       # 33 tiles and 33 histogram trips per warp chunk


def check_geometry(label, n, P, cta):
    g = geometry(n, P, cta)
    ok = {"two_tiles": lambda: g.warp_mode and g.tiles == 2 and g.nchunks % 8 != 0 and 256 < g.last_chunk_rows < 512,
          "w256": lambda: g.warp_mode and g.tiles == 1 and g.nchunks == g.warps and g.last_chunk_rows == 256,
          "w256p1": lambda: g.warp_mode and g.tiles == 2 and g.last_chunk_rows == 1,
          "cta_tiles": lambda: not g.warp_mode and g.tiles >= 3 and g.chunk % 2048 and g.last_chunk_rows % 2048,
          "large": lambda: g.warp_mode and g.tiles >= 33 and g.hist_trips >= 32 and g.last_chunk_rows % 256}[label]()
    assert ok, (label, n, P, g)
    return g


# ---- partitioning functions --------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Config:
    fn: str               # "hash" (bucket function) or "local" (LocalPartitionGenerator)
    buckets: int
    b2p: tuple = None

    @property
    def P(self):
        return max(self.b2p) + 1 if self.b2p else self.buckets


_GAP40 = [q for q in range(40) if q != 17]
CONFIGS = {**{"hash%d" % p: Config("hash", p) for p in (2, 3, 4, 5, 6, 7, 8, 9, 37, 64, 65)},
           "gap8": Config("hash", 32, tuple([0, 2, 3, 4, 5, 6, 7][b % 7] for b in range(32))),    # partition 1 stays empty
           "last8": Config("hash", 16, (7,) * 16),                                                   # every bucket to partition 7
           "gap40": Config("hash", 96, tuple(_GAP40[b % 39] for b in range(96))),                    # 40 partitions, 17 empty
           **{"local%d" % p: Config("local", p) for p in (2, 4, 8)}}


def make_operator(ctx, keys, cfg):
    fn = abi.PARTITION_LOCAL if cfg.fn == "local" else abi.PARTITION_HASH_BUCKET
    return ops.PartitionedOutputOperatorFactory(ctx, keys, cfg.buckets, list(cfg.b2p) if cfg.b2p else None, -1, False,
                                                partition_function=fn).create_operator()


# ---- the forms -----------------------------------------------------------------------------------------------------------------
HW_T, HW_F, OFF = "xchg_hist_warp_kernel<true>", "xchg_hist_warp_kernel<false>", "xchg_offsets_kernel"
CTA_HIST, CTA_SCATTER, IDS = "xchg_hist_kernel(", "xchg_scatter_kernel<4>", "partition_ids_kernel"


def LEAN(nc, minb):
    return "xchg_scatter_lean8_kernel<%d,%d>" % (nc, minb)


def WARP(vec, keys):
    return "xchg_scatter_warp_kernel<%s,%s>" % (str(vec).lower(), str(keys).lower())


@dataclass(frozen=True)
class Form:
    """A page shape and the kernels it launches.  Column codes: K plain BIGINT key, K? BIGINT key with a validity buffer, KD DOUBLE key,
    KI second (INTEGER) key column; values B BIGINT, D DOUBLE, I INTEGER, S SMALLINT, T TINYINT, R REAL, '?' = nullable (30 % NULL).
    `shift`: (channel, bytes) - a device page whose column starts that many bytes past its allocation.  `mode` picks the partition
    counts and sizes it runs over (MODE_CONFIGS, MULTI_PLAN)."""
    name: str
    cols: tuple
    mode: str
    kernels: tuple
    env: tuple = ()
    shift: tuple = ()
    absent: tuple = ()

    @property
    def kind(self):
        return "bigint_null" if "K?" in self.cols else "double" if "KD" in self.cols else "pair" if "KI" in self.cols else "bigint"

    @property
    def keys(self):
        return [self.cols.index(c) for c in ("K", "K?", "KD", "KI") if c in self.cols]

    @property
    def multisplit(self):
        return "xchg_" not in self.absent


_LANES48 = ("K?",) + tuple("BDISTR"[i % 6] + "?" for i in range(23))      # 24 nullable columns = 48 lanes (XMAXC)
FORMS = [
    # one plain BIGINT key, every lane an aligned 8-byte column without NULLs, <= 4 lanes: ids recomputed from the key
    Form("lean1", ("K",), "warp", (HW_T, OFF, LEAN(1, 3))),
    Form("lean2_key1", ("D", "K"), "warp", (HW_T, LEAN(2, 3))),
    Form("lean3_key2", ("B", "D", "K"), "warp", (HW_T, LEAN(3, 3))),
    Form("lean4_key3", ("D", "B", "D", "K"), "warp", (HW_T, LEAN(4, 3))),
    Form("lean4_key0", ("K", "D", "B", "D"), "warp", (HW_T, LEAN(4, 3))),
    Form("lean1_minb2", ("K",), "warp", (HW_T, LEAN(1, 2)), env=(("TGPU_XCHG_LEAN_MINB", "2"),)),
    Form("lean2_minb2", ("K", "D"), "warp", (HW_T, LEAN(2, 2)), env=(("TGPU_XCHG_LEAN_MINB", "2"),)),
    Form("lean3_minb4", ("B", "K", "D"), "warp", (HW_T, LEAN(3, 4)), env=(("TGPU_XCHG_LEAN_MINB", "4"),)),
    Form("lean4_minb4", ("D", "D", "B", "K"), "warp", (HW_T, LEAN(4, 4)), env=(("TGPU_XCHG_LEAN_MINB", "4"),)),
    # plain key, ids recomputed, generic warp scatter: narrow lanes, a NULL-byte lane, more than 4 lanes, or the lean form switched off
    Form("keys_narrow", ("K", "I", "S", "T", "R"), "warp", (HW_T, WARP(True, True))),
    Form("keys_nullable_value", ("D?", "K"), "warp", (HW_T, WARP(True, True))),
    Form("keys_five_lanes", ("K", "B", "D", "B", "D"), "warp", (HW_T, WARP(True, True))),
    Form("keys_no_lean", ("K", "D"), "warp", (HW_T, WARP(True, True)), env=(("TGPU_XCHG_NO_LEAN", "1"),)),
    Form("keys_unaligned_key", ("K", "D"), "warp", (HW_T, WARP(False, True)), shift=((0, 8),)),
    Form("keys_unaligned_value", ("K", "D"), "warp", (HW_T, WARP(False, True)), shift=((1, 8),)),
    # the 1-byte id array between the passes
    Form("ids_pid_array", ("K", "D"), "warp", (HW_T, WARP(True, False)), env=(("TGPU_XCHG_PID_ARRAY", "1"),)),
    Form("ids_pid_array_unaligned", ("K", "D", "B"), "warp", (HW_T, WARP(False, False)), env=(("TGPU_XCHG_PID_ARRAY", "1"),), shift=((1, 8),)),
    Form("ids_nullable_key", ("K?", "D", "I"), "warp", (HW_F, WARP(True, False))),
    Form("ids_nullable_key_unaligned", ("K?", "D"), "warp", (HW_F, WARP(False, False)), shift=((1, 8),)),
    Form("ids_double_key", ("KD", "B", "R?"), "warp", (HW_F, WARP(True, False))),
    Form("ids_two_keys", ("K", "D", "KI"), "warp", (HW_F, WARP(True, False))),
    # LocalPartitionGenerator's function recomputed per row in the scatter (process_raw_hash with a negative count)
    Form("local_lean", ("K", "D"), "local", (HW_T, LEAN(2, 3))),
    Form("local_keys_narrow", ("K", "I", "D?"), "local", (HW_T, WARP(True, True))),
    # CTA-granular kernels: <= 8 partitions under the switch (register counters in the histogram), and more than 8 partitions
    Form("cta_plain_key", ("K", "D?", "S", "T"), "cta", (CTA_HIST, OFF, CTA_SCATTER), env=(("TGPU_XCHG_CTA", "1"),)),
    Form("cta_nullable_key", ("K?", "R", "B"), "cta", (CTA_HIST, CTA_SCATTER), env=(("TGPU_XCHG_CTA", "1"),)),
    Form("cta_wide", ("K", "D?", "I"), "wide", (CTA_HIST, OFF, CTA_SCATTER)),
    Form("cta_wide_two_keys", ("K", "KI", "D"), "wide", (CTA_HIST, CTA_SCATTER)),
    # the lane limit: 24 nullable columns take the multi-split, 25 the sort path
    Form("lanes48", _LANES48, "lanes", (HW_F, WARP(True, False))),
    Form("lanes50", _LANES48 + ("B?",), "lanes", (IDS,), absent=("xchg_",)),
    # the sort + gather strategy: more than 64 partitions, or the switch
    Form("sort_65", ("K", "D?", "I"), "sort", (IDS,), absent=("xchg_",)),
    Form("sort_switch", ("K", "D", "I?"), "warp", (IDS,), env=(("TGPU_PARTITION_SORT", "1"),), absent=("xchg_",)),
]
FORM_BY_NAME = {f.name: f for f in FORMS}

MODE_CONFIGS = {"warp": ("hash2", "hash3", "hash5", "hash8", "gap8", "last8"),
                "local": ("local2", "local4", "local8"),
                "cta": ("hash2", "hash3", "hash4", "hash5", "hash6", "hash7", "hash8", "gap8", "last8"),
                "wide": ("hash9", "hash37", "hash64", "gap40"),
                "lanes": ("hash3", "hash8"),
                "sort": ("hash65",)}
ROUTE_CONFIG = {"warp": "hash8", "local": "local8", "cta": "hash8", "wide": "hash37", "lanes": "hash8", "sort": "hash65"}
# multi-tile cases per mode: (size, config, patterns)
MULTI_PLAN = {"warp": (("two_tiles", "hash8", PATTERNS), ("two_tiles", "hash3", ("uniform",)), ("two_tiles", "gap8", ("lanes8",)),
                       ("two_tiles", "last8", ("uniform",)), ("w256", "hash8", ("uniform",)), ("w256p1", "hash5", ("runs256",))),
              "local": (("two_tiles", "local8", PATTERNS), ("two_tiles", "local2", ("uniform",)), ("w256p1", "local4", ("runs256",))),
              "cta": (("cta_tiles", "hash8", PATTERNS), ("cta_tiles", "hash3", ("uniform",)), ("cta_tiles", "last8", ("uniform",))),
              "wide": (("cta_tiles", "hash64", ("uniform", "all_last", "lanes8")), ("cta_tiles", "hash9", ("uniform", "runs256")),
                       ("cta_tiles", "gap40", ("uniform",))),
              "lanes": (("w256p1", "hash8", ("uniform",)),),
              "sort": (("two_tiles", "hash65", ("uniform",)),)}


# ---- data ----------------------------------------------------------------------------------------------------------------------
N_CAND, N_POOL = 1 << 17, 1 << 16


def _seed(*parts):
    return zlib.crc32(repr(parts).encode())


def _distinct_first(values):
    """values with later duplicates dropped, order kept"""
    _, first = np.unique(values, return_index=True)
    return values[np.sort(first)]


@functools.lru_cache(None)
def candidates(kind):
    """N_CAND candidate keys (a list of (type, values, nulls) key columns).  The first N_POOL are the uniform pool; INT64_MIN,
    INT64_MAX, 0 and -1 (DOUBLE: both zeros, NaN payloads, denormals, infinities) lead it."""
    rng = np.random.default_rng(_seed("candidates", kind))
    if kind == "double":
        bits = np.concatenate([np.array(DOUBLE_SPECIALS, dtype=np.uint64).view(np.int64), np.zeros(1, np.int64),
                               rng.integers(INT64_MIN, INT64_MAX, 2 * N_CAND, dtype=np.int64, endpoint=True)])
        return [(abi.FLOAT64, _distinct_first(bits)[:N_CAND].view(np.float64), None)]
    specials = np.array([INT64_MIN, INT64_MAX, 0, -1, 1, INT64_MIN + 1, INT64_MAX - 1], dtype=np.int64)
    rest = np.concatenate([rng.integers(-(1 << 20), 1 << 20, N_CAND // 4), rng.integers(INT64_MIN, INT64_MAX, 2 * N_CAND, dtype=np.int64, endpoint=True)])
    rng.shuffle(rest)
    vals = _distinct_first(np.concatenate([specials, rest]))[:N_CAND]
    if kind == "bigint":
        return [(abi.INT64, vals, None)]
    if kind == "bigint_null":
        nulls = rng.random(N_CAND) < 0.05
        nulls[:len(specials)] = False
        return [(abi.INT64, vals, nulls)]
    assert kind == "pair"
    return [(abi.INT64, vals, None), (abi.INT32, rng.integers(-(1 << 31), 1 << 31, N_CAND, dtype=np.int32), None)]


def _block(typ, values, nulls):
    b = Block(typ, values, nulls)
    b.nulls = nulls       # (a validity buffer even without NULLs: the shape, not the data, picks the kernel form)
    return b


@functools.lru_cache(None)
def pool_ids(kind, cfg_name):
    """the oracle's partition id of every candidate key"""
    cfg = CONFIGS[cfg_name]
    page = Page(*[_block(*c) for c in candidates(kind)])
    if cfg.fn == "local":
        return o.local_partition_ids(page, [0], cfg.P).astype(np.uint8)
    return o.partition_ids(page, list(range(page.channel_count)), cfg.buckets, list(cfg.b2p) if cfg.b2p else None).astype(np.uint8)


@functools.lru_cache(None)
def subpools(kind, cfg_name):
    ids = pool_ids(kind, cfg_name)
    return {q: np.flatnonzero(ids == q) for q in range(CONFIGS[cfg_name].P) if (ids == q).any()}


def patterns_of(kind, cfg_name, wanted=PATTERNS):
    """skewed patterns need two non-empty partitions to differ from the uniform one"""
    return [p for p in wanted if p == "uniform" or len(subpools(kind, cfg_name)) > 1]


@functools.lru_cache(maxsize=10)
def key_rows(n, kind, cfg_name, pattern):
    """(candidate index per row, partition id per row, the rows in (partition, position) order)"""
    rng = np.random.default_rng(_seed("keys", n, kind, cfg_name, pattern))
    if pattern == "uniform":
        idx = rng.integers(0, N_POOL, n).astype(np.int32)
    else:
        sub = subpools(kind, cfg_name)
        present = sorted(sub)
        r = np.arange(n)
        target = {"all_first": np.full(n, present[0]), "all_last": np.full(n, present[-1]),
                  "runs256": np.where((r >> 8) & 1, present[0], present[-1]),            # 256-row runs alternating between two partitions
                  "lanes8": np.array(present[::-1])[(r >> 3) % len(present)]}[pattern]  # every 8-row group (one lane's rows) in one partition
        idx = np.empty(n, dtype=np.int32)
        for q in np.unique(target):
            m = target == q
            idx[m] = sub[q][rng.integers(0, len(sub[q]), int(m.sum()))]
    ids = pool_ids(kind, cfg_name)[idx]
    return idx, ids, np.argsort(ids, kind="stable")


@functools.lru_cache(maxsize=16)
def value_column(n, code, channel):
    rng = np.random.default_rng(_seed("values", n, code, channel))
    base = code[0]
    if base in "BD":
        v = rng.integers(INT64_MIN, INT64_MAX, n, dtype=np.int64, endpoint=True)
        specials = np.array(DOUBLE_SPECIALS, dtype=np.uint64).view(np.int64) if base == "D" else np.array([INT64_MIN, INT64_MAX, 0, -1], dtype=np.int64)
        v[channel::97] = np.resize(specials, len(v[channel::97]))
        v = v.view(np.float64) if base == "D" else v
    elif base in "IR":
        v = rng.integers(-(1 << 31), 1 << 31, n, dtype=np.int32)
        if base == "R":
            v[channel::89] = np.resize(np.array(REAL_SPECIALS, dtype=np.uint32).view(np.int32), len(v[channel::89]))
            v = v.view(np.float32)
    else:
        dt = np.int16 if base == "S" else np.int8
        v = rng.integers(np.iinfo(dt).min, np.iinfo(dt).max, n, dtype=dt, endpoint=True)
    nulls = rng.random(n) < 0.3 if code.endswith("?") else None
    return VALUE_TYPES[base], v, nulls


def clear_caches():
    key_rows.cache_clear()
    value_column.cache_clear()


def page_columns(form, n, cfg_name, pattern):
    """the form's columns as (type, values, nulls), the reference partition ids and the rows in (partition, position) order"""
    idx, ids, order = key_rows(n, form.kind, cfg_name, pattern)
    keycols = candidates(form.kind)
    cols = []
    for ch, code in enumerate(form.cols):
        if code.startswith("K"):
            typ, v, nulls = keycols[1 if code == "KI" else 0]
            cols.append((typ, v[idx], None if nulls is None else nulls[idx]))
        else:
            cols.append(value_column(n, code, ch))
    return cols, ids, order


def host_page(cols):
    return Page(*[_block(*c) for c in cols])


def device_page(ctx, cols, shift, n):
    """columns uploaded to ctx.malloc allocations; a shifted column starts `bytes` past its allocation"""
    shift = dict(shift)
    ptrs, dcols = [], []
    for ch, (typ, v, nulls) in enumerate(cols):
        s = shift.get(ch, 0)
        raw = v.view(np.uint8)
        p = ctx.to_device(np.concatenate([np.zeros(s, np.uint8), raw]) if s else raw)
        ptrs.append(p)
        if s:
            assert (p + s) % 16 == s % 16 != 0
        vp = None
        if nulls is not None:
            vp = ctx.to_device(np.packbits(~nulls, bitorder="little"))
            ptrs.append(vp)
        dcols.append(ops.DeviceColumn(typ, p + s, n, vp))
    return ops.DevicePage(dcols, n), ptrs


# ---- running and checking ------------------------------------------------------------------------------------------------------
def drain(op):
    got = []
    while True:
        r = op.get_output_with_partition()
        if r is None:
            return got
        got.append(r)


def check_page(page, q, cols, sel, label):
    """partition q's output page against the input rows `sel`, bit for bit"""
    assert page.position_count == len(sel), (label, q, page.position_count, len(sel))
    for c, (typ, v, nulls) in enumerate(cols):
        blk = page.get_block(c)
        assert blk.type == typ, (label, q, c)
        want_nulls = None if nulls is None else nulls[sel]
        if want_nulls is None or not want_nulls.any():
            assert blk.nulls is None or not blk.nulls.any(), (label, q, c, "NULLs where the input has none")
            keep = None
        else:
            assert blk.nulls is not None and np.array_equal(blk.nulls, want_nulls), (label, q, c, "NULL mask")
            keep = ~want_nulls
        iv = INT_VIEW[v.itemsize]
        want, got = v.view(iv)[sel], blk.values.view(iv)
        if keep is not None:
            want, got = want[keep], got[keep]
        if not np.array_equal(got, want):
            bad = int(np.flatnonzero(got != want)[0])
            raise AssertionError("%s: partition %d column %d value %d of %d: got %#x, want %#x" % (label, q, c, bad, len(want), int(got[bad]), int(want[bad])))


def check_pages(got, cols, ids, order, P, label):
    """one page per non-empty partition, in partition order, each holding that partition's rows in input order"""
    counts = np.bincount(ids, minlength=P)
    assert [q for q, _ in got] == [q for q in range(P) if counts[q]], (label, [q for q, _ in got], counts.tolist())
    offs = np.concatenate([[0], np.cumsum(counts)])
    for q, page in got:
        check_page(page, q, cols, order[offs[q]:offs[q + 1]], label)


def run_case(ctx, form, cfg_name, n, pattern, check_ids=False):
    cfg = CONFIGS[cfg_name]
    cols, ids, order = page_columns(form, n, cfg_name, pattern)
    label = "%s %s n=%d %s" % (form.name, cfg_name, n, pattern)
    op = make_operator(ctx, form.keys, cfg)
    ptrs = []
    try:
        if form.shift:
            page, ptrs = device_page(ctx, cols, form.shift, n)
        else:
            page = host_page(cols)
        op.add_input(page)
        got = drain(op)
        if check_ids and not form.shift:
            assert np.array_equal(op.get_partitions(page), ids), (label, "get_partitions")
    finally:
        op.close()
        for p in ptrs:
            ctx.free(p)
    check_pages(got, cols, ids, order, cfg.P, label)


@pytest.fixture
def switches(monkeypatch):
    """no tuning switch inherited from the environment; `apply(env)` sets exactly the given ones (read on every add_input)"""
    def apply(env=()):
        for s in SWITCHES:
            monkeypatch.delenv(s, raising=False)
        for k, v in env:
            monkeypatch.setenv(k, v)
    apply()
    return apply


def small_sizes(P):
    # 2P - 1 rows take the row-wise strategy (a control); 2P is the smallest multi-split page
    return (2 * P - 1, 2 * P, 255, 256, 257, 8 * 1024 + 3)


# ---- the form matrix -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("form", FORMS, ids=lambda f: f.name)
def test_small_pages(ctx, switches, form):
    """Every form at 2P - 1, 2P, 255, 256, 257 and 8195 rows, every partition count of its mode, uniform and skewed keys.  Catches: rows
    of a ragged tile (or of the lanes past the page end) given a partition; a rank or tile offset that is wrong when a lane's 8 rows or a
    whole tile share a partition (4-bit fields of 8, 16-bit fields of 256); the top 3- and 4-bit fields (partition 7); an empty
    partition that still emits a page; a key channel other than 0 read as the key; a lane staged from the wrong source column.
    CTA forms already hold two 2048-row tiles per chunk at 8195 rows (asserted)."""
    switches(form.env)
    if form.mode in ("cta", "wide"):
        g = geometry(8 * 1024 + 3, 8 if form.mode == "cta" else 9, cta=True)
        assert g.tiles == 2 and g.chunk % 2048 and g.nchunks > 1, g
    for cfg_name in MODE_CONFIGS[form.mode]:
        for n in small_sizes(CONFIGS[cfg_name].P):
            for pattern in patterns_of(form.kind, cfg_name):
                run_case(ctx, form, cfg_name, n, pattern)


@pytest.mark.parametrize("form", FORMS, ids=lambda f: f.name)
def test_multi_tile_pages(ctx, switches, form):
    """Every form at sizes whose warp chunks hold two 256-row tiles (or CTA chunks three 2048-row tiles and a ragged fourth), with a
    ragged last tile and a grid whose last CTA is partly idle; skewed keys at P = 8.  Catches: a per-partition running offset not carried
    from one tile of a chunk to the next; a chunk's block offset taken from the wrong chunk; a ragged last tile of a multi-tile chunk;
    a warp past the last chunk that writes.  get_partitions (partition_ids_kernel) is checked against the same reference."""
    switches(form.env)
    for label, cfg_name, wanted in MULTI_PLAN[form.mode]:
        n = size_of(label)
        if form.multisplit:
            check_geometry(label, n, CONFIGS[cfg_name].P, form.mode == "cta")
        for pattern in patterns_of(form.kind, cfg_name, wanted):
            run_case(ctx, form, cfg_name, n, pattern, check_ids=pattern == "uniform")


def test_large_page_crosses_the_histogram_flush(ctx, switches):
    """One key-only BIGINT page of ~104 M rows (on 132 SMs) whose warp chunks hold 33 tiles, every row in partition 7: each lane's byte
    counter for partition 7 gains 8 per trip and must be flushed after 31 trips.  Run through lean8<1,3> and through the id-array path
    (xchg_hist_warp_kernel<true> writing ids, xchg_scatter_warp_kernel<true,false>).  The one output page must be the input.  Catches: a
    byte counter that wraps at 256 rows; a flush that drops or double-counts; a running offset lost after many tiles."""
    clear_caches()
    n = size_of("large")
    check_geometry("large", n, 8, False)
    sub = subpools("bigint", "hash8")[7][:N_POOL]
    keys = candidates("bigint")[0][1][sub][np.random.default_rng(_seed("large")).integers(0, len(sub), n, dtype=np.uint16)]
    page = Page(Block.bigint(keys))
    op = make_operator(ctx, [0], CONFIGS["hash8"])
    try:
        for env in ((), (("TGPU_XCHG_PID_ARRAY", "1"),)):
            switches(env)
            op.add_input(page)
            r = op.get_output_with_partition()
            assert r is not None and r[0] == 7 and r[1].position_count == n, env
            assert np.array_equal(r[1].get_block(0).values, keys), env
            del r
            assert op.get_output() is None
        assert (op.get_partitions(page) == 7).all()
    finally:
        op.close()


# ---- operator-level cases: the output pages of one page alias one buffer per column -----------------------------------------------
def _device_outputs(ctx, op, limit=None):
    """(partition, DeviceOutputPage) of the next `limit` (all) output pages"""
    outs = []
    while limit is None or len(outs) < limit:
        d = op.get_output_device()
        if d is None:
            break
        q = C.c_int32()
        ctx.check(ctx.lib.tgpu_partition_last_output_partition(op.h, C.byref(q)))
        outs.append((q.value, d))
    return outs


@pytest.mark.parametrize("order", ["reverse", "interleaved"])
def test_output_pages_released_in_any_order(ctx, switches, order):
    """Partition pages of one page are slices of one buffer per column (and one per NULL-byte lane).  Take every page with
    get_output_device and release them one by one.  After each release, partition another page of the same size (its input and output
    buffers come from the same allocator and block cache) and read every remaining page while those are live.  Catches: a release that
    frees the shared column buffer, or hands it back to the block cache, while sibling pages still point into it."""
    form = FORM_BY_NAME["keys_nullable_value"]
    switches(form.env)
    n = size_of("two_tiles")
    cols, ids, rows = page_columns(form, n, "hash8", "uniform")
    other = host_page(page_columns(form, n, "hash8", "all_last")[0])
    counts = np.bincount(ids, minlength=8)
    offs = np.concatenate([[0], np.cumsum(counts)])
    op = make_operator(ctx, form.keys, CONFIGS["hash8"])
    live = {}
    try:
        op.add_input(host_page(cols))
        live.update(enumerate(_device_outputs(ctx, op)))
        assert [q for q, _ in live.values()] == [q for q in range(8) if counts[q]]
        k = len(live)
        seq = list(range(k))[::-1] if order == "reverse" else list(range(1, k, 2)) + list(range(0, k, 2))[::-1]
        for i in seq:
            live.pop(i)[1].release()
            churn = make_operator(ctx, form.keys, CONFIGS["hash8"])
            try:
                churn.add_input(other)
                for q, d in live.values():
                    check_page(d.to_host(), q, cols, rows[offs[q]:offs[q + 1]], "after releasing page %d (%s)" % (i, order))
            finally:
                churn.close()
    finally:
        for _, d in live.values():
            d.release()
        op.close()


def test_next_page_waits_until_every_page_is_taken(ctx, switches):
    """Add a page and take three of its partition pages.  Until the rest are taken the operator needs no input, and adding the next
    page is refused (Operator.addInput, M/operator/Operator.java:49-53) without touching the pending pages.  Take the rest, add the next
    page: its outputs are its own, and every page of the first page still holds that page's rows.  Catches: a refused add_input that
    drops or overwrites pending pages; the next page's scatter writing into buffers that the first page's pages still use."""
    form = FORM_BY_NAME["lean2_key1"]
    switches(form.env)
    n1, n2 = size_of("w256p1"), 8 * 1024 + 3
    cols1, ids1, order1 = page_columns(form, n1, "hash8", "uniform")
    cols2, ids2, order2 = page_columns(form, n2, "hash8", "lanes8")
    counts1 = np.bincount(ids1, minlength=8)
    offs1 = np.concatenate([[0], np.cumsum(counts1)])
    op = make_operator(ctx, form.keys, CONFIGS["hash8"])
    taken = []

    def check_first(what):
        assert [q for q, _ in taken] == [q for q in range(8) if counts1[q]], what
        for q, d in taken:
            check_page(d.to_host(), q, cols1, order1[offs1[q]:offs1[q + 1]], what)

    try:
        op.add_input(host_page(cols1))
        taken += _device_outputs(ctx, op, 3)
        assert not op.needs_input()
        with pytest.raises(abi.TrinoGpuError, match="ILLEGAL_STATE"):
            op.add_input(host_page(cols2))
        taken += _device_outputs(ctx, op)
        assert op.needs_input()
        check_first("first page after a refused add_input")
        op.add_input(host_page(cols2))
        check_pages(drain(op), cols2, ids2, order2, 8, "second page")
        check_first("first page after the second")
    finally:
        for _, d in taken:
            d.release()
        op.close()


# ---- routing: the table above is what the pages launch -----------------------------------------------------------------------------
def routing_main():
    """Body of the routing test's child process: every form's 8195-row page (checked against the reference) observed by
    _kernels_launched; prints {form: kernel names, or None} as one JSON line."""
    ctx = ops.Context(0)
    launched = {}
    try:
        for form in FORMS:
            for s in SWITCHES:
                os.environ.pop(s, None)
            os.environ.update(dict(form.env))
            launched[form.name] = _kernels_launched(lambda: run_case(ctx, form, ROUTE_CONFIG[form.mode], 8 * 1024 + 3, "uniform"))
    finally:
        ctx.close()
    print(json.dumps(launched))


def test_every_form_launches_its_kernels():
    """For each form of FORMS, one 8195-row page under the profiler: the named instantiations are launched, and the sort-path forms
    launch no multi-split kernel.  The pages are also checked against the reference.  They run in a child process of their own: after
    profiler sessions of earlier tests in the same process, the profiler has been seen to record the library's copies but none of its
    kernels.  A form without a complete profiler session fails the test; the test skips only when no session delivers its markers."""
    tests_dir = os.path.dirname(os.path.abspath(__file__))
    env = {k: v for k, v in os.environ.items() if k not in SWITCHES}
    env["PYTHONPATH"] = os.pathsep.join([os.path.dirname(tests_dir), tests_dir] + ([env["PYTHONPATH"]] if env.get("PYTHONPATH") else []))
    args = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", "import test_gpu_multisplit as t; t.routing_main()"]
    r = subprocess.run(args, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    launched = json.loads(r.stdout.strip().splitlines()[-1])
    if all(names is None for names in launched.values()):
        pytest.skip("no profiler session recorded torch's own marker kernels, so the routing cannot be observed here")
    unobserved = [name for name, names in launched.items() if names is None]
    assert not unobserved, ("no complete profiler session", unobserved)
    wrong = {}
    for form in FORMS:
        names = launched[form.name]
        missing = [k for k in form.kernels if not any(k in nm for nm in names)]
        unexpected = [a for a in form.absent if any(a in nm for nm in names)]
        if missing or unexpected:
            wrong[form.name] = (missing, unexpected, names)
    assert not wrong, wrong
