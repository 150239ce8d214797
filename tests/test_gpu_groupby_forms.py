"""HashAggregationOperator (csrc/groupby.cu) form by form against the exact reference of agg_reference.py.

At run time the keyed operator picks one of several device forms from the plan, the page and a few switches.  FORMS names every form,
the page shape (`keys`), `expected_groups` or switch that reaches it, and the kernels it launches; test_every_form_launches_its_kernels
checks that mapping with the profiler.

  form                 reached by                                                       kernels
  S_L4 .. S_L32        <= 64 groups; 3 / 7 / 15 / 30 regular keys in one CTA force the   tg_agg_small_jit, agg_small_merge_kernel
                       key table of each CTA from L = 4 to 8, 16 and 32 slots (fewer
                       aggregates as L grows, so that the accumulators fit)
  S_scalar_*           TGPU_AGG_S_NO_VEC, or device columns that start one row past a    same (the scalar loader variant)
                       16-byte boundary
  S_width_refused      36 aggregates: (L + 2) x A x 256 threads x 8 bytes exceeds shared  tg_agg_general_jit, no path-S kernel
                       memory at L = 4
  S_spill              two pages on path S, then a page with 200 more groups            gf_migrate_kernel, then tg_agg_general_jit
  general_jit          expected_groups > 256                                            tg_agg_general_jit
  general_interpreted  TGPU_AGG_GENERAL_INTERPRETED                                     gf_page_kernel
  general_growth       expected_groups 300 (a 2^16-slot table), one page of 60 000 new   gf_rehash_kernel (deferred rows replayed)
                       groups: the table grows in the middle of the page
  multipass            TGPU_AGG_MULTIPASS (DOUBLE and hashed composite keys take it by   g_insert_kernel, g_accumulate_kernel
                       themselves: test_every_key_kind)
  sliced_copy_*        TGPU_AGG_SLICE_MIN_BYTES=0, TGPU_AGG_SLICE_BYTES=256 KiB,         gf_slice_hist_kernel + the any-order or the
                       +- TGPU_AGG_STABLE_SCATTER                                        stable multi-split scatter
  sliced_rowlist       the above + TGPU_AGG_ROWLIST_SLICES                              gf_slice_ids_kernel
  S_interpreted        a child process with TGPU_DISABLE_JIT=1 (jit_available() is       agg_small_kernel
                       decided once per process)

Every form runs every argument type (BIGINT, INTEGER, SMALLINT, TINYINT, DOUBLE) in an operator of its own, under count(*), count, sum,
avg, min and max, each without a mask and with a BOOLEAN mask that has NULLs, over pages of 1, 257, 0, 130, 515, 64 and 3001 rows
(n = 1, 2, 3 mod 4 for the tail of the four-row loader; a multi-CTA page).  The value column has no validity buffer, some NULLs, only
NULLs, a validity buffer without NULLs, or these four in turn across the pages of one operator (a channel gains and loses its bitmap,
so the path-S kernel is re-specialised and its dropped non-NULL counters are read back in the merge).  Values make every summation
order exact: DOUBLE values are k / 1024 with |k| < 2^30, integer values include the type's extremes (BIGINT stays within 2^40 so that
avg's double sum is exact), so sums and averages must match the reference bit for bit.
"""
import functools
import json
import math
import os
import struct
import subprocess
import sys
import zlib
from dataclasses import dataclass
from fractions import Fraction

import numpy as np
import pytest

from agg_reference import INT64_MAX, INT64_MIN, AggregateOverflow, aggregate
from helpers import kernels_launched
from trino_b200 import abi
from trino_b200 import operators as ops
from trino_b200.page import Block, Page

pytestmark = pytest.mark.gpu
A = ops.Aggregator
SWITCHES = ("TGPU_AGG_S_NO_VEC", "TGPU_AGG_S_MINB", "TGPU_AGG_GENERAL_INTERPRETED", "TGPU_AGG_MULTIPASS", "TGPU_AGG_SLICE_MIN_BYTES",
            "TGPU_AGG_SLICE_BYTES", "TGPU_AGG_STABLE_SCATTER", "TGPU_AGG_ROWLIST_SLICES", "TGPU_AGG_NO_SLICES", "TGPU_AGG_G_SIZE_PCT",
            "TGPU_AGG_G_MINB", "TGPU_AGG_G_ROWS")
FNS = (abi.AGG_COUNT_STAR, abi.AGG_COUNT, abi.AGG_SUM, abi.AGG_AVG, abi.AGG_MIN, abi.AGG_MAX)
ARGS = {"bigint": abi.INT64, "integer": abi.INT32, "smallint": abi.INT16, "tinyint": abi.INT8, "double": abi.FLOAT64}
ARG_NAME = {t: name for name, t in ARGS.items()}
MAKE = {abi.INT64: Block.bigint, abi.INT32: Block.integer, abi.INT16: Block.smallint, abi.INT8: Block.tinyint, abi.FLOAT64: Block.double}
SIZES = (1, 257, 0, 130, 515, 64, 3001)
SCENARIOS = ("none", "some", "all", "present", "mixed")

S_JIT, S_MERGE, G_JIT = "tg_agg_small_jit", "agg_small_merge_kernel", "tg_agg_general_jit"
NOT_S = (S_JIT, S_MERGE, "agg_small_kernel")
NOT_G = (G_JIT, "gf_", "g_insert", "g_accumulate")


@dataclass(frozen=True)
class Form:
    """`keys`: the key shape of the pages (s4 / s8 / s16 / s32: 3 / 7 / 15 / 30 regular BIGINT keys plus NULL and INT64_MIN; spill: s4
    then 200 more keys from the fourth page (the first after the empty one) on; many: 300 keys; growth: many, plus a 60 001-row page of new keys).  `plan`: the aggregate
    set (plan_of).  `offset`: every page as device columns that start one row into their allocation.  `nojit`: runs in a child process
    with TGPU_DISABLE_JIT=1."""
    name: str
    keys: str
    plan: str
    kernels: tuple
    absent: tuple = ()
    env: tuple = ()
    expected: int = 16
    offset: bool = False
    nojit: bool = False


_SLICED = (("TGPU_AGG_SLICE_MIN_BYTES", "0"), ("TGPU_AGG_SLICE_BYTES", str(256 << 10)))
FORMS = [
    Form("S_L4", "s4", "all", (S_JIT, S_MERGE), NOT_G),
    Form("S_L8", "s8", "L8", (S_JIT, S_MERGE), NOT_G),
    Form("S_L16", "s16", "L16", (S_JIT, S_MERGE), NOT_G),
    Form("S_L32", "s32", "L32", (S_JIT, S_MERGE), NOT_G),
    Form("S_scalar_env", "s4", "all", (S_JIT, S_MERGE), NOT_G, env=(("TGPU_AGG_S_NO_VEC", "1"),)),
    Form("S_scalar_offset", "s4", "all", (S_JIT, S_MERGE), NOT_G, offset=True),
    Form("S_width_refused", "s4", "wide", (G_JIT, "gf_gather_kernel"), NOT_S),
    Form("S_spill", "spill", "all", (S_JIT, S_MERGE, "gf_migrate_kernel", G_JIT, "gf_gather_kernel")),
    Form("general_jit", "many", "all", (G_JIT, "gf_gather_kernel"), NOT_S + ("gf_page_kernel", "g_insert", "gf_slice"), expected=1000),
    Form("general_interpreted", "many", "all", ("gf_page_kernel", "gf_gather_kernel"), NOT_S + (G_JIT,), env=(("TGPU_AGG_GENERAL_INTERPRETED", "1"),),
         expected=1000),
    Form("general_growth", "growth", "all", (G_JIT, "gf_rehash_kernel"), NOT_S, expected=300),
    Form("multipass", "many", "all", ("g_insert_kernel", "g_flag_kernel", "g_assign_kernel", "g_accumulate_kernel"), NOT_S + (G_JIT, "gf_"),
         env=(("TGPU_AGG_MULTIPASS", "1"),), expected=1000),
    Form("sliced_copy_any_order", "many", "all", ("gf_slice_hist_kernel", "xchg_scatter_unordered_kernel", G_JIT), NOT_S + ("gf_slice_ids",),
         env=_SLICED, expected=1000),
    Form("sliced_copy_stable", "many", "all", ("gf_slice_hist_kernel", "xchg_scatter_kernel", G_JIT), NOT_S + ("gf_slice_ids", "xchg_scatter_unordered"),
         env=_SLICED + (("TGPU_AGG_STABLE_SCATTER", "1"),), expected=1000),
    Form("sliced_rowlist", "many", "all", ("gf_slice_ids_kernel", G_JIT), NOT_S + ("gf_slice_hist",), env=_SLICED + (("TGPU_AGG_ROWLIST_SLICES", "1"),),
         expected=1000),
    Form("S_interpreted", "s4", "all", ("agg_small_kernel", S_MERGE), ("tg_agg_",) + NOT_G, nojit=True),
]
FORM_BY_NAME = {f.name: f for f in FORMS}


def plan_of(name, v=1, m=2, w=3):
    """aggregates (function, input channel, mask channel) over the page layout [key, v, mask, w]"""
    def arg(f, ch):
        return -1 if f == abi.AGG_COUNT_STAR else ch

    every = [(f, arg(f, v), mask) for mask in (-1, m) for f in FNS]
    return {"all": every,
            "L8": [(f, arg(f, v), -1) for f in FNS],
            "L16": [(f, arg(f, v), -1) for f in (abi.AGG_COUNT_STAR, abi.AGG_SUM, abi.AGG_MIN, abi.AGG_MAX)],
            "L32": [(abi.AGG_SUM, v, m), (abi.AGG_COUNT_STAR, -1, m)],     # 3 accumulator words: the only plan 34 slot sets hold
            # 34 - 38 accumulators: too many for 6 slot sets of 256 threads in shared memory, whatever the argument type
            "wide": every + [(f, arg(f, ch), mask) for ch in (w, m) for mask in (-1, m) for f in FNS]}[name]


def scenarios_of(form):
    if form.plan == "L32":
        return ("none",)              # a validity buffer keeps sum's non-NULL counter: 4 words no longer fit 34 slot sets
    if form.keys == "growth":
        return ("mixed",)
    return SCENARIOS


# ---- pages ---------------------------------------------------------------------------------------------------------------------
def _seed(*parts):
    return zlib.crc32(repr(parts).encode())


def _bits(x):
    return struct.unpack("<q", struct.pack("<d", x))[0]


def _double(bits):
    return struct.unpack("<d", struct.pack("<Q", bits & ((1 << 64) - 1)))[0]


@functools.lru_cache(None)
def regular_keys(count):
    """distinct BIGINT keys other than INT64_MIN, led by INT64_MAX, -1, 0, 1"""
    rng = np.random.default_rng(_seed("regular", count))
    head = [INT64_MAX, -1, 0, 1, INT64_MIN + 1]
    rest = rng.integers(INT64_MIN + 2, INT64_MAX, 2 * count + 16, dtype=np.int64).tolist()
    out = list(dict.fromkeys(head + rest))
    return out[:count]


def key_values(shape, page_index, n, rng):
    if shape == "growth" and n == 60_001:
        return [None] + regular_keys(60_300)[300:]
    regular = {"s4": 3, "s8": 7, "s16": 15, "s32": 30, "many": 300, "growth": 300}.get(shape)
    if shape == "spill":
        regular = 3 if page_index < 2 else 203
    pool = regular_keys(regular) + [None, INT64_MIN]
    keys = [pool[i] for i in rng.integers(0, len(pool), n)]
    if n >= len(pool) and shape != "many":
        head = list(pool)
        rng.shuffle(head)
        keys[:len(pool)] = head          # every key of the shape in this page (and in its first CTA)
    return keys


def value_block(arg, n, mode, rng, always_validity=False):
    if arg == abi.FLOAT64:
        v = rng.integers(-(1 << 30) + 1, 1 << 30, n) / 1024.0
    elif arg == abi.INT64:
        v = rng.integers(-(1 << 40), 1 << 40, n, dtype=np.int64)
    else:
        info = np.iinfo({abi.INT32: np.int32, abi.INT16: np.int16, abi.INT8: np.int8}[arg])
        v = rng.integers(info.min, info.max, n, endpoint=True).astype(info.dtype)
        v[::7] = info.min
        v[3::11] = info.max
    nulls = {"none": None, "some": rng.random(n) < 0.3, "all": np.ones(n, dtype=bool), "present": np.zeros(n, dtype=bool)}[mode]
    b = MAKE[arg](v, nulls)
    b.nulls = nulls          # (a validity buffer without NULLs too: the buffer, not the data, picks the kernel variant)
    if always_validity and b.nulls is None:
        b.nulls = np.zeros(n, dtype=bool)
    return b


def page_modes(scenario, count):
    cycle = ("none", "some", "all", "present")
    return [cycle[i % 4] if scenario == "mixed" else scenario for i in range(count)]


@functools.lru_cache(maxsize=64)
def case(shape, plan, arg, scenario):
    """(pages [key, v, mask, w], aggregates, reference rows or the AggregateOverflow)"""
    rng = np.random.default_rng(_seed("case", shape, plan, arg, scenario))
    sizes = SIZES[:4] + (60_001,) + SIZES[4:] if shape == "growth" else SIZES
    pages = []
    for i, (n, mode) in enumerate(zip(sizes, page_modes(scenario, len(sizes)))):
        key = Block.bigint(key_values(shape, i, n, rng))
        mask = Block.boolean(rng.random(n) < 0.6, rng.random(n) < 0.15)
        w = value_block(abi.FLOAT64, n, "some", rng, always_validity=True)
        pages.append(Page(key, value_block(arg, n, mode, rng), mask, w, position_count=n))
    aggs = plan_of(plan)
    return pages, aggs, aggregate(pages, [0], aggs)


# ---- running and checking ------------------------------------------------------------------------------------------------------
def device_page(ctx, page, keep):
    """the page as device columns that start one element past their allocation (never 16-byte aligned)"""
    cols = []
    for b in page.blocks:
        raw = np.ascontiguousarray(b.values)
        p = ctx.to_device(np.concatenate([np.zeros(1, raw.dtype), raw]))
        keep.append(p)
        vp = None
        if b.nulls is not None:
            vp = ctx.to_device(np.packbits(~b.nulls, bitorder="little"))
            keep.append(vp)
        cols.append(ops.DeviceColumn(b.type, p + raw.itemsize, page.position_count, vp))
    return ops.DevicePage(cols, page.position_count)


def run_operator(ctx, pages, key_channels, aggs, expected, offset=False):
    op = ops.HashAggregationOperatorFactory(ctx, key_channels, abi.STEP_SINGLE, [A(fn, ch, m) for fn, ch, m in aggs], expected).create_operator()
    keep = []
    try:
        if offset:
            pages = [device_page(ctx, p, keep) if p.position_count else p for p in pages]
        out = ops.drive(op, pages)
    finally:
        op.close()
        for p in keep:
            ctx.free(p)
    return [r for p in out for r in p.rows()]


def same(got, want, key):
    """exact comparison: integers by value, doubles by their bits (a NaN aggregate only has to be NaN: the device canonicalises the
    payload; a NaN key must be the first raw value), Fractions by the bits of their correctly rounded double"""
    if want is None:
        return got is None
    if isinstance(want, Fraction):
        return isinstance(got, float) and _bits(got) == _bits(float(want))
    if isinstance(want, float):
        if not isinstance(got, float):
            return False
        if want != want and not key:
            return got != got
        return _bits(got) == _bits(want)
    return type(got) is type(want) and got == want


def check_rows(got, want, nkeys, label):
    assert len(got) == len(want), (label, "groups", len(got), len(want))
    for g, (r, w) in enumerate(zip(got, want)):
        for c, (x, y) in enumerate(zip(r, w)):
            if not same(x, y, c < nkeys):
                raise AssertionError("%s: group %d column %d: got %r, want %r (row %r, reference %r)" % (label, g, c, x, y, r, w))


def run_form(ctx, form, arg, scenario):
    pages, aggs, want = case(form.keys, form.plan, arg, scenario)
    got = run_operator(ctx, pages, [0], aggs, form.expected, form.offset)
    check_rows(got, want, 1, "%s %s %s" % (form.name, ARG_NAME[arg], scenario))


def apply_switches(env):
    for s in SWITCHES:
        os.environ.pop(s, None)
    os.environ.update(dict(env))


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


# ---- the form matrix -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("arg", list(ARGS.values()), ids=list(ARGS))
@pytest.mark.parametrize("form", [f for f in FORMS if not f.nojit], ids=lambda f: f.name)
def test_form_matrix(ctx, switches, form, arg):
    """Every function, with and without a mask, over every NULL mode of the argument, on every page shape; exact against the reference.
    Catches: a narrow load that does not sign-extend (INT8_MIN, INT16_MIN, INT32_MIN in every page); tail rows of the four-row loader
    dropped or read twice (n = 1, 2, 3 mod 4); a mask ignored by min / max; a non-NULL counter read back from the wrong row counter
    after the kernel dropped it; the special groups (NULL, INT64_MIN) lost or merged with a regular one; a single dropped or doubled
    row in a DOUBLE sum."""
    switches(form.env)
    for scenario in scenarios_of(form):
        run_form(ctx, form, arg, scenario)


def _child(env_extra, body):
    """runs `body` (Python source, with this module imported as t) in a fresh interpreter; -> the JSON object it prints last"""
    tests_dir = os.path.dirname(os.path.abspath(__file__))
    env = {k: v for k, v in os.environ.items() if k not in SWITCHES}
    env.update(env_extra)
    env["PYTHONPATH"] = os.pathsep.join([os.path.dirname(tests_dir), tests_dir] + ([env["PYTHONPATH"]] if env.get("PYTHONPATH") else []))
    args = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", "import test_gpu_groupby_forms as t; " + body]
    r = subprocess.run(args, env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stderr[-4000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def child_matrix_main(names):
    """Body of a child process: the matrix of the named forms; prints {form: first failure or None}"""
    ctx = ops.Context(0)
    result = {}
    try:
        for name in names:
            form = FORM_BY_NAME[name]
            apply_switches(form.env)
            try:
                for arg in ARGS.values():
                    for scenario in scenarios_of(form):
                        run_form(ctx, form, arg, scenario)
                result[name] = None
            except Exception as e:          # reported to the parent, which fails
                result[name] = "%s: %s" % (type(e).__name__, str(e)[:2000])
    finally:
        ctx.close()
    print(json.dumps(result))


def test_interpreted_small_path():
    """Without NVRTC (TGPU_DISABLE_JIT=1: jit_available() is decided once per process, hence a child process) path S runs the
    interpreted agg_small_kernel, which keeps every non-NULL counter; the same matrix as test_form_matrix."""
    names = [f.name for f in FORMS if f.nojit]
    result = _child({"TGPU_DISABLE_JIT": "1"}, "t.child_matrix_main(%r)" % names)
    assert result == {n: None for n in names}, result


# ---- keys ------------------------------------------------------------------------------------------------------------------------
_NANS = (0x7FF8000000000000, 0x7FF8000000000123, 0xFFF8000000000000, 0x7FF0000000000001, 0xFFFFFFFFFFFFFFFF)


def key_pool(kind, many):
    """distinct-under-IDENTICAL key tuples (NULL fields included) of one key kind, as (types, list of tuples)"""
    rng = np.random.default_rng(_seed("keys", kind, many))
    count = 300 if many else 12
    if kind in ("integer", "smallint", "tinyint"):
        t = ARGS[kind]
        info = np.iinfo({abi.INT32: np.int32, abi.INT16: np.int16, abi.INT8: np.int8}[t])
        vals = [info.min, info.max, -1, 0, None, info.min + 1, -2] + rng.integers(info.min, info.max, 4 * count).tolist()
        return (t,), [(v,) for v in list(dict.fromkeys(vals))[:count]]
    if kind == "bigint":
        return (abi.INT64,), [(v,) for v in [INT64_MIN, None] + regular_keys(count - 2)]
    if kind == "packed":
        out = [(None, None, None), (-(1 << 31), -1, -128), (-1, -(1 << 15), 127), ((1 << 31) - 1, None, -1), (None, 5, None), (0, 0, 0)]
        while len(out) < count:
            t = tuple(None if rng.random() < 0.1 else int(x) for x in (rng.integers(-50, 50), rng.integers(-(1 << 15), 1 << 15), rng.integers(-128, 128)))
            if t not in out:
                out.append(t)
        return (abi.INT32, abi.INT16, abi.INT8), out
    if kind == "hashed":
        out = [(None, None), (INT64_MIN, -1), (-1, None), (None, -(1 << 31))]
        while len(out) < count:
            out.append((int(rng.integers(INT64_MIN, INT64_MAX)), int(rng.integers(-(1 << 31), 1 << 31))))
        return (abi.INT64, abi.INT32), out
    if kind == "double":
        vals = [None, 0.0, math.inf, -math.inf, _double(_NANS[0]), 5e-324, -2.5, 1e300]
        vals += [float(x) / 8 for x in rng.integers(-4000, 4000, count)]
        uniq, seen = [], set()
        for v in vals:
            ident = None if v is None else "NaN" if v != v else v
            if ident not in seen:
                seen.add(ident)
                uniq.append((v,))
        return (abi.FLOAT64,), uniq[:count]
    assert kind == "varchar"
    words = [None, "", "A", "N", "1234567", "12345678", "a much longer key than seven bytes", "naïve café"]
    words += ["k%d" % i for i in range(count)]
    return (abi.UTF8,), [(w,) for w in words[:count]]


def _variant(kind, value, rng):
    """another raw spelling of the same IDENTICAL key: the zero of the other sign, a NaN of another payload"""
    if kind != "double" or value is None:
        return value
    if value == 0:
        return -0.0 if rng.random() < 0.5 else 0.0
    if value != value:
        return _double(_NANS[rng.integers(0, len(_NANS))])
    return value


def key_blocks(types, rows):
    blocks = []
    for c, t in enumerate(types):
        vals = [r[c] for r in rows]
        blocks.append(Block.varchar(vals) if t == abi.UTF8 else MAKE[t](vals))
    return blocks


@functools.lru_cache(maxsize=32)
def key_case(kind, many):
    rng = np.random.default_rng(_seed("key_case", kind, many))
    types, pool = key_pool(kind, many)
    nk = len(types)
    pages = []
    for i, n in enumerate(SIZES):
        rows = [pool[j] for j in rng.integers(0, len(pool), n)]
        if i == 1:
            rows[:len(pool)] = pool[:n]
        rows = [tuple(_variant(kind, x, rng) for x in r) for r in rows]
        v = value_block(abi.INT32, n, ("some", "none", "present", "all")[i % 4], rng)
        pages.append(Page(*key_blocks(types, rows), v, Block.boolean(rng.random(n) < 0.5, rng.random(n) < 0.1), position_count=n))
    aggs = [(abi.AGG_COUNT_STAR, -1, -1), (abi.AGG_SUM, nk, -1), (abi.AGG_MAX, nk, -1)]     # (5 words: 16 key slots fit)
    return pages, list(range(nk)), aggs, aggregate(pages, list(range(nk)), aggs)


KEY_KINDS = ("bigint", "integer", "smallint", "tinyint", "packed", "double", "hashed", "varchar")


@pytest.mark.parametrize("kind", KEY_KINDS)
@pytest.mark.parametrize("form", ["S_L16", "S_spill", "general_jit", "general_interpreted", "multipass", "sliced_copy_any_order"])
def test_every_key_kind(ctx, switches, form, kind):
    """The group-id order and the output keys, bit for bit, for every key kind: BIGINT with INT64_MIN (the empty-slot sentinel) and
    NULL; INTEGER / SMALLINT / TINYINT alone (their extremes, negative values: the key columns must come back sign-extended) and packed
    into one word; DOUBLE keys whose first-seen spelling (-0.0 or +0.0, one of several NaN payloads) is the output; a composite key
    wider than 63 bits (hashed: always the multipass form); VARCHAR (dictionary ids).  A NULL field is part of the tuple."""
    f = FORM_BY_NAME[form]
    switches(f.env)
    many = f.expected > 256
    pages, keys, aggs, want = key_case(kind, many)
    if form == "S_spill":
        pages = key_case(kind, False)[0][:3] + key_case(kind, True)[0][3:]
        want = aggregate(pages, keys, aggs)
    got = run_operator(ctx, pages, keys, aggs, f.expected)
    check_rows(got, want, len(keys), "%s %s" % (form, kind))


# ---- DOUBLE specials, rounding, BIGINT range -------------------------------------------------------------------------------------
_SPECIAL_GROUPS = [
    [1.0, _double(0x7FF8000000000001), _double(0xFFF8000000000000)],          # NaN payloads and a negative NaN beside a number
    [_double(0x7FF0000000000001), _double(0xFFFFFFFFFFFFFFFF)],               # only NaNs
    [math.inf, -math.inf, 2.0],
    [math.inf, _double(0xFFF8000000000000)],                                   # max: NaN ranks below +Inf; min: above it
    [-math.inf, _double(0x7FF8000000000000)],
    [-0.0],                                                                    # sum = +0.0
    [0.0, -0.0],
    [-0.0, 0.0, -0.0],
    [5e-324, -5e-324, _double(0x000FFFFFFFFFFFFF)],                            # denormals (exact sums)
    [-math.inf],
    [math.inf, 1e308, 1e308],
]


@pytest.mark.parametrize("form", ["S_L16", "general_jit", "multipass"])
def test_double_specials(ctx, switches, form):
    """NaN (several payloads, negative NaN), +-Inf, -0.0 / +0.0 and denormals through sum, min and max.  Non-NaN results compare by
    their bits; a NaN result only has to be NaN."""
    f = FORM_BY_NAME[form]
    switches(f.env)
    rng = np.random.default_rng(3)
    keys, vals = [], []
    for g, xs in enumerate(_SPECIAL_GROUPS):
        keys += [g] * len(xs)
        vals += xs
    pages = []
    for n_rep in (1, 3):                                      # the 25 rows in order, then 75 rows (n = 3 mod 4) shuffled
        idx = np.arange(len(keys)) if n_rep == 1 else rng.permutation(np.repeat(np.arange(len(keys)), n_rep))
        kv = np.array(keys, dtype=np.int64)[idx]
        vv = np.array([_bits(x) for x in vals], dtype=np.int64)[idx].view(np.float64)
        pages.append(Page(Block.bigint(kv), Block.double(vv)))
    aggs = [(abi.AGG_SUM, 1, -1), (abi.AGG_MIN, 1, -1), (abi.AGG_MAX, 1, -1), (abi.AGG_COUNT, 1, -1)]
    got = run_operator(ctx, pages, [0], aggs, f.expected)
    check_rows(got, aggregate(pages, [0], aggs), 1, form)


@pytest.mark.parametrize("form", ["S_L16", "general_jit", "multipass"])
def test_double_sum_rounding(ctx, switches, form):
    """Sums that are not exact in any order (1e16, 1.0 and -1e16 mixed, and random magnitudes): whatever order the device adds in, the
    result lies within (n - 1) * 2^-53 * sum(|x|) of the exact sum (recursive summation's error bound)."""
    f = FORM_BY_NAME[form]
    switches(f.env)
    rng = np.random.default_rng(5)
    groups = 6
    pages = []
    for n in (1000, 3, 4001):
        k = rng.integers(0, groups, n)
        base = rng.choice(np.array([1e16, -1e16, 1.0, -1.0, 3.0, 0.1]), n)
        v = np.where(k % 2 == 0, base, rng.normal(0, 1, n) * 10.0 ** rng.integers(-8, 17, n))
        pages.append(Page(Block.bigint(k), Block.double(v)))
    got = run_operator(ctx, pages, [0], [(abi.AGG_SUM, 1, -1), (abi.AGG_COUNT, 1, -1)], f.expected)
    vals = {}
    for p in pages:
        for key, x in zip(p.get_block(0).values.tolist(), p.get_block(1).values.tolist()):
            vals.setdefault(key, []).append(x)
    assert [r[0] for r in got] == list(vals)
    for key, total, count in got:
        xs = vals[key]
        exact = sum(Fraction(x) for x in xs)
        bound = (len(xs) - 1) * Fraction(1, 1 << 53) * sum(Fraction(abs(x)) for x in xs)
        assert count == len(xs) and abs(Fraction(total) - exact) <= bound, (form, key, total, float(exact), float(bound))


@pytest.mark.parametrize("form", ["S_L16", "general_jit", "general_interpreted", "multipass"])
def test_bigint_sum_range(ctx, switches, form):
    """BIGINT extremes: totals of INT64_MAX and INT64_MIN exactly (every partial sum of any order in range) come back; a total one past
    either end raises NUMERIC_VALUE_OUT_OF_RANGE (the device checks the final 128-bit total, see agg_reference)."""
    f = FORM_BY_NAME[form]
    switches(f.env)
    inside = {0: [1 << 62, (1 << 62) - 1], 1: [-(1 << 62), -(1 << 62)], 2: [INT64_MIN], 3: [INT64_MAX], 4: [INT64_MIN + 1, -1], 5: [INT64_MAX, 0, 0]}
    aggs = [(abi.AGG_SUM, 1, -1), (abi.AGG_MIN, 1, -1), (abi.AGG_MAX, 1, -1), (abi.AGG_COUNT_STAR, -1, -1)]

    def pages_of(groups):
        keys = [k for k, xs in groups.items() for _ in xs]
        vals = [x for xs in groups.values() for x in xs]
        return [Page(Block.bigint(keys), Block.bigint(vals)), Page(Block.bigint([0]), Block.bigint([0]))]

    pages = pages_of(inside)
    want = aggregate(pages, [0], aggs)
    assert [r[1] for r in want] == [INT64_MAX, INT64_MIN, INT64_MIN, INT64_MAX, INT64_MIN, INT64_MAX]
    check_rows(run_operator(ctx, pages, [0], aggs, f.expected), want, 1, form)
    for outside in ({0: [1 << 62, 1 << 62]}, {7: [1, 2], 1: [-(1 << 62), -(1 << 62), -1]}, {0: [INT64_MAX, 1]}):
        pages = pages_of(outside)
        with pytest.raises(AggregateOverflow):
            aggregate(pages, [0], aggs)
        with pytest.raises(abi.TrinoGpuError) as e:
            run_operator(ctx, pages, [0], aggs, f.expected)
        assert e.value.code == abi.ERR_NUMERIC_VALUE_OUT_OF_RANGE, (form, outside)


# ---- routing: the table above is what the pages launch -----------------------------------------------------------------------------
ROUTE_ARG, ROUTE_SCENARIO = abi.INT16, "mixed"


def routing_main(names):
    """Body of the routing test's child processes: one case of every named form (checked against the reference) observed by
    kernels_launched; prints {form: kernel names, or None} as one JSON line."""
    ctx = ops.Context(0)
    launched = {}
    try:
        for name in names:
            form = FORM_BY_NAME[name]
            apply_switches(form.env)
            scenario = ROUTE_SCENARIO if ROUTE_SCENARIO in scenarios_of(form) else scenarios_of(form)[0]
            launched[name] = kernels_launched(lambda: run_form(ctx, form, ROUTE_ARG, scenario))
    finally:
        ctx.close()
    print(json.dumps(launched))


def test_every_form_launches_its_kernels():
    """For each form of FORMS, one case under the profiler: its kernels are launched and the ones it must not use are not.  The cases run
    in child processes (one with TGPU_DISABLE_JIT=1 for the interpreted forms): after profiler sessions of earlier tests in the same
    process, the profiler has been seen to record the library's copies but none of its kernels.  A form without a complete profiler
    session fails the test; the test skips only when no session delivers its markers."""
    launched = {}
    for nojit in (False, True):
        names = [f.name for f in FORMS if f.nojit == nojit]
        launched.update(_child({"TGPU_DISABLE_JIT": "1"} if nojit else {}, "t.routing_main(%r)" % names))
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
