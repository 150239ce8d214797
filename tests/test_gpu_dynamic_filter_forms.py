"""DynamicPageFilter (csrc/dynfilter.cu) form by form against the exact reference of oracle/dynamic_filter.py.

One kernel evaluates up to 16 column domains per row in their order, short-circuits, and counts per filter the rows that reached and
passed it (the EffectiveFilterProfiler's two counters); the selected rows are then compacted, or every block passes through when all
rows are selected.  Every case runs its pages through the operator and through DynamicFilterEvaluator side by side and compares, page
by page, the selected rows (values bit for bit, NULLs, order), whether the output passes the input blocks through, and is_effective(i)
of every filter.

  column types   BIGINT, INTEGER, DATE, SMALLINT, TINYINT, BOOLEAN and short DECIMAL under ALL / NONE / RANGE / DISCRETE; DOUBLE under
                 ALL / NONE / RANGE (by value); REAL, VARCHAR and long DECIMAL under ALL / NONE.  RANGE / DISCRETE over REAL, VARCHAR and
                 long DECIMAL and DISCRETE over DOUBLE are refused (NOT_SUPPORTED): the domain bounds are 64-bit integers.
  value edges    lo == hi, INT64_MIN / INT64_MAX and the type's own bounds, empty ranges; one value, unsorted and duplicate values, values
                 outside the type whose low bits equal a column value, negative values on narrow types, a 4002-value list (12 binary-
                 search steps); DOUBLE +-0.0, +-inf, NaN and the bounds themselves
  NULL forms     no validity buffer, a byte map, an Arrow bitmap whose tail bits are garbage, all NULL
  block forms    flat, DictionaryBlock, RunLengthEncodedBlock (also of NULL), a device page made by an upstream operator
  shapes         pages of 0 .. 8192 rows, 2^20 rows and 2.2 M rows (more than one wave of the grid-stride kernel on an H100 with 132 SMs);
                 1, 2 and 16 domains, several on one channel, none on channel 0
  profiler       the 2047-position boundary, output exactly threshold x input (the test is strict >), thresholds 0, 0.5 and 1, filters
                 starved by an earlier one, update() in the middle of a stream
"""
import ctypes as C
import zlib

import numpy as np
import pytest

from helpers import oracle_join_rows
from test_oracle_dynamic_filter import df, double_range_cases
from trino_b200 import abi
from trino_b200 import operators as ops
from trino_b200.page import AbiPage, Block, DictionaryBlock, Page, RunLengthEncodedBlock

pytestmark = pytest.mark.gpu
INT64_MIN, INT64_MAX = -2**63, 2**63 - 1
SIZES = (1, 31, 32, 33, 0, 255, 257, 8192)
NULL_FORMS = ("none", "bytemap", "bitmap", "all")
BLOCK_FORMS = ("flat", "dictionary", "rle", "device")

# integer family: (block constructor, the type's value range, bits of the physical value)
INT_TYPES = {
    "bigint": (Block.bigint, INT64_MIN, INT64_MAX, 64),
    "integer": (Block.integer, -2**31, 2**31 - 1, 32),
    "date": (Block.date, -719_162, 2_932_896, 32),          # 0001-01-01 .. 9999-12-31 in days since 1970-01-01
    "smallint": (Block.smallint, -2**15, 2**15 - 1, 16),
    "tinyint": (Block.tinyint, -128, 127, 8),
    "boolean": (Block.boolean, 0, 1, 8),
    "decimal(18,2)": (Block.bigint, -10**18 + 1, 10**18 - 1, 64),
}
OTHER_TYPES = ("double", "real", "varchar", "decimal(38,2)")
DOUBLE_SPECIALS = (0.0, -0.0, np.inf, -np.inf, np.nan, -np.nan, 1.5, -1.5, 2.25, -2.25, 1.0, -1.0, 5e-324, -5e-324)


# ---- pages ------------------------------------------------------------------------------------------------------------------------------
def _values(tname, rng, n):
    """values of a column of type tname: numpy array, or a list for VARCHAR and long DECIMAL"""
    if tname in INT_TYPES:
        _, lo, hi, _ = INT_TYPES[tname]
        v = np.where(rng.random(n) < 0.75, rng.integers(max(lo, -70), min(hi, 70), n, endpoint=True), rng.integers(lo, hi, n, endpoint=True))
        edge = rng.random(n)
        return np.where(edge < 0.02, lo, np.where(edge > 0.98, hi, v)).astype(np.int64)
    if tname == "double":
        return np.where(rng.random(n) < 0.5, rng.choice(np.array(DOUBLE_SPECIALS), n), rng.normal(0, 3, n))
    if tname == "real":
        return np.where(rng.random(n) < 0.3, np.float32(np.nan), rng.normal(0, 3, n)).astype(np.float32)
    if tname == "varchar":
        return [b"" if k == 0 else ("k%dé" % k).encode() for k in rng.integers(0, 40, n)]
    return [int(k) * 10**30 - 7 for k in rng.integers(-3, 4, n)]          # decimal(38,2)


def _block(tname, values, nulls):
    if tname == "varchar":
        return Block.varchar([None if nulls is not None and nulls[i] else v for i, v in enumerate(values)])
    if tname == "decimal(38,2)":
        return Block.int128(values, nulls)
    if tname in INT_TYPES:
        return INT_TYPES[tname][0](values, nulls)
    return Block.double(values, nulls) if tname == "double" else Block.real(values, nulls)


def _nulls(rng, n, null_form):
    if null_form == "none":
        return None
    if null_form == "all":
        return np.ones(n, dtype=bool)
    return rng.random(n) < 0.2


def _column(tname, rng, n, form, null_form):
    """the filtered column in one block form (the device form is made from a flat page by _feed)"""
    if form in ("flat", "device"):
        return _block(tname, _values(tname, rng, n), _nulls(rng, n, null_form))
    if form == "dictionary":
        m = n // 4 + 1
        return DictionaryBlock(_block(tname, _values(tname, rng, m), _nulls(rng, m, null_form)), rng.integers(0, m, n))
    value_is_null = null_form in ("all", "bitmap")                       # RLE of NULL in two of the four forms
    return RunLengthEncodedBlock(_block(tname, _values(tname, rng, 1), np.array([value_is_null]) if value_is_null else None), n)


def _garbage_tail_bits(col):
    """set the bits past the last position of an Arrow validity bitmap (they mean nothing; a kernel must not read them)"""
    n = col.length
    if col.validity and not (col.flags & abi.COL_NULLS_BYTEMAP) and n % 8:
        bits = np.ctypeslib.as_array((C.c_uint8 * ((n + 7) // 8)).from_address(col.validity))
        bits[-1] |= (0xFF << (n % 8)) & 0xFF
    if col.dictionary:
        _garbage_tail_bits(col.dictionary.contents)


def _abi_page(page, null_form):
    ap = AbiPage(page, nulls_as_bytemap=null_form != "bitmap")
    if null_form == "bitmap":
        for c in range(ap.ncols):
            _garbage_tail_bits(ap.columns[c])
    return ap


class Input:
    """One input page: `host` is what the page holds (the expected output's source), `feed` what add_input receives."""

    def __init__(self, host, feed, upstream=None):
        self.host, self.feed, self.upstream = host, feed, upstream

    def release(self):
        if self.upstream is not None:
            out, op = self.upstream
            out.release()
            op.close()


def _feed(ctx, page, null_form, device=False):
    """the page as a host tgpu_page in the given NULL form, or as the device page an upstream GPU operator (a pass-everything dynamic
    filter) hands on"""
    ap = _abi_page(page, null_form)
    if not device or page.position_count == 0:
        return Input(page, ap)
    up = ops.DynamicFilterOperatorFactory(ctx, []).create_operator()
    up.add_input(ap)
    out = up.get_output_device()
    return Input(page, out.as_device_page(), (out, up))


def _oracle_columns(page):
    """(int64 values or raw DOUBLE bits, nulls) per channel; REAL / VARCHAR / long DECIMAL values are never compared (ALL / NONE only)"""
    cols = []
    for b in page.blocks:
        f = b.flatten()
        if f.type == abi.FLOAT64:
            v = f.values.view(np.int64)
        elif f.type in (abi.INT64, abi.INT32, abi.INT16, abi.INT8):
            v = f.values.astype(np.int64)
        else:
            v = np.zeros(f.position_count, dtype=np.int64)
        cols.append((v, f.nulls))
    return cols


# ---- running both sides -----------------------------------------------------------------------------------------------------------------
def _gpu(d):
    return ops.ColumnDomain(d.channel, d.kind, d.null_allowed, d.lo, d.hi, None if d.values is None else d.values.tolist())


def _null_flags(b):
    return np.zeros(b.position_count, dtype=bool) if b.nulls is None else b.nulls


def _bits(values):
    return values.view(np.int64) if values.dtype == np.float64 else values.view(np.int32) if values.dtype == np.float32 else values


def _passthrough(ctx, out, c):
    src = C.c_int32(-2)
    ctx.check(ctx.lib.tgpu_page_passthrough_channel(out.pp, c, C.byref(src)))
    return src.value


def _assert_selected(got, host, sel, what):
    assert got.position_count == len(sel), what
    for c, blk in enumerate(host.blocks):
        want, g = blk.flatten(), got.get_block(c)
        assert g.type == want.type, what
        wn, gn = _null_flags(want)[sel], _null_flags(g)
        assert np.array_equal(wn, gn), f"{what}: NULLs of channel {c}"
        if want.type == abi.UTF8:
            assert g.to_pylist() == [want.get(int(i)) for i in sel], f"{what}: channel {c}"
        else:
            assert np.array_equal(_bits(want.values)[sel][~wn], _bits(g.values)[~gn]), f"{what}: values of channel {c}"


def _step(ctx, op, ev, item, what=""):
    """one page through the operator and the oracle: selected rows, pass-through, profiler state"""
    try:
        sel = ev.evaluate(_oracle_columns(item.host))
        op.add_input(item.feed)
        out = op.get_output_device()
        n = item.host.position_count
        if len(sel) == 0:
            assert out is None, f"{what}: no row selected, but an output page"
        else:
            assert out is not None, f"{what}: {len(sel)} rows selected, but no output page"
            try:
                src = [_passthrough(ctx, out, c) for c in range(out.num_columns)]
                assert src == (list(range(out.num_columns)) if len(sel) == n else [-1] * out.num_columns), f"{what}: pass-through {src}"
                got = out.to_host()
            finally:
                out.release()
            _assert_selected(got, item.host, sel, what)
    finally:
        item.release()
    assert [op.is_effective(i) for i in range(len(ev.domains))] == [not x for x in ev.ineffective], what
    return sel


def _run(ctx, domains, items, threshold=1.0, what=""):
    op = ops.DynamicFilterOperatorFactory(ctx, [_gpu(d) for d in domains], threshold).create_operator()
    ev = df.DynamicFilterEvaluator(domains, threshold)
    try:
        for k, item in enumerate(items):
            _step(ctx, op, ev, item, f"{what} page {k}")
    finally:
        op.close()


# ---- domains ----------------------------------------------------------------------------------------------------------------------------
def _int_domains(tname, ch, rng):
    _, lo, hi, bits = INT_TYPES[tname]
    R = lambda a, b: (df.RANGE, dict(lo=a, hi=b))
    D = lambda vals: (df.DISCRETE, dict(values=[int(x) for x in vals]))
    kinds = [(df.ALL, {}), (df.NONE, {}), R(-20, 45), R(7, 7), R(0, 0), R(INT64_MIN, 3), R(-3, INT64_MAX), R(INT64_MIN, INT64_MAX),
             R(10, -10), R(lo, hi), R(lo, lo), R(hi, hi), R(lo + 1, hi - 1),
             D([5]), D([40, -7, 3, 40, 0, -60, 3, 1]), D([lo, hi]), D([-1, -2, -60, lo]),
             D(list(rng.integers(-70, 71, 4000)) + [lo, hi])]                 # 4002 values with duplicates: 12 binary-search steps
    if bits < 64:
        # outside the type's range, with the low bits of values the column holds (300 on TINYINT is 44 in one byte): never equal
        kinds.append(D([v + (1 << bits) for v in (-1, -2, -60, lo, 44)] + [v - (1 << bits) for v in (1, 44, hi)] + [hi + 1, lo - 1, 300]))
    return [df.Domain(ch, k, na, **kw) for k, kw in kinds for na in (False, True)]


def _double_range(ch, lo, hi, null_allowed):
    d = ops.ColumnDomain.double_range(ch, lo, hi, null_allowed)
    return df.Domain(ch, df.RANGE, null_allowed, d.lo, d.hi, double=True)


def _domains(tname, ch, rng):
    if tname in INT_TYPES:
        return _int_domains(tname, ch, rng)
    doms = [df.Domain(ch, k, na) for k in (df.ALL, df.NONE) for na in (False, True)]
    if tname == "double":
        inf = np.inf
        for lo, hi in ((-1.5, 2.25), (0.0, 0.0), (-0.0, -0.0), (-inf, -0.0), (-inf, inf), (1.0, -1.0), (2.25, 2.25), (inf, inf), (-2.25, -1.0),
                       (5e-324, 1.0)):
            doms += [_double_range(ch, lo, hi, na) for na in (False, True)]
    return doms


# ---- column types x domain kinds x NULL forms x block forms -----------------------------------------------------------------------------
@pytest.mark.parametrize("form", BLOCK_FORMS)
@pytest.mark.parametrize("tname", list(INT_TYPES) + list(OTHER_TYPES))
def test_column_types_domains_and_block_forms(ctx, tname, form):
    """Each domain of the type, with and without NULLs allowed, filters channel 1 of a page sequence of every size in SIZES; the NULL
    form changes from page to page.  Channel 0 (row numbers) and 2 (VARCHAR with NULLs) come along: they are gathered or passed through."""
    rng = np.random.default_rng(zlib.crc32(f"{tname} {form}".encode()))
    items = []
    for k, n in enumerate(SIZES):
        null_form = NULL_FORMS[k % len(NULL_FORMS)]
        tags = Block.varchar([None if x % 7 == 0 else b"t%d" % x for x in range(n)]) if null_form != "none" else Block.varchar([b"t%d" % x for x in range(n)])
        page = Page(Block.bigint(np.arange(n)), _column(tname, rng, n, form, null_form), tags, position_count=n)
        items.append((page, null_form))
    for d in _domains(tname, 1, rng):
        what = f"{tname} {form} kind {d.kind} null_allowed {d.null_allowed} lo {d.lo} hi {d.hi}"
        _run(ctx, [d], [_feed(ctx, page, null_form, form == "device") for page, null_form in items], what=what)


def test_double_range_oracle_cases(ctx):
    """the oracle's pinned DOUBLE-range cases (-0.0 == 0.0, NaN in no range, negative bounds by value) on the device"""
    for name, domains, threshold, pages, expected in double_range_cases():
        items = []
        for columns in pages:
            vals, nulls = columns[0]
            items.append(_feed(ctx, Page(Block.double(vals.view(np.float64), nulls)), "bytemap"))
        _run(ctx, domains, items, threshold, name)


@pytest.mark.parametrize("tname,kind_name", [("real", "range"), ("real", "discrete"), ("varchar", "range"), ("varchar", "discrete"),
                                             ("decimal(38,2)", "range"), ("decimal(38,2)", "discrete"), ("double", "discrete")])
def test_value_sets_the_device_cannot_compare_are_refused(ctx, tname, kind_name):
    """RANGE / DISCRETE bounds are 64-bit integers (raw bits for DOUBLE): over REAL, VARCHAR and long DECIMAL channels and as a DOUBLE value
    list they cannot be compared, and the operator must refuse them rather than filter by some other bytes.  The long DECIMAL page holds
    10^30 everywhere: RANGE [0, 100] and DISCRETE {0 .. 100} select nothing."""
    kind = df.RANGE if kind_name == "range" else df.DISCRETE
    n = 64
    column = Block.int128([10**30] * n) if tname == "decimal(38,2)" else _block(tname, _values(tname, np.random.default_rng(5), n), None)
    page = Page(Block.bigint(np.arange(n)), column)
    d = ops.ColumnDomain(1, kind, False, 0, 100, list(range(101)) if kind == df.DISCRETE else None)
    op = ops.DynamicFilterOperatorFactory(ctx, [d]).create_operator()
    try:
        with pytest.raises(abi.TrinoGpuError) as err:
            op.add_input(page)
            out = op.get_output()
            pytest.fail(f"{kind_name} over {tname} was evaluated on the device and selected {0 if out is None else out.position_count} of {n} rows")
        assert err.value.code == abi.ERR_NOT_SUPPORTED
    finally:
        op.close()


# ---- shapes -----------------------------------------------------------------------------------------------------------------------------
def _wide_page(rng, n):
    cols = [Block.bigint(rng.integers(-1000, 1000, n), rng.random(n) < 0.03), Block.integer(rng.integers(-500, 500, n).astype(np.int32)),
            Block.smallint(rng.integers(-300, 300, n).astype(np.int16), rng.random(n) < 0.01), Block.tinyint(rng.integers(-128, 128, n).astype(np.int8)),
            Block.double(rng.normal(0, 10, n), rng.random(n) < 0.02)]
    return Page(*cols, position_count=n)


def _shape_domains(count, rng):
    """permissive domains (each drops a few percent) so that 16 of them in a row still leave rows; several per channel, none on channel 0
    for the 2-domain set"""
    pool = [df.Domain(2, df.RANGE, True, lo=-290, hi=295), df.Domain(1, df.DISCRETE, False, values=[v for v in range(-500, 500) if v % 37]),
            df.Domain(4, df.RANGE, False, *np.array([-25.0, 26.0]).view(np.int64).tolist(), double=True), df.Domain(3, df.RANGE, False, lo=-120, hi=127),
            df.Domain(0, df.RANGE, False, lo=-990, hi=INT64_MAX), df.Domain(1, df.RANGE, False, lo=-480, hi=499), df.Domain(3, df.DISCRETE, False, values=list(range(-128, 126))),
            df.Domain(0, df.DISCRETE, True, values=[v for v in range(-1000, 1000) if v % 53]), df.Domain(2, df.DISCRETE, True, values=list(range(-299, 300))),
            df.Domain(1, df.ALL, True), df.Domain(4, df.RANGE, True, *np.array([-np.inf, 24.0]).view(np.int64).tolist(), double=True),
            df.Domain(0, df.RANGE, True, lo=-1000, hi=980), df.Domain(3, df.RANGE, False, lo=-127, hi=127), df.Domain(2, df.RANGE, True, lo=INT64_MIN, hi=290),
            df.Domain(1, df.DISCRETE, False, values=rng.permutation(np.arange(-495, 500)).tolist()), df.Domain(0, df.ALL, True)]
    return pool[:count]


@pytest.mark.parametrize("count", [1, 2, 16])
def test_page_sizes_and_domain_counts(ctx, count):
    """1, 2 and 16 (DF_MAX) domains over pages from 1 row to 2.2 M rows: past one full wave of the kernel (132 SMs x 8 CTAs x 1024 rows)
    every thread strides over several rows and the per-warp counter sums carry real counts.  The threshold (0.97) sits between the pass
    rates of the filters, so the profiler's decisions depend on exact counts."""
    rng = np.random.default_rng(count)
    domains = _shape_domains(count, rng)
    items = [_feed(ctx, _wide_page(rng, n), "bytemap") for n in SIZES + (1 << 20, 2_200_000, 3000)]
    _run(ctx, domains, items, 0.97, f"{count} domains")


def test_domain_count_limit(ctx):
    """16 domains (DF_MAX) on one channel are evaluated; a 17th is refused at create and at update"""
    doms16 = [df.Domain(0, df.RANGE, False, lo=i, hi=100 - i) for i in range(16)]
    _run(ctx, doms16, [_feed(ctx, Page(Block.bigint(np.arange(-5, 120))), "none")], what="16 domains on channel 0")
    doms17 = [_gpu(df.Domain(0, df.RANGE, False, lo=i, hi=100)) for i in range(17)]
    with pytest.raises(abi.TrinoGpuError) as err:
        ops.DynamicFilterOperatorFactory(ctx, doms17).create_operator()
    assert err.value.code == abi.ERR_NOT_SUPPORTED
    op = ops.DynamicFilterOperatorFactory(ctx, doms17[:1]).create_operator()
    with pytest.raises(abi.TrinoGpuError) as err:
        op.update(doms17)
    assert err.value.code == abi.ERR_NOT_SUPPORTED
    op.close()


# ---- output form ------------------------------------------------------------------------------------------------------------------------
def test_output_forms_and_protocol(ctx):
    """no row selected: no page; every row selected: the blocks pass through (tgpu_page_passthrough_channel(c) == c); otherwise gathered
    (-1).  Zero-row pages produce nothing and move no counter.  addInput while an output page is pending is an ILLEGAL_STATE."""
    d = [df.Domain(0, df.RANGE, False, lo=10, hi=19)]
    pages = [Page(Block.bigint(np.arange(10, 20)), Block.varchar(["a", None, "c", "", "e", "f", "g", "h", "i", "j"]), Block.double(np.linspace(-1, 1, 10))),
             Page(Block.bigint(np.arange(0, 10)), Block.varchar(["x"] * 10), Block.double(np.zeros(10))),
             Page(Block.bigint([], None), Block.varchar([]), Block.double([]), position_count=0),
             Page(Block.bigint(np.arange(5, 25)), Block.varchar(["y%d" % i for i in range(20)]), Block.double(np.ones(20)))]
    for null_form in ("none", "bytemap", "bitmap"):
        for device in (False, True):
            _run(ctx, d, [_feed(ctx, p, null_form, device) for p in pages], what=f"{null_form} device={device}")
    op = ops.DynamicFilterOperatorFactory(ctx, [_gpu(d[0])]).create_operator()
    op.add_input(pages[0])
    assert not op.needs_input()
    with pytest.raises(abi.TrinoGpuError) as err:
        op.add_input(pages[3])
    assert err.value.code == abi.ERR_ILLEGAL_STATE
    assert op.get_output().rows() == pages[0].rows()
    assert op.needs_input()
    op.close()


# ---- EffectiveFilterProfiler ------------------------------------------------------------------------------------------------------------
def _seq_page(values, n_channels=2):
    v = np.asarray(values, dtype=np.int64)
    return Page(*[Block.bigint(v) for _ in range(n_channels)], position_count=len(v))


def _profile(ctx, domains, threshold, pages):
    """run the pages; -> is_effective of every filter after every page (compared with the oracle on the way)"""
    op = ops.DynamicFilterOperatorFactory(ctx, [_gpu(d) for d in domains], threshold).create_operator()
    ev = df.DynamicFilterEvaluator(domains, threshold)
    states = []
    try:
        for k, p in enumerate(pages):
            _step(ctx, op, ev, _feed(ctx, p, "none"), f"threshold {threshold} page {k}")
            states.append([op.is_effective(i) for i in range(len(domains))])
    finally:
        op.close()
    return states


@pytest.mark.parametrize("threshold", [0.0, 0.5, 1.0])
def test_profiler_boundaries(ctx, threshold):
    """A filter is judged once it has seen 2047 positions, and switched off only when it passes MORE than threshold x input"""
    alternating = lambda n, first: [(first + i) % 2 for i in range(n)]
    # 2046 positions, every one passing: not judged yet; the 2047th: judged (off unless threshold 1.0, where 2047 > 2047 is false)
    states = _profile(ctx, [df.Domain(1, df.ALL, True)], threshold, [_seq_page(np.zeros(1023)), _seq_page(np.zeros(1023)), _seq_page([0])])
    assert states == [[True], [True], [threshold == 1.0]]
    # exactly half of 2048 positions pass: at 0.5, 1024 > 0.5 x 2048 is false and the filter stays on; one more passing row turns it off
    half = [df.Domain(0, df.RANGE, False, lo=0, hi=0)]
    states = _profile(ctx, half, threshold, [_seq_page(alternating(1024, 0)), _seq_page(alternating(1024, 1)), _seq_page([0])])
    assert states == [[True], [threshold != 0.0], [threshold == 1.0]]
    # a filter that passes nothing is never switched off, not even at threshold 0 (0 > 0 is false)
    states = _profile(ctx, [df.Domain(0, df.NONE, False)], threshold, [_seq_page(np.arange(3000))] * 2)
    assert states == [[True], [True]]


def test_starved_filter_keeps_its_counters(ctx):
    """Rows an earlier filter drops never reach the later ones: on a page where filter 0 selects nothing, filter 1's counters stay put
    (DynamicFilterEvaluator stops at an empty selection).  If they moved, filter 1 would pass 2047 positions on the second page and
    switch off one page early."""
    domains = [df.Domain(0, df.DISCRETE, False, values=list(range(0, 100))), df.Domain(1, df.ALL, True)]
    pages = [_seq_page(np.arange(2000) % 100), _seq_page(np.full(700, 500)), _seq_page(np.full(300, 7)), _seq_page(np.arange(100))]
    states = _profile(ctx, domains, 0.5, pages)
    # filter 0: 2000/2000 (not judged), 2000/2700 -> off; filter 1: 2000/2000, still 2000 (starved), then 2300/2300 -> off
    assert states == [[True, True], [False, True], [False, False], [False, False]]


def test_update_mid_stream_resets_every_counter(ctx):
    """update() installs a new predicate with a fresh profiler, whatever the number of domains before and after"""
    rng = np.random.default_rng(8)
    first = [df.Domain(0, df.RANGE, False, lo=0, hi=900), df.Domain(1, df.ALL, True)]
    op = ops.DynamicFilterOperatorFactory(ctx, [_gpu(d) for d in first], 0.5).create_operator()
    ev = df.DynamicFilterEvaluator(first, 0.5)
    page = lambda n: _feed(ctx, Page(Block.bigint(rng.integers(0, 1000, n)), Block.bigint(rng.integers(0, 1000, n)),
                                     Block.smallint(rng.integers(0, 1000, n).astype(np.int16))), "none")
    try:
        for n in (1000, 1000):
            _step(ctx, op, ev, page(n), "before the update")
        for domains in ([df.Domain(0, df.RANGE, False, lo=0, hi=950), df.Domain(2, df.DISCRETE, False, values=list(range(0, 999))),
                         df.Domain(1, df.RANGE, True, lo=5, hi=INT64_MAX)],
                        [df.Domain(2, df.RANGE, False, lo=10, hi=999)]):
            op.update([_gpu(d) for d in domains])
            ev = df.DynamicFilterEvaluator(domains, 0.5)
            for k, n in enumerate((1000, 1000, 40, 10, 2000)):
                _step(ctx, op, ev, page(n), f"after the update to {len(domains)} domains, page {k}")
    finally:
        op.close()


# ---- end to end: build-side key domain -> dynamic filter -> probe ------------------------------------------------------------------------
@pytest.mark.parametrize("max_values", [10_000, 16])
@pytest.mark.parametrize("tname", ["bigint", "integer", "date", "smallint", "tinyint", "decimal(18,2)"])
def test_key_domain_filters_the_probe_without_changing_the_join(ctx, tname, max_values):
    """The build side's key domain (DISCRETE while the distinct keys fit max_values, else RANGE [min, max]; NONE for no keys) in front of
    the probe drops only rows that cannot match: the inner join of the filtered pages equals the oracle's join of the unfiltered ones, row
    for row and in order.  Probe keys have NULLs and come flat and dictionary encoded."""
    make, lo, hi, _ = INT_TYPES[tname]
    rng = np.random.default_rng(len(tname) * 100 + max_values)
    span = min(hi, 120) - max(lo, -120)
    build_keys = rng.integers(max(lo, -120), min(hi, 120), 400, endpoint=True)[:: 1 + span // 100]
    build = Page(make(build_keys, rng.random(len(build_keys)) < 0.1), Block.bigint(np.arange(len(build_keys))))
    probes = [Page(make(rng.integers(max(lo, -128), min(hi, 127), n, endpoint=True), rng.random(n) < 0.1), Block.bigint(np.arange(n))) for n in (3000, 1)]
    dict_keys = make(rng.integers(max(lo, -128), min(hi, 127), 50, endpoint=True), rng.random(50) < 0.2)
    probes.append(Page(DictionaryBlock(dict_keys, rng.integers(0, 50, 2500)), Block.bigint(np.arange(2500))))
    for build_page in (build, Page(make([], None), Block.bigint([]), position_count=0)):
        bridge = ops.JoinBridge()
        b = ops.HashBuilderOperatorFactory(ctx, bridge, [0], [1]).create_operator()
        b.add_input(build_page)
        b.finish()
        lk = bridge.lookup_source
        klo, khi, cnt, values, _ = lk.key_domain(max_values)
        if cnt == 0:
            domain = ops.ColumnDomain.none(0)
        elif values is not None:
            domain = ops.ColumnDomain.multiple_values(0, values.tolist())
        else:
            domain = ops.ColumnDomain.range(0, klo, khi + 1)
        f = ops.DynamicFilterOperatorFactory(ctx, [domain]).create_operator()
        filtered = ops.drive(f, probes)
        f.close()
        j = ops.LookupJoinOperatorFactory(ctx, bridge, abi.JOIN_INNER, False, [0], [0, 1]).create_operator()
        got = [r for p in ops.drive(j, filtered) for r in p.rows()]
        j.close(); b.close(); lk.close()
        flat = [Page(*[b.flatten() for b in p.blocks]) for p in probes]
        want = [r for p in flat for r in oracle_join_rows(build_page, p, 0, 0, [0, 1], [1], abi.JOIN_INNER, False)]
        assert got == want, f"{tname} build of {build_page.position_count} rows"
        assert sum(p.position_count for p in filtered) < sum(p.position_count for p in probes)     # the filter did drop rows
