"""String functions in FilterAndProject (length, substr, ltrim / rtrim / trim, concat) against string_function_reference.py, byte for byte:
the offsets, bytes and validity of every VARCHAR output column.

Forms, each fed the same pages:
- chunked:             a filter with fixed-width pass-through channels (the two-pass form without a selection vector)
- selection_vector:    the same program with TGPU_FP_SELECTION_VECTOR=1
- varchar_passthrough: a VARCHAR pass-through channel, which only the selection-vector form handles
- no_filter:           no filter (the all-rows projection)
test_interpreter_forms_in_child_process runs the file again with TGPU_DISABLE_JIT=1 (fp_filter_kernel / fp_project_kernel).
"""
import os
import subprocess
import sys

import numpy as np
import pytest

import string_function_reference as sref
from agg_reference import aggregate
from trino_b200 import abi
from trino_b200 import operators as ops
from trino_b200.page import Block, DictionaryBlock, Page, RunLengthEncodedBlock

pytestmark = pytest.mark.gpu
B, BOOL, S = abi.V_BIGINT, abi.V_BOOLEAN, abi.V_VARCHAR
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NO_JIT = bool(os.environ.get("TGPU_DISABLE_JIT"))
FORMS = ("chunked", "selection_vector", "varchar_passthrough", "no_filter")
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1

WS = ["\t", "\n", "\r", "\x1f", " ", "\u1680", "\u2000", "\u2028", "\u2029", "\u3000"]      # Character.isWhitespace
NOT_WS = ["\u00a0", "\u2007", "\u202f"]
POOL = [b"", b"a", b"ab", b" ", b"  ", b"hello", b"  hello world  ", b"Quadratically", b"13-555-123-4567", b"31-101-000-0000",
        b"DELIVER IN PERSON", b"1-URGENT", b"Clerk#000000951"] + [s.encode() for s in [
            "a\u00f1\u540d\U0001F600z", "\u4fe1\u5ff5,\u7231,\u5e0c\u671b", "\U0001F600", "\u00e9", "na\u00efve caf\u00e9", "\u2028 x \u2028", "\u00a0x\u00a0", "\u2007\u202fy\u2007",
            "".join(WS) + "mid" + "".join(WS), "".join(NOT_WS) + "k", "\U0001F600 \U0001F600 "]] + [
        b"\x80\x80a", b"a\xc3", b"\xf0\x9f\x98", b"\xff\xfe", b" \xc3 ", b"x\xe2\x80\xa8", b"s" * 300, "\u540d".encode() * 50]
EDGE = [0, 1, -1, 2, -2, 3, -3, 4, 5, 6, -5, -6, 12, 13, 14, -13, -14, 50, -50, INT64_MIN, INT64_MAX, INT64_MIN + 1, INT64_MAX - 1,
        (1 << 31) - 1, 1 << 31, -(1 << 31), -(1 << 31) - 1]


class Data:
    """c0 VARCHAR (NULLs), c1 VARCHAR, c2 BIGINT start (NULLs, edge values), c3 BIGINT length (edge values), c4 INTEGER"""

    def __init__(self, n, seed):
        rng = np.random.default_rng(seed)
        pick = lambda k: [POOL[i] for i in rng.integers(0, len(POOL), k)]
        self.n = n
        self.c0 = [None if x else v for x, v in zip(rng.random(n) < 0.15, pick(n))]
        self.c1 = pick(n)
        self.c2 = [None if x else EDGE[i] for x, i in zip(rng.random(n) < 0.1, rng.integers(0, len(EDGE), n))]
        self.c3 = [EDGE[i] for i in rng.integers(0, len(EDGE), n)]
        self.c4 = rng.integers(-50, 50, n).astype(np.int32)

    def rows(self, idx):
        return [(self.c0[i], self.c1[i], self.c2[i], self.c3[i], int(self.c4[i])) for i in idx]

    def page(self, idx, encoding="flat"):
        idx = list(idx)
        c2 = [self.c2[i] for i in idx]
        v0 = [self.c0[i] for i in idx]
        b0 = Block.varchar(v0)
        if encoding == "offset":
            # a UTF8 block whose offsets start past 0, behind bytes no row owns
            b0 = Block(abi.UTF8, np.concatenate([np.frombuffer(b"junk\xff" * 3, np.uint8), b0.values]), b0.nulls, b0.offsets + 15)
        blocks = [b0, Block.varchar([self.c1[i] for i in idx]),
                  Block.bigint(np.array([0 if v is None else v for v in c2], np.int64), np.array([v is None for v in c2]) if any(v is None for v in c2) else None),
                  Block.bigint(np.array([self.c3[i] for i in idx], np.int64)), Block.integer(self.c4[idx])]
        if encoding == "dict":
            for c in (0, 1):
                vals = [blocks[c].get(k) for k in range(len(idx))]
                uniq = sorted(set(vals), key=lambda v: (v is None, v or b""))
                pos = {v: k for k, v in enumerate(uniq)}
                blocks[c] = DictionaryBlock(Block.varchar(uniq), np.array([pos[v] for v in vals], np.int32))
        return Page(*blocks, position_count=len(idx))


C0, C1, C2, C3, C4 = ops.Col(0, S), ops.Col(1, S), ops.Col(2, B), ops.Col(3, B), ops.Col(4, B)
K = lambda v: ops.Const(v, B)
T = lambda v: ops.Const(v, S)
call = ops.Call


# ---- reference evaluation ------------------------------------------------------------------------------------------------------
def _leaves(e):
    if isinstance(e, ops.Call) and e.op == abi.EX_CONCAT:
        return _leaves(e.args[0]) + _leaves(e.args[1])
    return [e]


def ev(e, row):
    """the value of expression e over one row (None = NULL); raises sref.ConcatTooLarge"""
    if isinstance(e, ops.Col):
        return row[e.channel]
    if isinstance(e, ops.Const):
        return e.value.encode() if isinstance(e.value, str) else e.value
    if isinstance(e, ops.Null):
        return None
    op = e.op
    if op == abi.EX_CONCAT:
        return sref.concat(*[ev(x, row) for x in _leaves(e)])       # the variadic call the chain stands for
    a = [ev(x, row) for x in e.args]
    if op == abi.EX_IS_NULL:
        return a[0] is None
    if op in (abi.EX_AND, abi.EX_OR):
        x, y = a
        if op == abi.EX_AND:
            return False if (x is False or y is False) else None if (x is None or y is None) else True
        return True if (x is True or y is True) else None if (x is None or y is None) else False
    if any(v is None for v in a):
        return None
    if op == abi.EX_LENGTH:
        return sref.length(a[0])
    if op == abi.EX_SUBSTR:
        return sref.substring(a[0], a[1], a[2] if len(a) > 2 else None, java_int_wrap=False)
    if op in (abi.EX_LTRIM, abi.EX_RTRIM, abi.EX_TRIM):
        return {abi.EX_LTRIM: sref.ltrim, abi.EX_RTRIM: sref.rtrim, abi.EX_TRIM: sref.trim}[op](a[0])
    if op == abi.EX_IN:
        return a[0] in [v.encode() if isinstance(v, str) else v for v in e.in_list]
    if op == abi.EX_NOT:
        return not a[0]
    if op == abi.EX_BETWEEN:
        return a[1] <= a[0] <= a[2]
    cmp = {abi.EX_EQ: lambda x, y: x == y, abi.EX_NE: lambda x, y: x != y, abi.EX_LT: lambda x, y: x < y, abi.EX_GT: lambda x, y: x > y,
           abi.EX_LE: lambda x, y: x <= y, abi.EX_GE: lambda x, y: x >= y}
    return cmp[op](a[0], a[1])


def expected(filt, projs, rows):
    """(raises, selected rows, output columns): the filter for every row, then the projections of the selected rows"""
    sel, raises = [], False
    for i, r in enumerate(rows):
        try:
            if filt is None or ev(filt, r) is True:
                sel.append(i)
        except sref.ConcatTooLarge:
            raises = True
    cols = [[] for _ in projs]
    for i in sel:
        for c, p in enumerate(projs):
            try:
                cols[c].append(rows[i][p] if isinstance(p, int) else ev(p, rows[i]))
            except sref.ConcatTooLarge:
                raises = True
    return raises, sel, cols


def run_fp(ctx, prog, pages):
    op = ops.FilterAndProjectOperatorFactory(ctx, prog).create_operator()
    try:
        return ops.drive(op, pages)
    finally:
        op.close()


def check_utf8_block(b, want, what):
    """offsets, bytes and validity of one VARCHAR output block"""
    assert b.type == abi.UTF8, what
    lens = [0 if v is None else len(v) for v in want]
    assert list(np.asarray(b.offsets, np.int64)) == [0] + list(np.cumsum(lens, dtype=np.int64)), what
    assert bytes(np.asarray(b.values, np.uint8)[:sum(lens)]) == b"".join(v for v in want if v is not None), what
    nulls = [v is None for v in want]
    got_nulls = [False] * len(want) if b.nulls is None else [bool(x) for x in b.nulls]
    assert got_nulls == nulls, what


def check(ctx, form, filt, projs, rows, pages, monkeypatch):
    if form == "selection_vector":
        monkeypatch.setenv("TGPU_FP_SELECTION_VECTOR", "1")
    if form == "no_filter":
        filt = None
    elif filt is None:
        filt = ops.Const(True, BOOL)
    projs = list(projs) + ([0] if form == "varchar_passthrough" else [4, 3])
    prog = ops.PageProcessorProgram(filt, projs)
    raises, sel, want = expected(filt, projs, rows)
    if raises:
        with pytest.raises(abi.TrinoGpuError) as exc:
            run_fp(ctx, prog, pages)
        assert exc.value.code == abi.ERR_INVALID_FUNCTION_ARGUMENT and "Concatenated string is too large" in str(exc.value)
        return None
    out = run_fp(ctx, prog, pages)
    assert sum(p.position_count for p in out) == len(sel), form
    for c, p in enumerate(projs):
        if isinstance(p, int) or p.vtype != S:
            got = []
            for pg in out:
                got += [v if isinstance(v, (bytes, type(None))) else int(v) for v in pg.get_block(c).to_pylist()]
            assert got == want[c], (form, c)
            continue
        at = 0
        for pg in out:
            n = pg.position_count
            check_utf8_block(pg.get_block(c), want[c][at:at + n], (form, c))
            at += n
    return len(sel)


# ---- programs ------------------------------------------------------------------------------------------------------------------
EVERY = [
    call(abi.EX_LENGTH, C0), call(abi.EX_LENGTH, T("a\u00f1\u540d\U0001F600z")),
    call(abi.EX_SUBSTR, C0, C2), call(abi.EX_SUBSTR, C0, C2, C3), call(abi.EX_SUBSTR, C1, K(1), K(2)), call(abi.EX_SUBSTR, T("Quadratically"), C2, K(4)),
    call(abi.EX_LTRIM, C0), call(abi.EX_RTRIM, C1), call(abi.EX_TRIM, C0), call(abi.EX_TRIM, T("  x  ")),
    ops.concat(C0, C1), ops.concat(C1, T("-"), C0), ops.concat(T("store"), C1),
    # view temps as operands, and chains
    call(abi.EX_LENGTH, call(abi.EX_TRIM, call(abi.EX_SUBSTR, C0, K(-5)))),
    ops.concat(C0, T("-"), call(abi.EX_SUBSTR, C1, K(2), K(3))),
    call(abi.EX_SUBSTR, call(abi.EX_TRIM, C1), C2, C3), call(abi.EX_RTRIM, call(abi.EX_LTRIM, C0)),
    ops.concat(call(abi.EX_TRIM, C0), call(abi.EX_SUBSTR, C1, C2), T("|"), call(abi.EX_LTRIM, C1)),
    call(abi.EX_SUBSTR, call(abi.EX_SUBSTR, C0, K(2)), K(-3), K(2)),
    ops.concat(C0, ops.Null(S)), call(abi.EX_LENGTH, ops.Null(S)), call(abi.EX_SUBSTR, C0, ops.Null(B)),
]
FILTERS = {   # none, all, some and no rows selected
    "none": None,
    "all": call(abi.EX_GE, call(abi.EX_LENGTH, C1), K(0)),
    "some": call(abi.EX_IN, call(abi.EX_SUBSTR, C1, K(1), K(2)), in_list=["13", "31", "ab", "he", "  "]),
    "some_trim": call(abi.EX_GT, call(abi.EX_LENGTH, call(abi.EX_TRIM, C0)), K(2)),
    "no_rows": call(abi.EX_EQ, call(abi.EX_SUBSTR, C1, K(1), K(3)), T("zzz")),
}
_DATA = {}


def data(n, seed=7):
    if (n, seed) not in _DATA:
        _DATA[(n, seed)] = Data(n, seed)
    return _DATA[(n, seed)]


@pytest.mark.parametrize("filter_kind", sorted(FILTERS))
@pytest.mark.parametrize("form", FORMS)
def test_every_function(ctx, form, filter_kind, monkeypatch):
    d = data(3000)
    idx = np.arange(d.n)
    for k in range(0, len(EVERY), 3):      # three projections per program: within the 8 temporaries
        sel = check(ctx, form, FILTERS[filter_kind], EVERY[k:k + 3], d.rows(idx), [d.page(idx)], monkeypatch)
        if filter_kind == "no_rows" and form != "no_filter":
            assert sel == 0
        if filter_kind == "some" and form != "no_filter":
            assert 0 < sel < d.n


@pytest.mark.parametrize("encoding", ["dict", "offset", "rle", "device"])
@pytest.mark.parametrize("form", FORMS)
def test_block_shapes(ctx, form, encoding, monkeypatch):
    """DictionaryBlock, RunLengthEncodedBlock, UTF8 offsets that start past 0, device-resident pages"""
    d = data(2000, seed=11)
    idx = np.arange(d.n)
    rows = d.rows(idx)
    if encoding == "rle":
        v = "  \u540d x\u2028 ".encode()
        rows = [(v, v, 3, 2, int(r[4])) for r in rows]
        page = Page(RunLengthEncodedBlock(Block.varchar([v]), d.n), RunLengthEncodedBlock(Block.varchar([v]), d.n),
                    RunLengthEncodedBlock(Block.bigint(np.array([3], np.int64)), d.n), RunLengthEncodedBlock(Block.bigint(np.array([2], np.int64)), d.n),
                    Block.integer(d.c4[idx]))
        pages = [page]
    elif encoding == "device":
        pages = [_device_page(ctx, d.page(idx, "offset"))]
    else:
        pages = [d.page(idx, encoding)]
    projs = [EVERY[3], EVERY[14], EVERY[13], EVERY[17]]
    check(ctx, form, FILTERS["some_trim"], projs, rows, pages, monkeypatch)


@pytest.mark.parametrize("n", [1, 31, 32, 33, 1023, 1024, 1025, 300_001])
def test_page_sizes(ctx, n, monkeypatch):
    """pages of one row, of one tile (32 rows for the byte assembly, 1024 for the chunked form) +- 1, and of several chunks"""
    d = data(n, seed=n)
    idx = np.arange(n)
    projs = [call(abi.EX_SUBSTR, C1, K(1), K(2)), ops.concat(C0, T("-"), call(abi.EX_TRIM, C1))]
    for form in ("chunked", "no_filter"):
        check(ctx, form, FILTERS["some_trim"], projs, d.rows(idx), [d.page(idx)], monkeypatch)


def test_substr_start_and_length_edges(ctx, monkeypatch):
    """every start and length edge (0, +-1, the string length +- 1, INT64_MIN / INT64_MAX) over every string of the pool"""
    strs = POOL + [None]
    rows = [(s, s, a, b, 0) for s in strs for a in EDGE for b in EDGE[:14] + [INT64_MIN, INT64_MAX]]
    page = Page(Block.varchar([r[0] for r in rows]), Block.varchar([r[1] for r in rows]), Block.bigint(np.array([r[2] for r in rows], np.int64)),
                Block.bigint(np.array([r[3] for r in rows], np.int64)), Block.integer(np.zeros(len(rows), np.int32)))
    projs = [call(abi.EX_SUBSTR, C0, C2), call(abi.EX_SUBSTR, C0, C2, C3), call(abi.EX_LENGTH, C0)]
    for form in ("no_filter", "chunked"):
        check(ctx, form, None, projs, rows, [page], monkeypatch)


def test_concat_limit(ctx, monkeypatch):
    """1 MiB passes, 1 MiB + 1 raises INVALID_FUNCTION_ARGUMENT - in a selected row only; a NULL piece beside an oversized one raises
    nothing"""
    big = b"x" * (1 << 19)
    rows = [(big, big, 1, 0, 0), (big, b"", 1, 0, 0), (None, big + big, 1, 0, 0), (big, big + b"y", 0, 0, 0)]
    page = lambda rs: Page(Block.varchar([r[0] for r in rs]), Block.varchar([r[1] for r in rs]), Block.bigint(np.array([r[2] for r in rs], np.int64)),
                           Block.bigint(np.zeros(len(rs), np.int64)), Block.integer(np.zeros(len(rs), np.int32)))
    sel = call(abi.EX_EQ, C2, K(1))
    for form in ("chunked", "selection_vector", "no_filter"):
        # row 3 (1 MiB + 1) is rejected by the filter: no error where the filter runs; the all-rows form raises
        r = check(ctx, form, sel, [ops.concat(C0, C1)], rows, [page(rows)], monkeypatch)
        assert (r is None) == (form == "no_filter")
        monkeypatch.delenv("TGPU_FP_SELECTION_VECTOR", raising=False)
    # three pieces: the chain checks the total once, like the variadic call; a NULL third piece gives NULL and no error
    rows2 = [(big, big, 1, 0, 0)]
    assert check(ctx, "chunked", sel, [ops.concat(C0, C1, T("z"))], rows2, [page(rows2)], monkeypatch) is None
    assert check(ctx, "chunked", sel, [ops.concat(C0, C1, T("z"), ops.Null(S))], rows2, [page(rows2)], monkeypatch) == 1
    assert check(ctx, "chunked", sel, [ops.concat(C1, C0, ops.Null(S), C0)], rows2, [page(rows2)], monkeypatch) == 1


def test_column_byte_limit(ctx, monkeypatch):
    """a VARCHAR projection past the bytes a UTF8 column holds fails with INSUFFICIENT_RESOURCES before it is written (INT32_MAX,
    lowered here so that a small page reaches it)"""
    d = data(1000, seed=3)
    idx = np.arange(d.n)
    prog = ops.PageProcessorProgram(None, [ops.concat(C1, C1)])
    _, _, want = expected(None, [ops.concat(C1, C1)], d.rows(idx))
    total = sum(len(v) for v in want[0] if v is not None)
    monkeypatch.setenv("TGPU_UTF8_COLUMN_LIMIT", str(total))
    check_utf8_block(run_fp(ctx, prog, [d.page(idx)])[0].get_block(0), want[0], "at the limit")
    monkeypatch.setenv("TGPU_UTF8_COLUMN_LIMIT", str(total - 1))
    with pytest.raises(abi.TrinoGpuError) as exc:
        run_fp(ctx, prog, [d.page(idx)])
    assert exc.value.code == abi.ERR_INSUFFICIENT_RESOURCES


def test_refusals_at_create(ctx):
    for prog in (ops.PageProcessorProgram(call(abi.EX_EQ, ops.concat(C0, C1), T("x")), [4]),
                 ops.PageProcessorProgram(None, [call(abi.EX_LENGTH, ops.concat(C0, C1))])):
        with pytest.raises(abi.TrinoGpuError) as exc:
            ops.FilterAndProjectOperatorFactory(ctx, prog).create_operator()
        assert exc.value.code == abi.ERR_NOT_SUPPORTED


def _device_page(ctx, page):
    cols = []
    for c in range(page.channel_count):
        b = page.get_block(c)
        valid = None
        if b.nulls is not None:
            valid = ctx.to_device(np.packbits(~np.asarray(b.nulls, bool), bitorder="little"))
        if b.type == abi.UTF8:
            cols.append(ops.DeviceColumn(abi.UTF8, ctx.to_device(b.values), b.position_count, valid, ctx.to_device(b.offsets)))
        else:
            cols.append(ops.DeviceColumn(b.type, ctx.to_device(b.values), b.position_count, valid))
    return ops.DevicePage(cols, page.position_count)


def test_q22_pipeline_on_device_pages(ctx):
    """TPC-H Q22's customer scan: substring(c_phone, 1, 2) IN (...) as the filter and as the projected key, then
    HashAggregationOperator keyed on it (count(*), sum(c_acctbal)), device page to device page, against the exact aggregate"""
    rng = np.random.default_rng(22)
    n = 200_000
    phones = [f"{c}-{rng.integers(100, 999)}-{rng.integers(100, 999)}-{rng.integers(1000, 9999)}".encode() for c in rng.integers(10, 35, n)]
    bal = rng.integers(-99999, 999999, n).astype(np.int64)
    page = Page(Block.varchar(phones), Block.bigint(bal))
    codes = ["13", "31", "23", "29", "30", "18", "17"]
    key = call(abi.EX_SUBSTR, ops.Col(0, S), K(1), K(2))
    filt = call(abi.EX_AND, call(abi.EX_IN, key, in_list=codes), call(abi.EX_GT, ops.Col(1, B), K(0)))
    prog = ops.PageProcessorProgram(filt, [key, 1])
    fp = ops.FilterAndProjectOperatorFactory(ctx, prog).create_operator()
    agg = ops.HashAggregationOperatorFactory(ctx, [0], abi.STEP_SINGLE, [ops.Aggregator(abi.AGG_COUNT_STAR), ops.Aggregator(abi.AGG_SUM, 1)], 64).create_operator()
    try:
        fp.add_input(_device_page(ctx, page))
        mid = []
        while True:
            o = fp.get_output_device()
            if o is None:
                break
            mid.append(o.to_host())
            agg.add_input(o)
            o.release()
        agg.finish()
        rows = []
        while not agg.is_finished():
            p = agg.get_output()
            if p is not None:
                rows.extend(p.rows())
    finally:
        fp.close()
        agg.close()
    _, _, want_cols = expected(filt, [key, 1], [(phones[i], int(bal[i])) for i in range(n)])
    ref_page = Page(Block.varchar(want_cols[0]), Block.bigint(np.array(want_cols[1], np.int64)))
    want = aggregate([ref_page], [0], [(abi.AGG_COUNT_STAR, -1, -1), (abi.AGG_SUM, 1, -1)])
    assert sorted(rows) == sorted(want)
    assert len(want) == len(codes)
    assert [p.get_block(0).to_pylist() for p in mid] and sum(p.position_count for p in mid) == len(want_cols[0])


def test_interpreter_forms_in_child_process():
    """fp_filter_kernel / fp_project_kernel (vm_run's string branch): the kernels that run where NVRTC is off"""
    if NO_JIT:
        pytest.skip("already the child")
    env = dict(os.environ, TGPU_DISABLE_JIT="1")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", "-p", "no:cacheprovider", os.path.abspath(__file__)],
                       cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-6000:]
    assert " passed" in r.stdout and "1 skipped" in r.stdout, r.stdout[-2000:]
