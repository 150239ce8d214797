"""VARCHAR predicates in every FilterAndProject form against an exact reference (varchar_reference.py, like_reference.py).

Forms, each fed the same pages:
- chunked:             a filter with fixed-width pass-through channels (the two-pass form without a selection vector)
- selection_vector:    the same program with TGPU_FP_SELECTION_VECTOR=1
- varchar_passthrough: a VARCHAR pass-through channel, which only the selection-vector form handles
- no_filter:           no filter; the string predicates are BOOLEAN output columns
test_interpreter_forms_in_child_process runs the file again with TGPU_DISABLE_JIT=1 (fp_filter_kernel / fp_project_kernel).

Programs are seeded random trees that mix string predicates with numeric operations, one of which raises DIVISION_BY_ZERO, so AND / OR
short-circuit and error placement next to string operations are checked.  Strings cover the empty string, equal prefixes, strings that
differ in their last byte, bytes >= 0x80, NUL bytes, 2- to 4-byte UTF-8, malformed UTF-8 and strings of several KB, with NULLs; blocks are
flat, DICT32 and RLE, on host and device pages.
"""
import os
import random
import subprocess
import sys

import numpy as np
import pytest

import varchar_reference as vref
from trino_b200 import abi
from trino_b200 import operators as ops
from trino_b200.page import Block, DictionaryBlock, Page, RunLengthEncodedBlock

pytestmark = pytest.mark.gpu
B, BOOL, S = abi.V_BIGINT, abi.V_BOOLEAN, abi.V_VARCHAR
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NO_JIT = bool(os.environ.get("TGPU_DISABLE_JIT"))
FORMS = ("chunked", "selection_vector", "varchar_passthrough", "no_filter")

SHIPMODES = [b"REG AIR", b"AIR", b"RAIL", b"SHIP", b"TRUCK", b"MAIL", b"FOB"]
INSTRUCTIONS = [b"DELIVER IN PERSON", b"COLLECT COD", b"NONE", b"TAKE BACK RETURN"]
POOL = sorted(set(SHIPMODES + INSTRUCTIONS + [
    b"", b"a", b"ab", b"abc", b"abd", b"ab\x00", b"a\x00b", b"\x00", b"a\xff", b"a\x80", b"\xff\xff", b"MAI", b"MAILS", b"MAIL\x00",
    b"BUILDING", b"BUILDINGS", b"Brand#45", b"Brand#44", b"MEDIUM POLISHED BRASS", b"MEDIUM POLISHED TIN", b"LARGE BRUSHED BRASS",
    b"forest green chiffon", b"green", b"greeN", b"F", b"O", b"P", b"ASIA", b"EUROPE",
    "café 名誉 \U0001F600 special".encode(), "é".encode(), "名".encode(), "\U0001F600".encode(),
    b"x\xc3(y", b"xa\xc3(y", b"xa\xffy", b"x\xe2\x82y", b"\xc3", b"\xf0\x9f\x98",
    b"quickly special packages wake requests", b"special requests", b"requests special", b"specialrequests",
    b"the special deposits sleep among the requests furiously", b"specia requests",
    b"s" * 4000, b"s" * 3999 + b"t", (b"special" * 300) + b"requests", b"xyza1234567890123456", b"x%_abcx", b"\\abc%",
]))
SHORT = [p for p in POOL if len(p) < 100]     # constants of the random programs (the pool of one program holds at most 4096 bytes)
PATTERNS = [  # (pattern, escape): a literal prefix / suffix only, FJS, DFA, NFA, escapes
    ("%special%requests%", None), ("MEDIUM POLISHED%", None), ("%BRASS", None), ("%green%", None), ("_", None), ("__", None),
    ("a_%", None), ("%_", None), ("x%a_y", None), ("%a%b_", None), ("%e_u%", None), ("x_%y", None), ("_a%b_", None), ("%", None),
    ("xxx%x_abcxx", "x"), ("\\\\abc\\%", "\\"), ("%a________________", None), ("café%", None), ("%名_%", None),
    ("%\U0001F600%", None), ("%_\U0001F600%", None), ("", None),
]


# ---- pages ---------------------------------------------------------------------------------------------------------------------
class Data:
    """columns: c0 VARCHAR (NULLs), c1 VARCHAR, c2 BIGINT (NULLs, zeros), c3 INTEGER, c4 VARCHAR (ship instruction)"""

    def __init__(self, n, seed, long_strings=True):
        rng = np.random.default_rng(seed)
        pool = POOL if long_strings else [p for p in POOL if len(p) < 100]
        pick = lambda k: [pool[i] for i in rng.integers(0, len(pool), k)]
        self.n = n
        self.c0 = [None if x else v for x, v in zip(rng.random(n) < 0.15, pick(n))]
        self.c1 = pick(n)
        self.c2 = [None if x else int(v) for x, v in zip(rng.random(n) < 0.1, rng.integers(-3, 4, n))]
        self.c3 = rng.integers(-50, 50, n).astype(np.int32)
        self.c4 = [INSTRUCTIONS[i] for i in rng.integers(0, 4, n)]

    def rows(self, idx):
        return [(self.c0[i], self.c1[i], self.c2[i], int(self.c3[i]), self.c4[i]) for i in idx]

    def page(self, idx, encoding="flat"):
        idx = list(idx)
        c2 = [self.c2[i] for i in idx]
        blocks = [Block.varchar([self.c0[i] for i in idx]), Block.varchar([self.c1[i] for i in idx]),
                  Block.bigint(np.array([0 if v is None else v for v in c2], np.int64), np.array([v is None for v in c2]) if any(v is None for v in c2) else None),
                  Block.integer(self.c3[idx]), Block.varchar([self.c4[i] for i in idx])]
        if encoding == "dict":
            for c in (0, 1, 4):
                vals = [blocks[c].get(k) for k in range(len(idx))]
                uniq = sorted(set(vals), key=lambda v: (v is None, v or b""))
                pos = {v: k for k, v in enumerate(uniq)}
                blocks[c] = DictionaryBlock(Block.varchar(uniq), np.array([pos[v] for v in vals], np.int32))
        return Page(*blocks, position_count=len(idx))


def rle_page(value, n):
    """every channel RLE but c3"""
    return Page(RunLengthEncodedBlock(Block.varchar([value]), n), RunLengthEncodedBlock(Block.varchar([value]), n),
                RunLengthEncodedBlock(Block.bigint(np.array([1], np.int64)), n), Block.integer(np.arange(n, dtype=np.int32) % 7),
                RunLengthEncodedBlock(Block.varchar([b"NONE"]), n))


# ---- random programs ------------------------------------------------------------------------------------------------------------
C0, C1, C2, C3, C4 = ops.Col(0, S), ops.Col(1, S), ops.Col(2, B), ops.Col(3, B), ops.Col(4, S)


def _const(rng):
    return ops.Const(rng.choice(SHORT), S)


def string_leaf(rng):
    col = rng.choice([C0, C1, C4])
    k = rng.randrange(9)
    if k == 0:
        return ops.Call(rng.choice([abi.EX_EQ, abi.EX_NE]), col, _const(rng))
    if k == 1:
        return ops.Call(rng.choice([abi.EX_LT, abi.EX_LE, abi.EX_GT, abi.EX_GE]), col, _const(rng))
    if k == 2:
        return ops.Call(rng.choice([abi.EX_EQ, abi.EX_NE, abi.EX_LT, abi.EX_GE]), C0, C1)
    if k == 3:
        lo, hi = sorted([rng.choice(SHORT), rng.choice(SHORT)])
        return ops.Call(abi.EX_BETWEEN, col, ops.Const(lo, S), ops.Const(hi, S))
    if k == 4:
        return ops.Call(abi.EX_IN, col, in_list=rng.sample(SHORT, rng.randrange(1, 5)))
    if k == 5:
        return ops.Call(rng.choice([abi.EX_IS_NULL, abi.EX_IS_NOT_NULL]), col)
    if k == 6:
        return ops.Call(abi.EX_EQ, col, ops.Null(S))
    p, e = rng.choice(PATTERNS)
    return ops.Call(abi.EX_LIKE, col, pattern=p, escape=e)


def numeric_leaf(rng):
    k = rng.randrange(3)
    if k == 0:
        return ops.Call(abi.EX_GT, ops.Call(abi.EX_DIV, C3, C2), ops.Const(1, B))       # raises where c2 = 0
    if k == 1:
        return ops.Call(abi.EX_EQ, C2, ops.Const(rng.randrange(-3, 4), B))
    return ops.Call(abi.EX_IS_NULL, C2)


def tree(rng, depth):
    if depth == 0 or rng.random() < 0.3:
        return string_leaf(rng) if rng.random() < 0.8 else numeric_leaf(rng)
    k = rng.randrange(3)
    if k == 2:
        return ops.Call(abi.EX_NOT, tree(rng, depth - 1))
    return ops.Call(abi.EX_AND if k == 0 else abi.EX_OR, tree(rng, depth - 1), tree(rng, depth - 1))


def random_program(seed):
    rng = random.Random(seed)
    return tree(rng, 2), [string_leaf(rng), tree(rng, 1)]


# ---- one form over one set of pages ---------------------------------------------------------------------------------------------
def form_outputs(form, projs):
    exprs = [("expr", p) for p in projs]
    if form in ("chunked", "selection_vector"):
        return [("pass", 3), ("pass", 2)] + exprs
    if form == "varchar_passthrough":
        return [("pass", 0)] + exprs + [("pass", 3)]
    return exprs + [("pass", 3)]


def expected(filt, outputs, rows):
    """(error codes, selected row positions, [column values]) as PageProcessor gives them"""
    sel, errors = [], set()
    for i, r in enumerate(rows):
        if filt is None:
            sel.append(i)
            continue
        v, err = vref.try_evaluate(filt, r)
        if err is not None:
            errors.add(err)
        elif v is True:
            sel.append(i)
    if errors:
        return errors, sel, None
    cols = []
    for kind, e in outputs:
        if kind == "pass":
            cols.append([rows[i][e] for i in sel])
            continue
        col = []
        for i in sel:
            v, err = vref.try_evaluate(e, rows[i])
            if err is not None:
                errors.add(err)
            col.append(None if v is None else int(v))
        cols.append(col)
    return errors, sel, cols


def got_columns(pages, ncols):
    cols = [[] for _ in range(ncols)]
    for p in pages:
        for c in range(ncols):
            b = p.get_block(c)
            cols[c] += [v if isinstance(v, (bytes, type(None))) else int(v) for v in b.to_pylist()]
    return cols


def run_fp(ctx, prog, pages):
    op = ops.FilterAndProjectOperatorFactory(ctx, prog).create_operator()
    try:
        return ops.drive(op, pages)
    finally:
        op.close()


def check(ctx, form, filt, projs, data, idx, encoding="flat", monkeypatch=None, page=None):
    if form == "selection_vector":
        monkeypatch.setenv("TGPU_FP_SELECTION_VECTOR", "1")
    if form == "no_filter":
        filt = None
    elif filt is None:
        filt = ops.Const(True, BOOL)
    outputs = form_outputs(form, projs)
    prog = ops.PageProcessorProgram(filt, [e for _, e in outputs])
    rows = data.rows(idx) if page is None else [tuple(page.get_block(c).get(i) for c in range(5)) for i in range(page.position_count)]
    errors, sel, want = expected(filt, outputs, rows)
    pg = page if page is not None else data.page(idx, encoding)
    if errors:
        with pytest.raises(abi.TrinoGpuError) as exc:
            run_fp(ctx, prog, [pg])
        assert exc.value.code in errors, (form, str(exc.value), errors)
        return "raised"
    got = got_columns(run_fp(ctx, prog, [pg]), len(outputs))
    for c, (w, g) in enumerate(zip(want, got)):
        if w != g:
            r = next((k for k, (a, b) in enumerate(zip(w, g)) if a != b), min(len(w), len(g)))
            row = rows[sel[r]] if r < len(sel) else None
            raise AssertionError(f"{form}: output {c} {outputs[c]} differs at output row {r} of {len(w)} / {len(g)}: want "
                                 f"{w[r] if r < len(w) else '<end>'!r} got {g[r] if r < len(g) else '<end>'!r}; row {row!r}")
    return len(sel)


# ---- tests ----------------------------------------------------------------------------------------------------------------------
_DATA = {}


def data(n, seed=7, long_strings=True):
    key = (n, seed, long_strings)
    if key not in _DATA:
        _DATA[key] = Data(n, seed, long_strings)
    return _DATA[key]


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("seed", range(24))
def test_random_programs(ctx, seed, form, monkeypatch):
    """seeded trees over a 3000-row page (three 1024-row tiles); a page that raises is checked for the code, then its clean rows"""
    d = data(3000)
    filt, projs = random_program(seed)
    idx = np.arange(d.n)
    if check(ctx, form, filt, projs, d, idx, monkeypatch=monkeypatch) == "raised":
        rows = d.rows(idx)
        clean = [i for i, r in zip(idx, rows) if all(vref.try_evaluate(e, r)[1] is None for e in [filt] + projs)]
        check(ctx, form, filt, projs, d, np.array(clean, np.int64), monkeypatch=monkeypatch)


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("pattern,escape", PATTERNS)
def test_like_patterns(ctx, pattern, escape, form, monkeypatch):
    """each LIKE pattern (every matcher) over every pool string, NULLs included, as filter and as output column"""
    d = data(len(POOL) * 3, seed=11)
    like = ops.Call(abi.EX_LIKE, C1, pattern=pattern, escape=escape)
    check(ctx, form, like, [like, ops.Call(abi.EX_LIKE, C0, pattern=pattern, escape=escape)], d, np.arange(d.n), monkeypatch=monkeypatch)


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("encoding", ["flat", "dict"])
def test_encodings_and_comparisons(ctx, encoding, form, monkeypatch):
    """every comparison of c0 with every pool constant, over flat and DICT32 blocks"""
    d = data(2500, seed=3)
    rng = random.Random(5)
    for k in range(6):
        const = ops.Const(POOL[rng.randrange(len(POOL))], S)
        projs = [ops.Call(op, C0, const) for op in (abi.EX_EQ, abi.EX_NE, abi.EX_LT, abi.EX_LE, abi.EX_GT, abi.EX_GE)]
        check(ctx, form, ops.Call(abi.EX_GE, C1, const), projs, d, np.arange(d.n), encoding, monkeypatch)


@pytest.mark.parametrize("form", FORMS)
def test_rle_blocks(ctx, form, monkeypatch):
    for v in (b"MAIL", b"", b"s" * 4000, None):
        page = rle_page(v, 2048 + 17)
        filt = ops.Call(abi.EX_OR, ops.Call(abi.EX_IN, C0, in_list=["MAIL", "SHIP"]), ops.Call(abi.EX_IS_NULL, C1))
        check(ctx, form, filt, [ops.Call(abi.EX_LIKE, C1, pattern="%s%"), ops.Call(abi.EX_EQ, C4, ops.Const("NONE", S))], None, None,
              monkeypatch=monkeypatch, page=page)


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


TPCH = {
    "q12_shipmode_in": ops.Call(abi.EX_IN, C1, in_list=["MAIL", "SHIP"]),
    "q19_conjunct": ops.Call(abi.EX_AND, ops.Call(abi.EX_IN, C1, in_list=["AIR", "REG AIR"]), ops.Call(abi.EX_EQ, C4, ops.Const("DELIVER IN PERSON", S))),
    "q13_not_like": ops.Call(abi.EX_NOT, ops.Call(abi.EX_LIKE, C0, pattern="%special%requests%")),
    "q3_mktsegment": ops.Call(abi.EX_EQ, C1, ops.Const("BUILDING", S)),
    "q9_name_like": ops.Call(abi.EX_LIKE, C1, pattern="%green%"),
    "q2_type_like": ops.Call(abi.EX_LIKE, C1, pattern="%BRASS"),
    "q16_brand_type": ops.Call(abi.EX_AND, ops.Call(abi.EX_NE, C1, ops.Const("Brand#45", S)),
                               ops.Call(abi.EX_NOT, ops.Call(abi.EX_LIKE, C0, pattern="MEDIUM POLISHED%"))),
    "q21_orderstatus": ops.Call(abi.EX_EQ, C1, ops.Const("F", S)),
    "q5_region": ops.Call(abi.EX_EQ, C1, ops.Const("ASIA", S)),
}


@pytest.mark.parametrize("name", sorted(TPCH))
def test_tpch_predicates_on_device_pages(ctx, name):
    """the TPC-H predicates over synthetic columns, on a device-resident page, row for row (chunked form)"""
    d = data(20000, seed=19, long_strings=False)
    idx = np.arange(d.n)
    page = d.page(idx)
    dp = _device_page(ctx, page)
    filt = TPCH[name]
    prog = ops.PageProcessorProgram(filt, [3, 2])
    _, sel, want = expected(filt, [("pass", 3), ("pass", 2)], d.rows(idx))
    got = got_columns(run_fp(ctx, prog, [dp]), 2)
    assert got == want, name
    assert len(sel) > 0 or name == "q21_orderstatus"


def test_million_row_page(ctx):
    """one page of 1 M rows (many chunks and tiles): the Q19 conjunct and a LIKE, filter + output"""
    rng = np.random.default_rng(23)
    n = 1 << 20
    modes, instr = rng.integers(0, len(SHIPMODES), n), rng.integers(0, len(INSTRUCTIONS), n)
    def utf8_block(pool, ids):
        lens = np.array([len(pool[i]) for i in ids], np.int64)
        offsets = np.zeros(n + 1, np.int32)
        np.cumsum(lens, out=offsets[1:])
        data = np.frombuffer(b"".join(pool[i] for i in ids), np.uint8).copy()
        return Block(abi.UTF8, data, None, offsets)
    page = Page(utf8_block(SHIPMODES, modes), utf8_block(SHIPMODES, modes), Block.bigint(np.arange(n, dtype=np.int64)),
                Block.integer(np.arange(n, dtype=np.int32)), utf8_block(INSTRUCTIONS, instr))
    filt = TPCH["q19_conjunct"]
    like = ops.Call(abi.EX_LIKE, C0, pattern="%AI%")
    prog = ops.PageProcessorProgram(filt, [2, like])
    out = run_fp(ctx, prog, [page])
    modes_ok = np.isin(modes, [SHIPMODES.index(b"AIR"), SHIPMODES.index(b"REG AIR")]) & (instr == 0)
    want_rows = np.nonzero(modes_ok)[0]
    got_rows = np.concatenate([p.get_block(0).values for p in out])
    assert np.array_equal(got_rows, want_rows)
    got_like = np.concatenate([p.get_block(1).values for p in out]).astype(bool)
    assert np.array_equal(got_like, np.array([b"AI" in SHIPMODES[m] for m in modes[want_rows]]))


def test_refusals_that_need_a_context(ctx):
    like = ops.Call(abi.EX_LIKE, C1, pattern="%a%")
    # fused aggregation pre-stage: NOT_SUPPORTED at create
    prog = ops.PageProcessorProgram(like, [3, 2])
    for global_agg in (False, True):
        with pytest.raises(abi.TrinoGpuError) as exc:
            if global_agg:
                ops.AggregationOperatorFactory(ctx, abi.STEP_SINGLE, [ops.Aggregator(abi.AGG_COUNT_STAR)], pre=prog,
                                               input_types=[abi.UTF8, abi.UTF8, abi.INT64, abi.INT32]).create_operator()
            else:
                ops.HashAggregationOperatorFactory(ctx, [0], abi.STEP_SINGLE, [ops.Aggregator(abi.AGG_COUNT_STAR)], expected_groups=16,
                                                   pre=prog).create_operator()
        assert exc.value.code == abi.ERR_NOT_SUPPORTED, str(exc.value)
    # a filtered join build: NOT_SUPPORTED at create
    with pytest.raises(abi.TrinoGpuError) as exc:
        ops.HashBuilderOperatorFactory(ctx, ops.JoinBridge(), [0], [1], filter=ops.Call(abi.EX_EQ, ops.Col(1, S), ops.Col(3, S)),
                                       num_build_channels=2).create_operator()
    assert exc.value.code == abi.ERR_NOT_SUPPORTED, str(exc.value)
    # a VARCHAR operation over a channel that is not UTF8 on the page: INVALID_ARGUMENT at that page
    d = data(100, seed=1, long_strings=False)
    prog = ops.PageProcessorProgram(ops.Call(abi.EX_EQ, ops.Col(3, S), ops.Const("x", S)), [3])
    with pytest.raises(abi.TrinoGpuError) as exc:
        run_fp(ctx, prog, [d.page(np.arange(100))])
    assert exc.value.code == abi.ERR_INVALID_ARGUMENT, str(exc.value)
    # a numeric operation over a UTF8 channel keeps NOT_SUPPORTED
    prog = ops.PageProcessorProgram(ops.Call(abi.EX_EQ, ops.Col(0, B), ops.Const(1, B)), [3])
    with pytest.raises(abi.TrinoGpuError) as exc:
        run_fp(ctx, prog, [d.page(np.arange(100))])
    assert exc.value.code == abi.ERR_NOT_SUPPORTED, str(exc.value)


def test_interpreter_forms_in_child_process():
    """fp_filter_kernel / fp_project_kernel (vm_run's string branch): the kernels that run where NVRTC is off"""
    if NO_JIT:
        pytest.skip("already the child")
    env = dict(os.environ, TGPU_DISABLE_JIT="1")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", "-p", "no:cacheprovider", os.path.abspath(__file__)],
                       cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-6000:]
    assert " passed" in r.stdout and "1 skipped" in r.stdout, r.stdout[-2000:]
