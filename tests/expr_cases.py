"""Seeded expression programs and pages for the evaluator tests, and the expected results of every form of the evaluator.

A case is a program (filter + projections over typed channels) and pages of rows drawn from a pool of at most POOL distinct rows:
the reference (expr_reference) evaluates each pool row once, so pages of millions of rows cost no more on the host than a few
thousand.  Page sizes straddle the 1024-row tiles of the chunked FilterAndProject form; columns are TINYINT, SMALLINT, INTEGER,
BIGINT, DOUBLE and BOOLEAN, non-nullable, about 30% NULL or all NULL, as flat, dictionary or RLE blocks; half of their values come
from pools of edge values.
"""
import math
import struct

import numpy as np

import expr_reference as ref
from trino_b200 import abi
from trino_b200 import operators as ops
from trino_b200.page import Block, DictionaryBlock, Page, RunLengthEncodedBlock

B, D, BOOL = abi.V_BIGINT, abi.V_DOUBLE, abi.V_BOOLEAN
I64_MIN, I64_MAX = ref.INT64_MIN, ref.INT64_MAX
POOL = 4096
SIZES = (1, 7, 1023, 1024, 1025, 4097, 300_001)
BIG_PAGE = 2_000_003          # several chunks of the chunked form

# channel layout of the random cases; Case appends a TINYINT key channel and a VARCHAR channel to every case
RANDOM_TYPES = (abi.INT8, abi.INT16, abi.INT32, abi.INT64, abi.FLOAT64, "boolean", abi.FLOAT64, abi.INT64)
VTYPE_OF = {abi.INT8: B, abi.INT16: B, abi.INT32: B, abi.INT64: B, abi.FLOAT64: D, "boolean": BOOL}
_NP = {abi.INT8: np.int8, abi.INT16: np.int16, abi.INT32: np.int32, abi.INT64: np.int64, abi.FLOAT64: np.float64, "boolean": np.int8}
_BLOCK = {abi.INT8: Block.tinyint, abi.INT16: Block.smallint, abi.INT32: Block.integer, abi.INT64: Block.bigint, abi.FLOAT64: Block.double,
          "boolean": Block.boolean}

_P63 = 2.0 ** 63
DOUBLE_EDGES = (0.0, -0.0, math.nan, math.inf, -math.inf, 5e-324, 1.7976931348623157e308, -1.7976931348623157e308, 1.0, -1.0,
                0.5, -0.5, 1.5, -1.5, 2.5, -2.5, 0.49999999999999994, _P63, -_P63, math.nextafter(_P63, 0), math.nextafter(_P63, math.inf),
                math.nextafter(-_P63, 0), math.nextafter(-_P63, -math.inf), 2.0 ** 53, 2.0 ** 31, 3037000499.0)
BIGINT_EDGES = (I64_MIN, I64_MAX, I64_MIN + 1, I64_MAX - 1, -1, 0, 1, 2 ** 31, -2 ** 31, 2 ** 53, 2 ** 53 + 1, 3037000499, 3037000500,
                -3037000500, 2 ** 62, 2)
INT_EDGES = {abi.INT8: (-128, 127, -1, 0, 1, -127), abi.INT16: (-32768, 32767, -1, 0, 1, 255), abi.INT32: (-2 ** 31, 2 ** 31 - 1, -1, 0, 1, 65536),
             abi.INT64: BIGINT_EDGES}
INT_RANGE = {abi.INT8: 128, abi.INT16: 32768, abi.INT32: 2 ** 31, abi.INT64: 2 ** 63}

# every (op, operand vtype) pair the evaluator accepts
OP_PAIRS = {(op, vt) for op in (abi.EX_ADD, abi.EX_SUB, abi.EX_MUL, abi.EX_DIV, abi.EX_MOD, abi.EX_NEG) for vt in (B, D)}
OP_PAIRS |= {(op, vt) for op in (abi.EX_EQ, abi.EX_NE, abi.EX_LT, abi.EX_LE, abi.EX_GT, abi.EX_GE, abi.EX_IS_NULL, abi.EX_IS_NOT_NULL, abi.EX_MOV)
             for vt in (B, D, BOOL)}
OP_PAIRS |= {(abi.EX_AND, BOOL), (abi.EX_OR, BOOL), (abi.EX_NOT, BOOL), (abi.EX_BETWEEN, B), (abi.EX_BETWEEN, D), (abi.EX_IN, B), (abi.EX_IN, D),
             (abi.EX_CAST_BIGINT_TO_DOUBLE, B), (abi.EX_CAST_DOUBLE_TO_BIGINT, D)}


def _result_pairs(vt):
    """(op, operand vtype) pairs whose result has type vt"""
    out = []
    for op, ovt in sorted(OP_PAIRS):
        if op in (abi.EX_CAST_BIGINT_TO_DOUBLE,):
            res = D
        elif op == abi.EX_CAST_DOUBLE_TO_BIGINT:
            res = B
        elif op in (abi.EX_ADD, abi.EX_SUB, abi.EX_MUL, abi.EX_DIV, abi.EX_MOD, abi.EX_NEG, abi.EX_MOV):
            res = ovt
        else:
            res = BOOL
        if res == vt:
            out.append((op, ovt))
    return out


_ARITY = {abi.EX_NEG: 1, abi.EX_NOT: 1, abi.EX_IS_NULL: 1, abi.EX_IS_NOT_NULL: 1, abi.EX_MOV: 1, abi.EX_CAST_BIGINT_TO_DOUBLE: 1,
          abi.EX_CAST_DOUBLE_TO_BIGINT: 1, abi.EX_IN: 1, abi.EX_BETWEEN: 3}


# ---- programs ---------------------------------------------------------------------------------------------------------------
class ProgramGen:
    """Typed random trees of depth <= 5.  Prefers (op, vtype) pairs not yet generated, so a few dozen programs use them all."""

    def __init__(self, rng, channels_by_vtype, seen=None, bigint_channels=()):
        self.rng, self.channels, self.bigint_channels = rng, channels_by_vtype, list(bigint_channels)
        self.seen = seen if seen is not None else {}

    def const(self, vt):
        r = self.rng
        if r.random() < 0.07:
            return ops.Null(vt)
        if vt == BOOL:
            return ops.Const(bool(r.integers(0, 2)), BOOL)
        if vt == D:
            return ops.Const(float(r.choice(DOUBLE_EDGES)) if r.random() < 0.4 else float(r.integers(-20, 21)) / 4, D)
        return ops.Const(int(r.choice(BIGINT_EDGES)) if r.random() < 0.3 else int(r.integers(-10, 11)), B)

    def leaf(self, vt):
        if self.rng.random() < 0.75:
            return ops.Col(int(self.rng.choice(self.channels[vt])), vt)
        return self.const(vt)

    def expr(self, vt, depth):
        r = self.rng
        if depth <= 0 or r.random() < 0.2:
            return self.leaf(vt)
        pairs = _result_pairs(vt)
        w = np.array([40.0 if p not in self.seen else 1.0 for p in pairs])
        op, ovt = pairs[int(r.choice(len(pairs), p=w / w.sum()))]
        self.seen[(op, ovt)] = self.seen.get((op, ovt), 0) + 1
        if op == abi.EX_IN:
            vals = [self.const(ovt) for _ in range(int(r.integers(1, 5)))]
            vals = [v.value for v in vals if isinstance(v, ops.Const)] or [0]
            return ops.Call(op, self.expr(ovt, depth - 1), in_list=vals)
        args = [self.expr(ovt, depth - 1) for _ in range(_ARITY.get(op, 2))]
        if op in (abi.EX_DIV, abi.EX_MOD) and ovt == B and r.random() < 0.7:
            # x / -1 and x % -1 where x is a BIGINT column, which holds INT64_MIN
            args[1] = ops.Const(int(r.choice([-1, -1, -1, 2])), B)
            if self.bigint_channels:
                args[0] = ops.Col(int(r.choice(self.bigint_channels)), B)
        return ops.Call(op, *args)

    def program(self, max_depth=5):
        """(filter, projections) that PageProcessorProgram compiles within 8 temporaries and 64 instructions"""
        while True:
            filt = self.expr(BOOL, int(self.rng.integers(2, max_depth + 1)))
            projs = [self.expr(int(self.rng.choice([B, D, BOOL], p=[0.4, 0.4, 0.2])), int(self.rng.integers(1, max_depth + 1)))
                     for _ in range(int(self.rng.integers(1, 4)))]
            try:
                p = ops.PageProcessorProgram(filt, projs)
            except ValueError:
                continue
            if len(p.insns) <= 64:
                return filt, projs


_OPNAME = {abi.EX_ADD: "+", abi.EX_SUB: "-", abi.EX_MUL: "*", abi.EX_DIV: "/", abi.EX_MOD: "%", abi.EX_EQ: "=", abi.EX_NE: "<>",
           abi.EX_LT: "<", abi.EX_LE: "<=", abi.EX_GT: ">", abi.EX_GE: ">=", abi.EX_AND: "AND", abi.EX_OR: "OR"}
_TNAME = {B: "bigint", D: "double", BOOL: "boolean"}


def show(e):
    """SQL-like text of an expression tree"""
    if isinstance(e, ops.Col):
        return f"c{e.channel}"
    if isinstance(e, ops.Const):
        return repr(e.value) if e.vtype != D else f"DOUBLE '{e.value!r}'"
    if isinstance(e, ops.Null):
        return f"CAST(NULL AS {_TNAME[e.vtype]})"
    a = [show(x) for x in e.args]
    if e.op in _OPNAME:
        return f"({a[0]} {_OPNAME[e.op]} {a[1]})"
    return {abi.EX_NEG: lambda: f"(-{a[0]})", abi.EX_NOT: lambda: f"(NOT {a[0]})", abi.EX_IS_NULL: lambda: f"({a[0]} IS NULL)",
            abi.EX_IS_NOT_NULL: lambda: f"({a[0]} IS NOT NULL)", abi.EX_MOV: lambda: a[0],
            abi.EX_BETWEEN: lambda: f"({a[0]} BETWEEN {a[1]} AND {a[2]})", abi.EX_IN: lambda: f"({a[0]} IN {tuple(e.in_list)!r})",
            abi.EX_CAST_BIGINT_TO_DOUBLE: lambda: f"CAST({a[0]} AS double)", abi.EX_CAST_DOUBLE_TO_BIGINT: lambda: f"CAST({a[0]} AS bigint)"}[e.op]()


# ---- columns and pages ------------------------------------------------------------------------------------------------------
class Column:
    """One channel: `values` (numpy, POOL entries or fewer) and `nulls` over the pool, and the block encoding of the pages"""

    def __init__(self, type_, values, nulls, encoding="flat"):
        self.type, self.encoding = type_, encoding
        self.values = np.ascontiguousarray(np.asarray(values, dtype=_NP[type_] if type_ != abi.UTF8 else object))
        self.nulls = np.asarray(nulls, dtype=bool)
        if encoding == "rle":               # one value for every row
            self.values[:] = self.values[0]
            self.nulls[:] = self.nulls[0]

    def pylist(self):
        if self.type == abi.UTF8:
            return [None if n else v for v, n in zip(self.values.tolist(), self.nulls.tolist())]
        vals = self.values.tolist()
        return [None if n else v for v, n in zip(vals, self.nulls.tolist())]

    def block(self, idx):
        nulls = self.nulls if self.nulls.any() else None
        if self.type == abi.UTF8:
            return Block.varchar([None if self.nulls[i] else self.values[i] for i in idx.tolist()])
        if self.encoding == "rle":
            return RunLengthEncodedBlock(_BLOCK[self.type](self.values[:1], self.nulls[:1] if nulls is not None else None), len(idx))
        if self.encoding == "dict":
            return DictionaryBlock(_BLOCK[self.type](self.values, nulls), idx)
        return _BLOCK[self.type](np.ascontiguousarray(self.values[idx]), None if nulls is None else self.nulls[idx])


def random_column(rng, type_, k, null_mode, encoding):
    if type_ == "boolean":
        vals = rng.integers(0, 2, k)
    elif type_ == abi.FLOAT64:
        vals = np.where(rng.random(k) < 0.5, rng.choice(np.array(DOUBLE_EDGES), k), np.round(rng.normal(0, 50, k), 2))
    else:
        lim = INT_RANGE[type_]
        tame = rng.integers(-100, 101, k)
        wide = rng.integers(-lim, lim, k, dtype=np.int64) if type_ != abi.INT64 else rng.integers(I64_MIN, I64_MAX, k, dtype=np.int64, endpoint=True)
        vals = np.where(rng.random(k) < 0.5, rng.choice(np.array(INT_EDGES[type_], dtype=np.int64), k), np.where(rng.random(k) < 0.8, tame, wide))
    nulls = {"none": np.zeros(k, bool), "some": rng.random(k) < 0.3, "all": np.ones(k, bool)}[null_mode]
    return Column(type_, vals, nulls, encoding)


class Case:
    """A program over columns, and the pool rows of each page (`pages`: list of index arrays into the pool)"""

    def __init__(self, name, columns, filt, projs, pages, seed=None):
        self.name, self.filt, self.projs, self.seed = name, filt, list(projs), seed
        k = len(columns[0].values)
        rng = np.random.default_rng(12345 if seed is None else seed + 1)
        words = np.array(["", "a", "bb", "ccc", "x" * 20, "été"], dtype=object)
        columns = list(columns)
        self.fixed = list(range(min(3, len(columns))))                   # pass-through channels of the chunked form
        self.key = len(columns)
        columns.append(Column(abi.INT8, rng.integers(-3, 5, k), rng.random(k) < 0.1))      # <= 8 values and NULL: the small aggregation path
        self.varchar = len(columns)                                      # last: only the pages of the VARCHAR form carry it
        columns.append(Column(abi.UTF8, words[rng.integers(0, len(words), k)], rng.random(k) < 0.2))
        self.columns, self.pages = columns, [np.asarray(p, dtype=np.int64) for p in pages]
        cols = [c.pylist() for c in columns]
        self.rows = list(zip(*cols))
        self._memo = {}

    def describe(self):
        s = f"case {self.name}" + (f" (seed {self.seed})" if self.seed is not None else "") + "\n"
        s += "  channels: " + ", ".join(f"c{i}:{_type_name(c.type)}/{c.encoding}/{_null_mode(c)}" for i, c in enumerate(self.columns)) + "\n"
        s += f"  filter: {show(self.filt) if self.filt is not None else '-'}\n"
        for i, p in enumerate(self.projs):
            s += f"  projection {i}: {show(p)}\n"
        s += "  page sizes: " + ", ".join(str(len(p)) for p in self.pages)
        return s

    def evaluate(self, expr):
        """per pool row: (values, error codes) of one expression; memoised"""
        key = id(expr)
        if key not in self._memo:
            vals, errs = [], []
            for r in self.rows:
                v, e = ref.try_evaluate(expr, r)
                vals.append(v)
                errs.append(e)
            self._memo[key] = (expr, vals, errs)      # holding expr keeps its id from being reused
        return self._memo[key][1:]

    def page(self, idx, varchar=False):
        cols = self.columns if varchar else self.columns[:self.varchar]
        return Page(*[c.block(idx) for c in cols], position_count=len(idx))


def _type_name(t):
    return {abi.INT8: "tinyint", abi.INT16: "smallint", abi.INT32: "integer", abi.INT64: "bigint", abi.FLOAT64: "double", "boolean": "boolean",
            abi.UTF8: "varchar"}[t]


def _null_mode(c):
    return "all-null" if c.nulls.all() else ("nullable" if c.nulls.any() else "non-null")


def random_case(seed, seen=None, sizes=None):
    rng = np.random.default_rng(seed)
    k = POOL
    columns = []
    for t in RANDOM_TYPES:
        null_mode = rng.choice(["none", "some", "all"], p=[0.45, 0.45, 0.1])
        enc = rng.choice(["flat", "dict", "rle"], p=[0.6, 0.3, 0.1])
        columns.append(random_column(rng, t, k, null_mode, enc))
    by_vt = {B: [], D: [], BOOL: []}
    for c, t in enumerate(RANDOM_TYPES):
        by_vt[VTYPE_OF[t]].append(c)
    gen = ProgramGen(rng, by_vt, seen, [c for c, t in enumerate(RANDOM_TYPES) if t == abi.INT64])
    filt, projs = gen.program()
    mode = ["some", "some", "none", "all"][seed % 4]
    if mode == "all":
        filt = ops.Call(abi.EX_OR, ops.Const(True, BOOL), filt)
    elif mode == "none":
        filt = ops.Call(abi.EX_AND, ops.Const(False, BOOL), filt)
    sizes = sizes or [SIZES[seed % len(SIZES)], SIZES[(seed + 3) % len(SIZES)]]
    pages = [rng.integers(0, k, n) for n in sizes]
    return Case(f"random-{seed}-{mode}", columns, filt, projs, pages, seed=seed)


def random_cases(n=16):
    seen = {}
    cases = []
    for s in range(n):
        sizes = [BIG_PAGE, 1025] if s == 5 else None
        cases.append(random_case(1000 + s, seen, sizes))
    return cases, seen


def bits(x):
    return struct.unpack("<q", struct.pack("<d", x))[0]
