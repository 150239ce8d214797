"""Generic-key joins (several key channels, or one VARCHAR / long DECIMAL / REAL channel: the lookups keyed by the row hash and verified
against the key columns) on every probe, outer and semi-join path, against the plain-Python reference of join_reference.py.

Every output row is identified by an INTEGER row-id channel on each side; the id arrays are compared in order, and the payload
channels (a nullable BIGINT, a VARCHAR with NULLs, a long DECIMAL, a DOUBLE compared by its bits) are functions of the ids.
The case generators are seeded and take a size, so test_join_reference.py runs them small, without a device, against the oracle."""
import functools

import numpy as np
import pytest

import join_reference as jr
from helpers import _M, _P1, _P2, _rotl, _rotr
from trino_b200 import abi
from trino_b200 import operators as ops
from trino_b200.page import Block, DictionaryBlock, Page, RunLengthEncodedBlock

pytestmark = pytest.mark.gpu

JOIN_TYPES = {"inner": abi.JOIN_INNER, "probe_outer": abi.JOIN_PROBE_OUTER, "lookup_outer": abi.JOIN_LOOKUP_OUTER, "full_outer": abi.JOIN_FULL_OUTER}
TRACKING = (abi.JOIN_LOOKUP_OUTER, abi.JOIN_FULL_OUTER)
SHAPES = {
    "varchar": ["varchar"], "real": ["real"], "int128": ["int128"],
    "double": ["double"],                                   # one DOUBLE channel: keyed by value, not generic; same reference
    "bigint+integer": ["bigint", "integer"], "bigint+varchar+double": ["bigint", "varchar", "double"], "varchar+varchar": ["varchar", "varchar"],
    "int128+real": ["int128", "real"],
    "tuple8": ["bigint", "smallint", "tinyint", "boolean", "varchar", "integer", "real", "double"],     # MAX_KEY_COLS channels
}
FORMS = ["unique", "dups3", "heavy", "nulls", "null_last", "all_null", "one_row", "empty", "paged", "encoded"]
PROBE_SIZES = (1, 255, 256, 257, 1023, 1024, 1025, 4097)
_RADIX_CAP = {"boolean": 2, "tinyint": 200, "smallint": 30000}
_TYPE = {"bigint": abi.INT64, "integer": abi.INT32, "smallint": abi.INT16, "tinyint": abi.INT8, "boolean": abi.INT8, "double": abi.FLOAT64,
         "real": abi.FLOAT32, "varchar": abi.UTF8, "int128": abi.INT128}
_NAN64 = np.array([0x7FF8000000000000, 0xFFF8000000000001, 0x7FF0000000000001, 0xFFFFFFFFFFFFFFFF], dtype=np.uint64)
_NAN32 = np.array([0x7FC00000, 0xFFC00001, 0x7F800001, 0xFFFFFFFF], dtype=np.uint32)


# ---------------------------------------------------------------------------------------------------- case generators
def _string_of(d):
    if d == 0:
        return ""
    return "v%d" % d + ("ü€" if d % 5 == 0 else "") + ("x" * 40 if d % 7 == 0 else "")   # prefixes of one another, multi-byte, long


def _int128_of(d):
    if d % 3 == 0:
        return (7 << 64) + d                # one high word, low words differ
    if d % 2 == 0:
        return (d << 64) + 5                # one low word, high words differ
    return -(d << 70) - d


def _digits(kinds, count):
    """`count` distinct key tuples as one digit per channel (mixed radix): single channels repeat across tuples, tuples never do"""
    free = sum(1 for k in kinds if k not in _RADIX_CAP)
    assert free, "every key shape has a channel with a large domain"
    radix = int(np.ceil(count ** (1.0 / free))) + 1
    out, t = [], np.arange(count, dtype=np.int64)
    for k in kinds:
        r = min(radix, _RADIX_CAP.get(k, radix))
        out.append(t % r)
        t = t // r
    assert not t.any()
    return out


def _key_block(kind, d, rng, null_frac, nan_frac):
    """the channel's value for every digit of d, with NULLs, NaNs of several encodings and -0.0 sprinkled in"""
    n = len(d)
    nulls = rng.random(n) < null_frac if null_frac else None
    if kind == "varchar":
        return Block.varchar([None if nulls is not None and nulls[i] else _string_of(x) for i, x in enumerate(d.tolist())])
    if kind == "int128":
        return Block.int128([_int128_of(x) for x in d.tolist()], nulls)
    if kind == "double":
        bits = (d * 0.5 - 2.0).view(np.uint64).copy()
        bits[(bits == 0) & (rng.random(n) < 0.5)] = 1 << 63                  # -0.0 joins +0.0
        if nan_frac:
            at = rng.random(n) < nan_frac
            bits[at] = rng.choice(_NAN64, int(at.sum()))
        return Block.double(bits.view(np.float64), nulls)
    if kind == "real":
        bits = (d * 0.25 - 1.0).astype(np.float32).view(np.uint32).copy()
        bits[(bits == 0) & (rng.random(n) < 0.5)] = 1 << 31
        if nan_frac:
            at = rng.random(n) < nan_frac
            bits[at] = rng.choice(_NAN32, int(at.sum()))
        return Block.real(bits.view(np.float32), nulls)
    if kind == "bigint":
        return Block.bigint((d - 3) * 10_000_000_019 + 1, nulls)
    if kind == "integer":
        return Block.integer(((d - 5) * 3).astype(np.int32), nulls)
    if kind == "smallint":
        return Block.smallint((d - 100).astype(np.int16), nulls)
    if kind == "tinyint":
        return Block.tinyint((d - 100).astype(np.int8), nulls)
    return Block.boolean(d.astype(bool), nulls)


def _key_blocks(kinds, digits, tuples, rng, null_frac=0.0, nan_frac=0.0, null_last_only=False):
    blocks = []
    for c, kind in enumerate(kinds):
        nf = null_frac if not null_last_only or c == len(kinds) - 1 else 0.0
        blocks.append(_key_block(kind, digits[c][tuples], rng, nf, 0.0 if null_last_only else nan_frac))
    return blocks


def build_payload(ids):
    """the build side's payload channels as functions of the row id: nullable BIGINT, VARCHAR with NULLs and "", long DECIMAL, DOUBLE"""
    ids = np.asarray(ids, dtype=np.int64)
    dbl = (ids * 0.125).view(np.uint64).copy()
    dbl[ids % 17 == 0] = 0xFFF8000000000123
    dbl[ids % 19 == 1] = 1 << 63
    return [Block.bigint(ids * 7 - 3, ids % 9 == 0), Block.varchar([None if i % 11 == 0 else "" if i % 13 == 0 else "b%d" % i for i in ids.tolist()]),
            Block.int128([(i - 50) * (1 << 70) + i for i in ids.tolist()]), Block.double(dbl.view(np.float64))]


def probe_payload(ids):
    ids = np.asarray(ids, dtype=np.int64)
    return [Block.varchar([None if i % 7 == 0 else "p%d" % i for i in ids.tolist()]), Block.double(ids * 0.5, ids % 5 == 0)]


def build_page(key_blocks, first_id):
    n = key_blocks[0].position_count
    ids = np.arange(first_id, first_id + n)
    return Page(*key_blocks, Block.integer(ids.astype(np.int32)), *build_payload(ids), position_count=n)


def probe_page(key_blocks, first_id):
    n = key_blocks[0].position_count
    ids = np.arange(first_id, first_id + n)
    return Page(Block.integer(ids.astype(np.int32)), *key_blocks, *probe_payload(ids), position_count=n)


class Case:
    """build pages [keys..., id, 4 payloads] and probe pages [id, keys..., 2 payloads] of one key shape"""

    def __init__(self, shape, form, seed, kinds, build_pages, probe_pages):
        self.shape, self.form, self.seed, self.kinds = shape, form, seed, kinds
        nk = len(kinds)
        self.build_pages, self.probe_pages = build_pages, probe_pages
        self.build_keys, self.probe_keys = list(range(nk)), list(range(1, nk + 1))
        self.build_out, self.probe_out = list(range(nk, nk + 5)), [0, nk + 1, nk + 2]
        self.probe_out_types = [abi.INT32, abi.UTF8, abi.FLOAT64]

    @functools.cached_property
    def reference(self):
        return jr.JoinReference(self.build_pages, self.build_keys)

    @functools.cached_property
    def positions(self):
        return [self.reference.positions(p, self.probe_keys) for p in self.probe_pages]

    def say(self, join_type=None, single=None):
        name = {v: k for k, v in JOIN_TYPES.items()}.get(join_type)
        return f"shape={self.shape} form={self.form} seed={self.seed} join_type={name} single_match={single}"


def _split(blocks_of, tuples, sizes):
    """pages over consecutive slices of `tuples`; the last size takes what is left"""
    pages, at = [], 0
    for i, m in enumerate(sizes):
        m = len(tuples) - at if i == len(sizes) - 1 else m
        pages.append((blocks_of(tuples[at:at + m]), at))
        at += m
    return pages


def _encode(block, rng):
    """the same values behind a DictionaryBlock with a shuffled dictionary"""
    n = block.position_count
    perm = rng.permutation(n)
    inverse = np.empty(n, dtype=np.int32)
    inverse[perm] = np.arange(n, dtype=np.int32)
    return DictionaryBlock(block.get_positions(perm), inverse)


def make_case(shape, form, seed=1, scale=1.0, probe_sizes=PROBE_SIZES, build_rows=None):
    """One seeded case.  `scale` shrinks the row counts (the reference test runs the same generators small)."""
    kinds = SHAPES[shape]
    rng = np.random.default_rng([seed, sorted(SHAPES).index(shape), FORMS.index(form)])
    rows = build_rows or max(8, int((5074 if form == "paged" else 3000) * scale))      # paged: pages of 1, 64, 5000 and 9 rows
    heavy = max(8, int(10_000 * scale)) if form == "heavy" else 0
    distinct = rows if form in ("unique", "one_row") else max(2, rows // 3)
    if form == "one_row":
        rows = distinct = 1
    extra = max(2, distinct // 2)                                   # tuples no build row has: about a third of the probe misses
    digits = _digits(kinds, distinct + extra)
    if form == "unique" or form == "one_row":
        tuples = rng.permutation(distinct)
    else:
        tuples = rng.integers(0, distinct, rows)
    if heavy:
        tuples = np.concatenate([tuples, np.full(heavy, 1)])
        tuples = tuples[rng.permutation(len(tuples))]
    null_frac = 0.04 if form == "nulls" else 0.05 if form == "null_last" else 0.0
    nan_frac = 0.02 if form == "nulls" else 0.0
    blocks_of = lambda t: _key_blocks(kinds, digits, t, rng, null_frac, nan_frac, form == "null_last")
    if form == "empty":
        builds = [build_page(blocks_of(tuples[:0]), 0)]
    elif form == "paged":
        builds = [build_page(b, at) for b, at in _split(blocks_of, tuples, (1, 64, max(1, len(tuples) - 74), 9))]
        builds = [p for p in builds if p.position_count]
    else:
        builds = [build_page(blocks_of(tuples), 0)]
    if form == "all_null":
        first = builds[0].blocks[0]
        builds[0].blocks[0] = Block(first.type, first.values, np.ones(first.position_count, dtype=bool), first.offsets)
    if form == "encoded":
        builds[0].blocks[:len(kinds)] = [_encode(b, rng) for b in builds[0].blocks[:len(kinds)]]
    # probe pages: a third of the rows miss; then one page where every row matches and one where none does
    probes, first_id = [], 0
    built = np.unique(tuples) if form != "empty" else np.arange(0)
    for m in [max(1, int(s * scale)) if s > 1 else 1 for s in probe_sizes] + ["all", "none"]:
        if m == "all":
            m = max(4, int(1000 * scale))
            t = rng.choice(built[built != 1] if heavy else built, m) if len(built) else rng.integers(distinct, distinct + extra, m)
            keys = _key_blocks(kinds, digits, t, rng)
        elif m == "none":
            m = max(4, int(1000 * scale))
            keys = _key_blocks(kinds, digits, rng.integers(distinct, distinct + extra, m), rng)
        else:
            t = np.where(rng.random(m) < 0.33, rng.integers(distinct, distinct + extra, m), rng.integers(0, distinct, m))
            if heavy:
                t[t == 1] = 2
                t[0] = 1                                            # the 10 000-row key is probed once a page
            keys = _key_blocks(kinds, digits, t, rng, 0.03, 0.02)
        if form == "encoded" and m > 1:
            keys = [_encode(b, rng) if c % 2 == 0 else b for c, b in enumerate(keys)]
        probes.append(probe_page(keys, first_id))
        first_id += m
    if form == "encoded":           # a run-length encoded key tuple that is built, and a dictionary on the other channels
        t = np.full(300, tuples[0])
        keys = [RunLengthEncodedBlock(b.get_positions([0]), 300) for b in _key_blocks(kinds, digits, t, rng)]
        probes.append(probe_page(keys, first_id))
    return Case(shape, form, seed, kinds, builds, probes)


@functools.lru_cache(maxsize=None)
def cached_case(shape, form):
    return make_case(shape, form)


# xxHash64 (seed 0) of whole 8-byte little-endian words, for inputs shorter than 32 bytes, and its inverse in the last word: the reference
# hashes a long DECIMAL as xxh64(high word) ^ xxh64(low word) and a VARCHAR as xxh64(bytes), and a row as 31 * h + hash(channel), so two
# key tuples that differ in every channel can be given one row hash by solving for the last word of the last channel
_P3, _P4, _P5 = 0x165667B19E3779F9, 0x85EBCA77C2B2AE63, 0x27D4EB2F165667C5


def _xxh64_words(words):
    h = (_P5 + 8 * len(words)) & _M
    for v in words:
        h ^= (_rotl((v * _P2) & _M, 31) * _P1) & _M
        h = (_rotl(h, 27) * _P1 + _P4) & _M
    h ^= h >> 33; h = (h * _P2) & _M; h ^= h >> 29; h = (h * _P3) & _M; h ^= h >> 32
    return h


def _last_word_for(words, target):
    """w such that _xxh64_words(words + [w]) == target"""
    inv = lambda x: pow(x, -1, 1 << 64)
    h = target
    h ^= h >> 32; h = (h * inv(_P3)) & _M; h ^= h >> 29; h ^= h >> 58; h = (h * inv(_P2)) & _M; h ^= h >> 33
    h = _rotr(((h - _P4) * inv(_P1)) & _M, 27)
    before = (_P5 + 8 * (len(words) + 1)) & _M
    for v in words:
        before ^= (_rotl((v * _P2) & _M, 31) * _P1) & _M
        before = (_rotl(before, 27) * _P1 + _P4) & _M
    return (_rotr(((h ^ before) * inv(_P1)) & _M, 31) * inv(_P2)) & _M


def _hash_int128(x):
    return _xxh64_words([(x >> 64) & _M]) ^ _xxh64_words([x & _M])


def colliding_int128_tuples():
    """(A1, A2) and (B1, B2): the LOW words agree channel by channel, every high word differs, and the row hashes are equal"""
    a1, a2, b1, low = (3 << 64) + 9, (4 << 64) + 11, (5 << 64) + 9, 11
    want = (31 * _hash_int128(a1) + _hash_int128(a2) - 31 * _hash_int128(b1)) & _M
    high = _last_word_for([], want ^ _xxh64_words([low]))
    return (a1, a2), (b1, ((high - (1 << 64) if high >> 63 else high) << 64) + low)


def colliding_varchar_tuples():
    """(A1, A2) and (B1, B2): each A string is a proper prefix of its B string, and the row hashes are equal"""
    words = lambda b: [int.from_bytes(b[i:i + 8], "little") for i in range(0, len(b), 8)]
    a1, a2, b1 = b"abcdefgh", b"ijklmnop", b"abcdefghABCDEFGH"
    want = (31 * _xxh64_words(words(a1)) + _xxh64_words(words(a2)) - 31 * _xxh64_words(words(b1))) & _M
    return (a1, a2), (b1, a2 + _last_word_for(words(a2), want).to_bytes(8, "little"))


def edge_tables():
    """(name, kinds, build key rows, probe key rows): small explicit tables of the values hash tables and comparisons get wrong"""
    nan, inf = float("nan"), float("inf")
    long_a, long_b = "y" * 300 + "a", "y" * 300 + "b"
    strings = ["", None, "a", "ab", "abc", "abd", "\u00e9", "e\u0301", "\u20ac", "\u20ac\u20ac", long_a, long_b, "a", "", None, "ab\x00", "ab"]
    reals = np.array([0x3F800000, 0x3F800001, 0x3F7FFFFF, 0x00000001, 0x80000000, 0x00000000, 0x7FC00000, 0xFFC00001, 0x7F800000, 0xFF800000], dtype=np.uint32).view(np.float32)
    dbl = np.array([0x7FF8000000000000, 0xFFF8000000000000, 0x7FF0000000000001, 0x8000000000000000, 0, 0x3FF0000000000000, 0x3FF0000000000001, 0x7FF0000000000000],
                   dtype=np.uint64).view(np.float64)
    top = 1 << 127
    ints = [0, 1, 1 << 64, (1 << 64) + 1, 2 << 64, -1, -(1 << 64), -top, top - 1, -top + 1, top - 2, 5, (5 << 64) + 5, 5 << 64, None, 1]
    tables = [
        ("strings", ["varchar"], [(s,) for s in strings], [(s,) for s in strings + ["abcd", "b", "\u00e9\u00e9", "y" * 300, "y" * 301]]),
        ("tuple_boundaries", ["varchar", "varchar"], [("ab", "c"), ("a", "bc"), ("", "abc"), ("abc", ""), ("x", "y"), ("y", "x"), ("ab", None), (None, "c"), ("ab", "c")],
         [("a", "bc"), ("ab", "c"), ("abc", ""), ("", "abc"), ("y", "x"), ("x", "y"), ("x", "x"), ("ab", None), (None, None), ("a", "b"), ("", "")]),
        ("swapped_integers", ["bigint", "bigint"], [(1, 2), (2, 1), (1, 1), (0, 3), (3, 0), (1, 2)], [(2, 1), (1, 2), (2, 2), (3, 0), (0, 3), (0, 0), (1, None), (None, 2)]),
        ("real_bits", ["real"], [(float(v),) for v in reals], [(float(v),) for v in reals] + [(1.0000001,), (-0.0,), (None,)]),
        ("double_bits", ["double"], [(v,) for v in dbl], [(v,) for v in dbl] + [(-nan,), (-0.0,), (None,), (inf,), (-inf,)]),
        ("nan_and_zero_in_tuples", ["bigint", "double", "real"],
         [(1, 0.0, 0.0), (1, -0.0, 1.0), (1, nan, 1.0), (2, 1.0, nan), (2, 1.0, -0.0), (3, 0.0, None), (1, 0.0, -0.0), (4, dbl[1], 2.0), (5, 2.0, float(reals[7]))],
         [(1, -0.0, -0.0), (1, 0.0, 1.0), (1, nan, 1.0), (2, 1.0, nan), (2, 1.0, 0.0), (3, 0.0, None), (3, 0.0, 0.0), (4, nan, 2.0), (5, 2.0, nan), (4, dbl[0], 2.0)]),
        ("int128_words", ["int128"], [(v,) for v in ints], [(v,) for v in ints + [3 << 64, -2, (1 << 64) - 1, -top + 2]]),
        ("int128_in_tuples", ["int128", "real"], [(1 << 64, 1.0), (1, 1.0), ((1 << 64) + 1, 1.0), (-top, -0.0), (top - 1, float(reals[1])), (1, None)],
         [(1, 1.0), (1 << 64, 1.0), ((1 << 64) + 1, 2.0), (-top, 0.0), (top - 1, 1.0), (top - 1, float(reals[1])), (1, None), (None, 1.0)]),
    ]
    # two tuples on one row hash that only the compared high words / string lengths keep apart (the verify kernels' whole purpose)
    for name, kind, (a, b) in (("int128_colliding_tuples", "int128", colliding_int128_tuples()), ("varchar_colliding_tuples", "varchar", colliding_varchar_tuples())):
        tables.append((name, [kind, kind], [a, b, a], [b, a, (a[0], b[1]), (b[0], a[1])]))
    return tables


_MAKERS = {"varchar": Block.varchar, "int128": Block.int128, "double": Block.double, "real": Block.real, "bigint": Block.bigint, "integer": Block.integer,
           "smallint": Block.smallint, "tinyint": Block.tinyint, "boolean": Block.boolean}


def blocks_from_rows(kinds, rows):
    out = []
    for c, kind in enumerate(kinds):
        col = [r[c] for r in rows]
        if kind in ("double", "real"):        # keep NaN payloads: go through the raw values, not through a Python list of floats
            arr = np.array([0.0 if v is None else v for v in col], dtype=np.float64 if kind == "double" else np.float32)
            out.append(_MAKERS[kind](arr, [v is None for v in col] if any(v is None for v in col) else None))
        else:
            out.append(_MAKERS[kind](col))
    return out


def edge_case(name):
    for table, kinds, build_rows, probe_rows in edge_tables():
        if table == name:
            return Case("edge:" + name, "explicit", 0, kinds, [build_page(blocks_from_rows(kinds, build_rows), 0)], [probe_page(blocks_from_rows(kinds, probe_rows), 0)])
    raise KeyError(name)


EDGE_NAMES = ["strings", "tuple_boundaries", "swapped_integers", "real_bits", "double_bits", "nan_and_zero_in_tuples", "int128_words", "int128_in_tuples", "int128_colliding_tuples",
              "varchar_colliding_tuples"]


def collision_case(seed=5, ordinary=5000):
    """Three (BIGINT, BIGINT) tuples on one attempt-0 row hash, built 1, 2 and 5 times at scattered positions among ordinary rows, and a
    fourth colliding tuple that is never built: the rebuild loop must move two of the tuples to their next hash function and keep
    every chain pure."""
    from helpers import colliding_bigint_pairs
    rng = np.random.default_rng(seed)
    t1 = (11, 22)
    others = [(a, colliding_bigint_pairs(11, 22, a)) for a in (33, 44, 55)]
    built = [t1] * 1 + [others[0]] * 2 + [others[1]] * 5
    a = rng.integers(100, 1000, ordinary).astype(np.int64)         # the crafted tuples all start below 100
    b = rng.integers(100, 1000, ordinary).astype(np.int64)
    at = np.sort(rng.choice(ordinary, len(built), replace=False))
    order = rng.permutation(len(built))
    for where, which in zip(at, order):
        a[where], b[where] = built[which]
    pa = rng.integers(0, 1200, 4000).astype(np.int64)
    pb = rng.integers(0, 1000, 4000).astype(np.int64)
    for i, t in enumerate([others[2], t1, others[1], others[0], others[2], others[1], t1, (11, others[0][1]), (33, 22)]):
        pa[i * 37], pb[i * 37] = t
    case = Case("bigint+bigint", "three_tuples_on_one_row_hash", seed, ["bigint", "bigint"], [build_page([Block.bigint(a), Block.bigint(b)], 0)],
                [probe_page([Block.bigint(pa), Block.bigint(pb)], 0)])
    case.colliding = [t1] + others
    return case


# ---------------------------------------------------------------------------------------------------- running and checking
def _ids(block):
    """INTEGER id channel -> int64 array, -1 where NULL"""
    v = np.asarray(block.values, dtype=np.int64).copy()
    if block.nulls is not None:
        v[block.nulls] = -1
    return v


def _strings(block):
    data, offs = block.values.tobytes(), block.offsets.tolist()
    nulls = block.nulls.tolist() if block.nulls is not None else [False] * block.position_count
    return [None if z else data[offs[i]:offs[i + 1]] for i, z in enumerate(nulls)]


def assert_block_equal(got, want, present, what):
    """`want` holds the rows where `present`; elsewhere `got` must be NULL"""
    n = got.position_count
    assert got.type == want.type and n == len(present), what
    got_null = got.nulls if got.nulls is not None else np.zeros(n, dtype=bool)
    want_null = np.ones(n, dtype=bool)
    want_null[present] = want.nulls if want.nulls is not None else False
    assert np.array_equal(got_null, want_null), what + ": NULLs differ"
    if got.type == abi.UTF8:
        g = _strings(got)
        assert [g[i] for i in np.nonzero(present)[0].tolist()] == _strings(want), what
        return
    live = ~want_null
    g, w = np.asarray(got.values)[live], np.asarray(want.values)[live[present]]
    if g.dtype.kind == "f":
        g, w = g.view(np.uint64 if g.dtype.itemsize == 8 else np.uint32), w.view(np.uint64 if w.dtype.itemsize == 8 else np.uint32)
    assert np.array_equal(g, w), what


def check_output(out, want_probe, want_build, what):
    """probe ids and build ids in order, then every payload channel through the ids"""
    n = len(want_probe)
    if out is None:
        assert n == 0, f"{what}: no page, expected {n} rows"
        return np.zeros(0, dtype=np.int64)
    assert out.position_count == n, f"{what}: {out.position_count} rows, expected {n}"
    if n == 0:
        return np.zeros(0, dtype=np.int64)
    got_probe, got_build = _ids(out.blocks[0]), _ids(out.blocks[3])
    assert np.array_equal(got_probe, want_probe), f"{what}: probe rows differ, first at output row {np.argmax(got_probe != want_probe)}"
    assert np.array_equal(got_build, want_build), f"{what}: build rows differ, first at output row {np.argmax(got_build != want_build)}"
    every = np.ones(n, dtype=bool)
    for block, want in zip(out.blocks[1:3], probe_payload(want_probe)):
        assert_block_equal(block, want, every, what + ": probe payload")
    present = want_build >= 0
    for block, want in zip(out.blocks[4:], build_payload(want_build[present])):
        assert_block_equal(block, want, present, what + ": build payload")
    return got_build


def probe_ids_of(page, rows):
    return _ids(page.blocks[0])[rows]


def build_lookup(ctx, case, output=True):
    bridge = ops.JoinBridge()
    b = ops.HashBuilderOperatorFactory(ctx, bridge, case.build_keys, case.build_out if output else []).create_operator()
    for p in case.build_pages:
        assert b.needs_input()
        b.add_input(p)
    b.finish()
    return b, bridge


def run_join(ctx, case, join_type, single, by_reference=False, probe_pages=None, untouched=False):
    """Probe pages alternate over two operators of one factory; tracking join types end with the LookupOuterOperator's page."""
    what = case.say(join_type, single)
    ref = case.reference
    b, bridge = build_lookup(ctx, case)
    lookup = bridge.lookup_source
    assert lookup.get_join_position_count() == ref.position_count, what
    factory = ops.LookupJoinOperatorFactory(ctx, bridge, join_type, single, case.probe_keys, case.probe_out)
    joins = [factory.create_operator(), factory.create_operator()]
    if by_reference:
        for j in joins:
            j.set_passthrough_by_reference(True)
    emitted = []
    pages = case.probe_pages if probe_pages is None else probe_pages
    for i, page in enumerate(pages if not untouched else []):
        j = joins[i % 2]
        assert j.needs_input(), what
        j.add_input(page)
        out = j.get_output()
        assert j.get_output() is None, what
        positions = case.positions[i] if probe_pages is None else ref.positions(page, case.probe_keys)
        rows, build = ref.expand(positions, join_type, single)
        emitted.append(check_output(out, probe_ids_of(page, rows), build.astype(np.int64), f"{what} probe page {i} ({page.position_count} rows)"))
    for j in joins:
        j.finish()
        assert j.is_finished(), what
    if join_type in TRACKING:
        outer = ops.LookupOuterOperatorFactory(ctx, bridge, case.probe_out_types).create_operator()
        assert not outer.needs_input()
        page = outer.get_output()
        want = ref.unvisited(emitted).astype(np.int64)
        if page is None:
            assert len(want) == 0, f"{what}: no outer page, expected {len(want)} unvisited build rows"
        else:
            assert len(want) and page.position_count == len(want), f"{what}: outer page of {page.position_count} rows, expected {len(want)}"
            for block in page.blocks[:3]:
                assert block.nulls is not None and block.nulls.all(), f"{what}: outer page carries probe values"
            assert np.array_equal(_ids(page.blocks[3]), want), f"{what}: outer build rows differ"
            for block, wanted in zip(page.blocks[4:], build_payload(want)):
                assert_block_equal(block, wanted, np.ones(len(want), dtype=bool), what + ": outer payload")
        assert outer.get_output() is None and outer.is_finished(), what
        outer.close()
    for op in joins + [b]:
        op.close()
    lookup.close()
    return emitted


# ---------------------------------------------------------------------------------------------------- the join matrix
@pytest.mark.parametrize("single", [False, True], ids=["all_matches", "single_match"])
@pytest.mark.parametrize("join_type", list(JOIN_TYPES.values()), ids=list(JOIN_TYPES))
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_every_build_form(ctx, shape, form, join_type, single):
    run_join(ctx, cached_case(shape, form), join_type, single)


@functools.lru_cache(maxsize=None)
def large_probe_case(shape):
    return make_case(shape, "dups3", seed=2, probe_sizes=(300_001,))


@pytest.mark.parametrize("join_type,single", [(abi.JOIN_INNER, False), (abi.JOIN_PROBE_OUTER, True), (abi.JOIN_LOOKUP_OUTER, True), (abi.JOIN_FULL_OUTER, False)],
                         ids=["inner-all_matches", "probe_outer-single_match", "lookup_outer-single_match", "full_outer-all_matches"])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_probe_page_of_300001_rows(ctx, shape, join_type, single):
    run_join(ctx, large_probe_case(shape), join_type, single)


@pytest.mark.parametrize("join_type,single", [(abi.JOIN_INNER, False), (abi.JOIN_PROBE_OUTER, True), (abi.JOIN_FULL_OUTER, False)],
                         ids=["inner-all_matches", "probe_outer-single_match", "full_outer-all_matches"])
@pytest.mark.parametrize("form", ["unique", "nulls"])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_by_reference_probes_give_the_same_rows(ctx, shape, form, join_type, single):
    # a generic lookup needs every probe channel on the device, so the switch must change nothing; the single DOUBLE key does upload lazily
    run_join(ctx, cached_case(shape, form), join_type, single, by_reference=True)


@pytest.mark.parametrize("join_type", TRACKING, ids=["lookup_outer", "full_outer"])
@pytest.mark.parametrize("shape", ["varchar", "bigint+varchar+double", "int128+real"])
def test_outer_page_of_untouched_and_of_fully_visited_lookups(ctx, shape, join_type):
    case = cached_case(shape, "dups3")
    run_join(ctx, case, join_type, False, untouched=True)          # no probe page at all: every build row comes back
    # every build row visited: probe with the build's own keys (no NULL or NaN among them in this form) -> no outer page
    nk = len(case.kinds)
    everything = [probe_page(p.blocks[:nk], 0) for p in case.build_pages]
    emitted = run_join(ctx, case, join_type, False, probe_pages=everything)
    assert len(np.unique(np.concatenate(emitted))) == case.reference.position_count, case.say(join_type, False)


@pytest.mark.parametrize("single", [False, True], ids=["all_matches", "single_match"])
@pytest.mark.parametrize("join_type", list(JOIN_TYPES.values()), ids=list(JOIN_TYPES))
@pytest.mark.parametrize("name", EDGE_NAMES)
def test_edge_tables(ctx, name, join_type, single):
    run_join(ctx, edge_case(name), join_type, single)


# ---------------------------------------------------------------------------------------------------- table tiers
@pytest.mark.parametrize("shape,rows", [("bigint+integer", 70_000), ("varchar", 70_000), ("bigint+integer", 1_100_000)])
def test_load_factor_tiers(ctx, shape, rows):
    """the table is sized for a load factor of 0.25 up to 2^16 rows (every other case here), 0.5 up to 2^20 and 0.75 above"""
    case = make_case(shape, "dups3", seed=3, probe_sizes=(300_001,), build_rows=rows)
    case.probe_pages = case.probe_pages[:1]
    for join_type in (abi.JOIN_INNER, abi.JOIN_FULL_OUTER):
        run_join(ctx, case, join_type, False)


# ---------------------------------------------------------------------------------------------------- hash collisions
@pytest.mark.parametrize("single", [False, True], ids=["all_matches", "single_match"])
@pytest.mark.parametrize("join_type", list(JOIN_TYPES.values()), ids=list(JOIN_TYPES))
def test_three_tuples_on_one_row_hash(ctx, join_type, single):
    case = collision_case()
    run_join(ctx, case, join_type, single)
    b, bridge = build_lookup(ctx, case, output=False)
    lookup = bridge.lookup_source
    what = case.say(join_type, single)
    keys = Page(*case.probe_pages[0].blocks[1:3])
    positions = lookup.get_join_positions(keys)
    assert np.array_equal(positions, case.positions[0]), what
    assert lookup.has_position_links() and np.array_equal(lookup.position_links(), case.reference.links()), what + ": chains are not pure"
    heads = [positions[i * 37] for i in range(9)]
    assert heads[0] == -1 and heads[4] == -1 and heads[7] == -1 and heads[8] == -1 and min(heads[1], heads[2], heads[3]) >= 0, what
    assert len({heads[1], heads[2], heads[3]}) == 3 and heads[5] == heads[2] and heads[6] == heads[1], what
    b.close()
    lookup.close()


# ---------------------------------------------------------------------------------------------------- positions API
def _device_page(ctx, page, keep):
    cols = []
    for b in page.blocks:
        b = b.flatten()
        validity = None
        if b.nulls is not None:
            validity = ctx.to_device(np.packbits(~b.nulls, bitorder="little"))
            keep.append(validity)
        data = ctx.to_device(b.values)
        keep.append(data)
        offsets = None
        if b.type == abi.UTF8:
            offsets = ctx.to_device(b.offsets)
            keep.append(offsets)
        cols.append(ops.DeviceColumn(b.type, data, b.position_count, validity, offsets))
    return ops.DevicePage(cols, page.position_count)


@pytest.mark.parametrize("form", ["unique", "nulls"])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_positions_api_from_host_and_device_pages(ctx, shape, form):
    case = cached_case(shape, form)
    what = case.say()
    b, bridge = build_lookup(ctx, case, output=False)
    lookup = bridge.lookup_source
    ref = case.reference
    assert lookup.has_position_links() == ref.has_links(), what
    assert np.array_equal(lookup.position_links(), ref.links()), what
    for i in (3, 7, len(PROBE_SIZES)):
        keys = Page(*case.probe_pages[i].blocks[1:1 + len(case.kinds)])
        assert np.array_equal(lookup.get_join_positions(keys), case.positions[i]), f"{what} host page {i}"
        keep = []
        n = keys.position_count
        out = ctx.malloc(4 * n)
        lookup.get_join_positions_device(_device_page(ctx, keys, keep), out)
        got = ctx.to_host(out, np.int32, n)
        for p in keep + [out]:
            ctx.free(p)
        assert np.array_equal(got, case.positions[i]), f"{what} device page {i}"
    b.close()
    lookup.close()


# ---------------------------------------------------------------------------------------------------- semi-join
def run_semi(ctx, set_pages, probe, channel):
    bridge = ops.JoinBridge()
    sb = ops.SetBuilderOperatorFactory(ctx, bridge, 0).create_operator()
    for p in set_pages:
        sb.add_input(p)
    sb.finish()
    sj = ops.HashSemiJoinOperatorFactory(ctx, bridge, channel).create_operator()
    sj.add_input(probe)
    out = sj.get_output()
    sj.close()
    sb.close()
    bridge.lookup_source.close()
    return out


def semi_case(kind, set_nulls, probe_nulls, seed=1, scale=1.0):
    rng = np.random.default_rng([seed, sorted(_TYPE).index(kind), int(set_nulls), int(probe_nulls)])
    n_set, n_probe = max(4, int(2000 * scale)), max(8, int(20_000 * scale))
    digits = _digits([kind], n_set)
    set_block = _key_block(kind, digits[0][rng.integers(0, n_set // 2, n_set)], rng, 0.01 if set_nulls else 0.0, 0.01 if probe_nulls else 0.0)
    probe_block = _key_block(kind, digits[0][rng.integers(0, n_set, n_probe)], rng, 0.05 if probe_nulls else 0.0, 0.02)
    return set_block, probe_block


@pytest.mark.parametrize("probe_nulls", [False, True], ids=["probe_not_null", "probe_nulls"])
@pytest.mark.parametrize("set_nulls", [False, True], ids=["set_not_null", "set_nulls"])
@pytest.mark.parametrize("kind", ["varchar", "int128", "real"])
def test_semi_join_over_generic_sets(ctx, kind, set_nulls, probe_nulls):
    what = f"kind={kind} seed=1 set_nulls={set_nulls} probe_nulls={probe_nulls}"
    set_block, probe_block = semi_case(kind, set_nulls, probe_nulls)
    n = probe_block.position_count
    probe = Page(Block.integer(np.arange(n, dtype=np.int32)), probe_block, *probe_payload(np.arange(n)))
    half = set_block.position_count // 2
    pages = [Page(set_block.get_positions(np.arange(half))), Page(set_block.get_positions(np.arange(half, set_block.position_count)))]
    out = run_semi(ctx, pages, probe, 1)
    want = jr.semi(set_block, probe_block)
    assert out.blocks[4].to_pylist() == want, what
    assert True in want and (False in want) == (not set_nulls) and (None in want) == (set_nulls or probe_nulls), what
    every = np.ones(n, dtype=bool)
    for got, sent in zip(out.blocks[:4], probe.blocks):                       # the input channels pass through unchanged
        assert_block_equal(got, sent, every, what + ": pass-through")
    # an empty set answers FALSE for every row, NULL keys included
    empty = Page(set_block.get_positions(np.arange(0)), position_count=0)
    out = run_semi(ctx, [empty], probe, 1)
    assert out.blocks[4].to_pylist() == jr.semi(empty.blocks[0], probe_block) == [False] * n, what + " empty set"


# ---------------------------------------------------------------------------------------------------- argument errors
def test_nine_join_channels_are_refused(ctx):
    # one channel more than MAX_KEY_COLS: the build operator is not created at all (eight channels build and join in test_every_build_form)
    factory = ops.HashBuilderOperatorFactory(ctx, ops.JoinBridge(), list(range(9)), [])
    with pytest.raises(abi.TrinoGpuError) as e:
        factory.create_operator()
    assert e.value.code == abi.ERR_NOT_SUPPORTED


@pytest.mark.parametrize("kind", ["varchar", "real", "int128", "bigint"])
def test_build_that_never_saw_a_page(ctx, kind):
    """An empty build side sends no page, so the lookup knows no channel type: every probe row misses, whatever its key type, through
    the join, the semi-join and the positions API."""
    what = f"build without pages, probe key {kind}"
    bridge = ops.JoinBridge()
    b = ops.HashBuilderOperatorFactory(ctx, bridge, [0], []).create_operator()
    b.finish()
    lookup = bridge.lookup_source
    assert lookup.get_join_position_count() == 0, what
    key = _ONE[kind]()
    probe = Page(Block.integer([0, 1, 2]), key)
    assert lookup.get_join_positions(Page(key)).tolist() == [-1, -1, -1], what
    for join_type, want in ((abi.JOIN_INNER, []), (abi.JOIN_PROBE_OUTER, [0, 1, 2]), (abi.JOIN_FULL_OUTER, [0, 1, 2])):
        j = ops.LookupJoinOperatorFactory(ctx, bridge, join_type, False, [1], [0, 1]).create_operator()
        j.add_input(probe)
        out = j.get_output()
        assert ([] if out is None else _ids(out.blocks[0]).tolist()) == want, what
        if want:
            assert out.blocks[1].to_pylist() == key.to_pylist(), what
        j.close()
    sj = ops.HashSemiJoinOperatorFactory(ctx, bridge, 1).create_operator()
    sj.add_input(probe)
    assert sj.get_output().blocks[2].to_pylist() == jr.semi(key.get_positions([]), key) == [False, False, False], what
    sj.close()
    b.close()
    lookup.close()


def test_integer_channels_of_different_widths_join_by_value(ctx):
    bridge = ops.JoinBridge()
    b = ops.HashBuilderOperatorFactory(ctx, bridge, [0, 1], []).create_operator()
    b.add_input(Page(Block.bigint([1, 2, -3, 1 << 40]), Block.varchar(["a", "b", "c", "d"])))
    b.finish()
    lookup = bridge.lookup_source
    narrow = Page(Block.integer([-3, 2, 1, 0]), Block.varchar(["c", "b", "b", "d"]))
    assert lookup.get_join_positions(narrow).tolist() == [2, 1, -1, -1]
    b.close()
    lookup.close()


_ONE = {"varchar": lambda: Block.varchar(["a", "b", None]), "bigint": lambda: Block.bigint([1, 2, None]), "double": lambda: Block.double([1.0, 2.0, None]),
        "real": lambda: Block.real([1.0, 2.0, None]), "integer": lambda: Block.integer([1, 2, None]), "int128": lambda: Block.int128([1, 2, None])}
MISMATCHES = [("varchar", "bigint"), ("bigint", "varchar"), ("double", "bigint"), ("bigint", "double"), ("real", "integer"), ("integer", "real"),
              ("int128", "bigint"), ("bigint", "int128")]


def _expect_invalid(call, what):
    with pytest.raises(abi.TrinoGpuError) as e:
        call()
    assert e.value.code == abi.ERR_INVALID_ARGUMENT, f"{what}: {e.value}"


@pytest.mark.parametrize("second_channel", [False, True], ids=["single_channel", "second_of_two"])
@pytest.mark.parametrize("build_kind,probe_kind", MISMATCHES)
def test_probe_key_types_must_match_the_build(ctx, build_kind, probe_kind, second_channel):
    """Key channels are compared with the width and semantics of their type, so a probe channel of another type is an argument error from
    every entry point, and the operators take a correct page afterwards."""
    what = f"build {build_kind}, probe {probe_kind}, second_channel={second_channel}"
    lead = [Block.bigint([7, 7, 7])] if second_channel else []
    keys = list(range(len(lead) + 1))
    bridge = ops.JoinBridge()
    b = ops.HashBuilderOperatorFactory(ctx, bridge, keys, [0]).create_operator()
    b.add_input(Page(*lead, _ONE[build_kind]()))
    b.finish()
    lookup = bridge.lookup_source
    good, bad = Page(*lead, _ONE[build_kind]()), Page(*lead, _ONE[probe_kind]())
    j = ops.LookupJoinOperatorFactory(ctx, bridge, abi.JOIN_INNER, False, keys, keys).create_operator()
    _expect_invalid(lambda: j.add_input(bad), what + " add_input")
    _expect_invalid(lambda: lookup.get_join_positions(bad), what + " get_join_positions")
    assert j.needs_input(), what
    j.add_input(good)
    assert j.get_output().position_count == 2, what
    assert lookup.get_join_positions(good).tolist() == [0, 1, -1], what
    if not second_channel:
        sj = ops.HashSemiJoinOperatorFactory(ctx, bridge, 0).create_operator()
        _expect_invalid(lambda: sj.add_input(bad), what + " semi-join")
        sj.add_input(good)
        assert sj.get_output().blocks[1].to_pylist() == [True, True, None], what
        sj.close()
    j.close()
    b.close()
    lookup.close()


def test_probe_channel_count_must_match_the_build(ctx):
    bridge = ops.JoinBridge()
    b = ops.HashBuilderOperatorFactory(ctx, bridge, [0, 1], []).create_operator()
    b.add_input(Page(Block.bigint([1, 2]), Block.varchar(["a", "b"])))
    b.finish()
    lookup = bridge.lookup_source
    three = Page(Block.bigint([1, 2]), Block.varchar(["a", "b"]), Block.bigint([1, 2]))
    for channels, page in (([0], three), ([0, 1, 2], three)):
        j = ops.LookupJoinOperatorFactory(ctx, bridge, abi.JOIN_INNER, False, channels, [0]).create_operator()
        _expect_invalid(lambda: j.add_input(page), f"{len(channels)} probe channels, 2 build channels")
        j.close()
    _expect_invalid(lambda: lookup.get_join_positions(three), "3 key columns, 2 build channels")
    _expect_invalid(lambda: ops.HashSemiJoinOperatorFactory(ctx, bridge, 0).create_operator(), "semi-join over a two-channel lookup")
    j = ops.LookupJoinOperatorFactory(ctx, bridge, abi.JOIN_INNER, False, [0, 1], [0]).create_operator()
    j.add_input(three)
    assert j.get_output().position_count == 2
    j.close()
    b.close()
    lookup.close()
