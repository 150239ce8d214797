"""The plain-Python join reference (join_reference.py) against what pins it: the cases copied from the reference's own operator tests,
and the C++ oracle on every case generator of test_gpu_join_generic.py at reduced size.  Needs no device."""
import numpy as np
import pytest

import join_reference as jr
import oracle_lib as o
import test_gpu_join_generic as g
from helpers import join_type_of, reference_cases
from trino_b200 import abi
from trino_b200.page import Block, Page


def _rows(build, probe, build_key, probe_key, probe_out, build_out, join_type, single):
    ref = jr.JoinReference(build, build_key)
    rows, positions = ref.expand(ref.positions(probe, probe_key), join_type, single)
    pcols = [probe.get_block(c).to_pylist() for c in probe_out]
    bcols = [build.get_block(c).to_pylist() for c in build_out]
    return [tuple(c[p] for c in pcols) + tuple(c[b] if b >= 0 else None for c in bcols) for p, b in zip(rows.tolist(), positions.tolist())]


def test_golden_join_cases():
    for case in reference_cases()["join"]:
        build = Page(Block.bigint(case["build"])) if case["build"] else Page(Block.bigint([]), position_count=0)
        probe = Page(Block.bigint(case["probe"]))
        got = _rows(build, probe, [0], [0], [0], [0], join_type_of(case), case["single_match"])
        assert got == [tuple(r) for r in case["expected"]], case["source"]


@pytest.mark.parametrize("key", ["bigint", "varchar"])
def test_golden_probe_outer_sequence(key):
    c = reference_cases()["probe_outer_sequence"]
    make = Block.bigint if key == "bigint" else lambda v: Block.varchar([str(x) for x in v])
    sides = []
    for initial, n in ((c["build_initial"], c["build_rows"]), (c["probe_initial"], c["probe_rows"])):
        sides.append(Page(make([initial[0] + i for i in range(n)]), *[Block.bigint([x + i for i in range(n)]) for x in initial[1:]]))
    build, probe = sides
    rows = _rows(build, probe, [0], [0], [0, 1, 2], [0, 1, 2], abi.JOIN_PROBE_OUTER, False)
    k = (lambda v: v) if key == "bigint" else (lambda v: str(v).encode())
    assert len(rows) == 15
    assert rows[0] == (k(20), 1020, 2020, k(20), 30, 40) and rows[9] == (k(29), 1029, 2029, k(29), 39, 49) and rows[-1] == (k(34), 1034, 2034, None, None, None)


def test_golden_semi_join_cases():
    for case in reference_cases()["semi_join"]:
        assert jr.semi(Block.bigint(case["set"]), Block.bigint(case["probe"])) == case["expected"], case["source"]
    assert jr.semi(Block.bigint([]), Block.bigint([1, None])) == [False, False]


def _against_oracle(case):
    """positions, links and every expansion of one generated case: the reference and oracle_lib.Join agree.  The oracle takes one build
    page, so multi-page builds are concatenated for it; it accepts every key type the generators produce."""
    ref = case.reference
    if len(case.build_pages) == 1:
        whole = case.build_pages[0]
    else:
        nk = len(case.kinds)
        columns = [sum((p.get_block(c).flatten().to_pylist() for p in case.build_pages), []) for c in range(nk)]
        whole = Page(*g.blocks_from_rows(case.kinds, list(zip(*columns))))
    oj = o.Join(whole, case.build_keys)
    assert np.array_equal(oj.links(), ref.links()), case.say()
    assert oj.has_links() == ref.has_links(), case.say()
    for i, page in enumerate(case.probe_pages):
        want = oj.positions(page, case.probe_keys)
        assert np.array_equal(case.positions[i], want), f"{case.say()} probe page {i}"
        for join_type in g.JOIN_TYPES.values():
            for single in (False, True):
                rows, build = ref.expand(want, join_type, single)
                orows, obuild = oj.expand(want, join_type, single)
                assert np.array_equal(rows, orows) and np.array_equal(build, obuild), f"{case.say(join_type, single)} probe page {i}"
    oj.close()


@pytest.mark.parametrize("form", g.FORMS)
@pytest.mark.parametrize("shape", list(g.SHAPES))
def test_generated_cases_against_the_oracle(shape, form):
    case = g.make_case(shape, form, scale=0.1)
    _against_oracle(case)
    if form in ("unique", "dups3", "nulls"):
        hit = np.concatenate(case.positions) >= 0
        assert 0.2 < hit.mean() < 0.9, case.say()         # the generators do produce matches and misses


@pytest.mark.parametrize("name", g.EDGE_NAMES)
def test_edge_tables_against_the_oracle(name):
    _against_oracle(g.edge_case(name))


def test_collision_case_against_the_oracle():
    case = g.collision_case(ordinary=500)
    _against_oracle(case)
    a, b = zip(*case.colliding)
    hashes = o.row_hashes(Page(Block.bigint(list(a)), Block.bigint(list(b))), [0, 1])
    assert len(set(hashes.tolist())) == 1 and len(set(case.colliding)) == 4        # four tuples, one reference row hash
    chains = sorted(len(case.reference.chains[t]) for t in case.colliding[:3])
    assert chains == [1, 2, 5] and case.colliding[3] not in case.reference.chains


def test_edge_tables_hold_the_matches_they_are_written_for():
    """the explicit tables would prove nothing if their interesting rows did not match (or matched) in the reference itself"""
    def pos(name):
        case = g.edge_case(name)
        return case.positions[0].tolist()
    p = pos("strings")
    assert p[0] == 13 and p[1] == -1 and p[2] == 12 and p[3] == 16 and p[15] == 15 and p[6] == 6 and p[7] == 7 and p[17:] == [-1] * 5
    p = pos("tuple_boundaries")
    assert p[:6] == [1, 8, 3, 2, 5, 4] and p[6:] == [-1] * 5
    assert pos("swapped_integers") == [1, 5, -1, 4, 3, -1, -1, -1]
    p = pos("real_bits")
    assert p[0] == 0 and p[1] == 1 and p[2] == 2 and p[4] == 5 and p[5] == 5 and p[6] == -1 and p[7] == -1 and p[10] == 1 and p[11] == 5
    p = pos("double_bits")
    assert p[:3] == [-1] * 3 and p[3] == 4 and p[4] == 4 and p[5] == 5 and p[6] == 6 and p[8] == -1 and p[9] == 4
    assert pos("nan_and_zero_in_tuples") == [6, 1, -1, -1, 4, -1, -1, -1, -1, -1]
    p = pos("int128_words")
    assert p[:14] == [0, 15, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13] and p[14] == -1 and p[16:] == [-1] * 4
    assert pos("int128_in_tuples") == [1, 0, -1, 3, -1, 4, -1, -1]
    assert pos("int128_colliding_tuples") == [1, 2, -1, -1] and pos("varchar_colliding_tuples") == [1, 2, -1, -1]


@pytest.mark.parametrize("kind", ["int128", "varchar"])
def test_crafted_tuples_share_the_reference_row_hash(kind):
    """the two tuples differ in every channel, only in the high words / only by a longer string, and the oracle gives them one row hash"""
    a, b = g.colliding_int128_tuples() if kind == "int128" else g.colliding_varchar_tuples()
    page = Page(*g.blocks_from_rows([kind, kind], [a, b]))
    hashes = o.row_hashes(page, [0, 1])
    assert hashes[0] == hashes[1] and a[0] != b[0] and a[1] != b[1]
    if kind == "int128":
        assert all(x & ((1 << 64) - 1) == y & ((1 << 64) - 1) and x >> 64 != y >> 64 for x, y in zip(a, b))
    else:
        assert all(y.startswith(x) and len(y) > len(x) for x, y in zip(a, b))


@pytest.mark.parametrize("kind", ["bigint", "double", "real"])
@pytest.mark.parametrize("set_nulls,probe_nulls", [(False, False), (True, False), (False, True), (True, True)])
def test_semi_join_against_the_oracle(kind, set_nulls, probe_nulls):
    """the oracle restates the semi-join over BIGINT, DOUBLE and REAL only; VARCHAR and long DECIMAL sets rest on the golden cases' rules"""
    set_block, probe_block = g.semi_case(kind, set_nulls, probe_nulls, scale=0.2)
    want = o.semi_join_bigint(set_block, probe_block) if kind == "bigint" else o.semi_join_float(set_block, probe_block)
    assert jr.semi(set_block, probe_block) == want


@pytest.mark.parametrize("kind", ["varchar", "int128"])
def test_semi_join_rules_do_not_depend_on_the_key_type(kind):
    """a VARCHAR / long DECIMAL semi-join is the BIGINT one under an injective renaming of the keys"""
    rng = np.random.default_rng(4)
    sd, pd = rng.integers(0, 50, 200), rng.integers(0, 100, 1000)
    sn, pn = rng.random(200) < 0.02, rng.random(1000) < 0.05

    def block(d, nulls):
        b = g._key_block(kind, d, rng, 0.0, 0.0)
        return Block(b.type, b.values, nulls, b.offsets)
    assert jr.semi(block(sd, sn), block(pd, pn)) == jr.semi(Block.bigint(sd, sn), Block.bigint(pd, pn))


def test_semi_join_literal_varchar_and_int128_cases():
    """HashSemiJoinOperator.java:181-199 by hand: a match is TRUE; no match is FALSE, or NULL when the set holds a NULL; a NULL probe key is
    NULL, or FALSE over an empty set"""
    v = Block.varchar
    assert jr.semi(v(["a", "b", "b", None]), v(["a", None, "c", "", "b"])) == [True, None, None, None, True]
    assert jr.semi(v(["a", "", "ab"]), v(["a", "ab", "abc", None, "", "b"])) == [True, True, False, None, True, False]
    assert jr.semi(v([]), v(["a", None])) == [False, False]
    assert jr.semi(v([None]), v(["a", None])) == [None, None]
    d = Block.int128
    assert jr.semi(d([1 << 64, 1, -1]), d([1, 1 << 64, (1 << 64) + 1, None, -1, -(1 << 64)])) == [True, True, False, None, True, False]
    assert jr.semi(d([5, None, 5]), d([5, 6, None])) == [True, None, None]
    assert jr.semi(d([]), d([5, None])) == [False, False]
