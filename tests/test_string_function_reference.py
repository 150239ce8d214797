"""string_function_reference.py pinned on the reference's own vectors (TestStringFunctions, restated as data in
tests/golden/string_function_cases.json) and on the edges the GPU tests rely on.  Needs no GPU."""
import json
import os

import pytest

import string_function_reference as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = json.load(open(os.path.join(ROOT, "tests", "golden", "string_function_cases.json")))


def _arg(a):
    return a.encode() if isinstance(a, str) else a


@pytest.mark.parametrize("case", CASES["cases"], ids=lambda c: c["source"].rsplit(":", 1)[1] + "-" + c["function"])
def test_reference_vectors(case):
    args = [_arg(a) for a in case["args"]]
    got = ref.FUNCTIONS[case["function"]](*args)
    assert got == _arg(case["result"]), case["source"]


def test_every_function_has_vectors():
    assert {c["function"] for c in CASES["cases"]} == {"concat", "length", "substr", "ltrim", "rtrim"}


@pytest.mark.parametrize("case", CASES["concat_limit"], ids=lambda c: "+".join(map(str, c["pieces"])))
def test_concat_limit(case):
    pieces = [b"x" * n for n in case["pieces"]]
    if case["raises"]:
        with pytest.raises(ref.ConcatTooLarge):
            ref.concat(*pieces)
        assert ref.concat(*pieces, None) is None          # a NULL piece: NULL, no error
    else:
        assert len(ref.concat(*pieces)) == sum(case["pieces"])


def test_whitespace_set():
    """the two vectors the reference pins (ASCII space, U+2028) and Character.isWhitespace's exclusions"""
    assert ref.trim(" \u2028 a \u2028 ".encode()) == b"a"
    for c in ("\u00a0", "\u2007", "\u202f", "\u200b", "\u180e"):
        assert ref.trim((c + "a" + c).encode()) == (c + "a" + c).encode(), hex(ord(c))
    for c in ("\t", "\n", "\x0b", "\x0c", "\r", "\x1c", "\x1f", "\u1680", "\u2000", "\u200a", "\u2029", "\u205f", "\u3000"):
        assert ref.trim((c + "a" + c).encode()) == b"a", hex(ord(c))


def test_substring_edges():
    s = "añ名\U0001F600z".encode()         # 1- to 4-byte code points
    assert ref.length(s) == 5
    assert ref.substring(s, 2, 3) == "ñ名\U0001F600".encode()
    assert ref.substring(s, -1) == b"z" and ref.substring(s, -5) == s and ref.substring(s, -6) == b""
    assert ref.substring(s, 5) == b"z" and ref.substring(s, 6) == b"" and ref.substring(s, 0) == b""
    assert ref.substring(s, 1, 5) == s and ref.substring(s, 1, 6) == s and ref.substring(s, 1, 4) == s[:-1]
    assert ref.substring(s, -(1 << 63)) == b"" and ref.substring(s, (1 << 63) - 1) == b""
    assert ref.substring(s, 1, (1 << 63) - 1) == s and ref.substring(s, 2, -(1 << 63)) == b""
    assert ref.substring(s, -5, (1 << 63) - 1) == s                 # startCodePoint 0: no wrap
    with pytest.raises(ref.SliceOutOfBounds):                       # the reference's own failure
        ref.substring(s, -1, (1 << 63) - 1)
    assert ref.substring(s, -1, (1 << 63) - 1, java_int_wrap=False) == b"z"


def test_invalid_utf8_stays_in_bounds():
    for s in (b"\x80\x80a", b"a\xc3", b"\xf0\x9f\x98", b"\xff\xfe", b" \xc3 ", b"\xe2\x80\xa8\x80"):
        n = len(s)
        for start in range(-n - 2, n + 3):
            for length in (None, 0, 1, 2, n + 1):
                r = ref.substring(s, start, length, java_int_wrap=False)
                assert r in s
        assert ref.length(s) <= n
        for f in (ref.ltrim, ref.rtrim, ref.trim):
            assert f(s) in s
