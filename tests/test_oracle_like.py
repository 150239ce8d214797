"""The LIKE restatement (like_reference.py) pinned on the reference's own cases: every case of TestLikeMatcher (test, testEscape,
testExponentialBehavior and the all-code-point `_` loop) and the VARCHAR cases of TestLikeFunctions, restated as data in
tests/golden/like_cases.json with their file:line.  Also pins which matcher LikeMatcher.compile picks for a pattern."""
import json
import os

import pytest

import like_reference as lr

CASES = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "like_cases.json")))["cases"]


def _value(c):
    return bytes.fromhex(c["value_hex"]) if "value_hex" in c else c["value"].encode()


@pytest.mark.parametrize("case", CASES, ids=lambda c: f"{c['source'].rsplit('/', 1)[-1]}:{c['pattern']!r}:{c.get('value', c.get('value_hex'))!r}"[:80])
def test_reference_cases(case):
    if case["want"] == "error":
        with pytest.raises(lr.InvalidPattern):
            lr.Matcher(case["pattern"], case["escape"])
        return
    assert lr.like(_value(case), case["pattern"], case["escape"]) is case["want"]


def test_every_code_point_is_one_underscore():
    """TestLikeMatcher.java:102-114: '_' matches every code point alone, and '_a%b_' matches 'aa' + (char) i + 'bb' (a lone surrogate
    code unit is written as '?' by getBytes)"""
    single, multiple = lr.Matcher("_"), lr.Matcher("_a%b_")
    assert single.kind == "dfa" and multiple.kind == "dfa"         # no literal prefix / suffix to take: the middle is the whole pattern
    dfa = lr.Matcher("%_")          # Any before the ZeroOrMore after parsing: DenseDfaMatcher
    nfa = lr.Matcher("%x_")         # '_' after '%': NfaMatcher
    assert dfa.kind == "dfa" and nfa.kind == "nfa"
    for i in list(range(0, 0x800, 7)) + list(range(0x800, 0x10FFFF, 4099)) + [0x7F, 0x80, 0x7FF, 0xFFFF, 0x10000, 0x10FFFE]:
        ch = "?" if 0xD800 <= i <= 0xDFFF else chr(i)
        b = ch.encode()
        assert single.match(b)
        assert multiple.match(b"aa" + b + b"bb")
        assert lr.Matcher("x%a_y").match(b"xa" + b + b"y")        # NFA: one code point
        assert lr.Matcher("x_%y").match(b"x" + b + b"y")          # DFA: one well-formed sequence
    # the full loop for the DFA and the NFA middles over the BMP, where the cost is small
    for i in range(0, 0x10000, 97):
        b = ("?" if 0xD800 <= i <= 0xDFFF else chr(i)).encode()
        assert lr.Matcher("x_%y").match(b"x" + b + b"y") and lr.Matcher("x%a_y").match(b"xa" + b + b"y")


def test_matcher_selection_follows_compile():
    """LikeMatcher.compile :115-145: FJS without '_', DFA when no '_' follows a '%', NFA otherwise; prefix / suffix / exact"""
    m = lr.Matcher("%special%requests%")
    assert (m.kind, m.prefix, m.suffix, m.exact) == ("fjs", b"", b"", False)
    m = lr.Matcher("MEDIUM POLISHED%")
    assert (m.kind, m.prefix, m.max_size) == ("none", b"MEDIUM POLISHED", None)
    m = lr.Matcher("%BRASS")
    assert (m.kind, m.suffix) == ("none", b"BRASS")
    assert lr.Matcher("a_b%c").kind == "dfa"
    assert lr.Matcher("a%b_c").kind == "nfa"
    assert lr.Matcher("x%_y").kind == "dfa"           # parse puts Any(1) before the ZeroOrMore of a '%_' run
    m = lr.Matcher("ab__")
    assert (m.min_size, m.max_size) == (4, 10)


def test_malformed_utf8_differs_between_matchers():
    """The DFA consumes only well-formed lead / continuation sequences; the NFA decodes by the lead byte alone"""
    bad = b"x\xc3(y"                                  # a 2-byte lead followed by a non-continuation byte
    assert lr.Matcher("x_%y").match(bad) is False       # DFA: \xc3 needs a continuation byte
    assert lr.Matcher("x%a_y").match(b"xa\xc3(y") is True   # NFA: \xc3( decodes as one code point
    assert lr.Matcher("x%a_y").match(b"xa\xffy") is False   # a stray byte fails the NFA
    assert lr.Matcher("%b%").match(b"abc\xffxy") is True  # FJS is bytewise (TestLikeFunctions.testLikeInvalidUtf8Value)


@pytest.mark.parametrize("pattern,escape", [("a", "ab"), ("a", "😀")])
def test_escape_of_more_than_one_character_is_refused(pattern, escape):
    with pytest.raises(lr.InvalidPattern):
        lr.Matcher(pattern, escape)
