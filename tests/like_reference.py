"""Exact host-side restatement of the reference's LIKE over VARCHAR: LikeFunctions.likeVarchar (M/type/LikeFunctions.java:49-56) over
the matcher a constant pattern gets, LikeMatcher.compile(pattern, escape, optimize = true) (M/likematcher/LikeMatcher.java:58-153,
reached through M/type/LikePatternType.java:94).

The pattern is a Java String, so it is parsed as UTF-16 code units, as LikeMatcher.parse (:196-274) parses it: `_` counts one code unit
and the escape is one code unit.  The compiled matcher checks the length bounds (`_` counts 1 to 4 bytes, :62-84), the constant prefix
and suffix (:89-102, :160-183) and runs one of three matchers over the middle:
- FjsMatcher when the middle holds only literals and `%`: each literal at its leftmost occurrence after the previous one, bytewise;
- DenseDfaMatcher when the first `_` of the middle comes before any `%`: here the NFA that DenseDfa.makeNfa builds over BYTES, run as a
  set of states (the same language as its DFA).  `_` and `%` consume well-formed UTF-8 lead / continuation sequences only;
- NfaMatcher otherwise: `_` consumes one code point decoded from the lead byte alone (continuation bytes are not checked; a stray or
  truncated sequence fails the match), and a literal state matches a code point equal to its UTF-16 code unit.
"""
import struct

ANY, NONE = -1, -2


class InvalidPattern(ValueError):
    """Where the reference throws (an invalid escape use, an escape that is not one character): the library answers NOT_SUPPORTED"""


def _units(s):
    b = s.encode("utf-16-le", "surrogatepass")
    return list(struct.unpack("<%dH" % (len(b) // 2), b))


def _units_to_utf8(units):
    """String.getBytes(UTF_8): an unpaired surrogate becomes '?'"""
    out = bytearray()
    i = 0
    while i < len(units):
        u = units[i]
        if 0xD800 <= u <= 0xDBFF and i + 1 < len(units) and 0xDC00 <= units[i + 1] <= 0xDFFF:
            out += chr(0x10000 + ((u - 0xD800) << 10) + (units[i + 1] - 0xDC00)).encode()
            i += 2
            continue
        out += b"?" if 0xD800 <= u <= 0xDFFF else chr(u).encode()
        i += 1
    return bytes(out)


def parse(pattern, escape=None):
    """LikeMatcher.parse: [("lit", [units]) | ("any", n) | ("zom",)]"""
    units = _units(pattern)
    esc = None
    if escape is not None:
        e = _units(escape)
        if len(e) != 1:
            raise InvalidPattern("Escape string must be a single character")
        esc = e[0]
    result, literal, any_count, unbounded, in_escape = [], [], 0, False, False

    def flush():
        nonlocal any_count, unbounded
        if any_count:
            result.append(("any", any_count))
            any_count = 0
        if unbounded:
            result.append(("zom",))
            unbounded = False

    for ch in units:
        if in_escape:
            if ch not in (ord("%"), ord("_"), esc):
                raise InvalidPattern("Escape character must be followed by '%', '_' or the escape character itself")
            literal.append(ch)
            in_escape = False
        elif esc is not None and ch == esc:
            in_escape = True
            flush()
        elif ch in (ord("%"), ord("_")):
            if literal:
                result.append(("lit", literal))
                literal = []
            if ch == ord("%"):
                unbounded = True
            else:
                any_count += 1
        else:
            flush()
            literal.append(ch)
    if in_escape:
        raise InvalidPattern("Escape character must be followed by '%', '_' or the escape character itself")
    if literal:
        result.append(("lit", literal))
    else:
        flush()
    return result


class Matcher:
    def __init__(self, pattern, escape=None):
        items = parse(pattern, escape)
        self.items = items
        self.min_size = self.max_size = 0
        unbounded = False
        for it in items:
            if it[0] == "lit":
                n = len(_units_to_utf8(it[1]))
                self.min_size += n
                self.max_size += n
            elif it[0] == "any":
                self.min_size += it[1]
                self.max_size += 4 * it[1]
            else:
                unbounded = True
        if unbounded:
            self.max_size = None
        self.prefix = self.suffix = b""
        start, end = 0, len(items) - 1
        if items and items[0][0] == "lit":
            self.prefix = _units_to_utf8(items[0][1])
            start += 1
        if len(items) > 1 and items[-1][0] == "lit":
            self.suffix = _units_to_utf8(items[-1][1])
            end -= 1
        self.exact = True
        if start <= end and items[end][0] == "zom":
            self.exact = False
            end -= 1
        self.middle = items[start:end + 1]
        self.kind = "none"
        if self.middle:
            has_any = any_after_zom = zom = False
            for it in self.middle:
                if it[0] == "any":
                    any_after_zom, has_any = zom, True
                    break
                if it[0] == "zom":
                    zom = True
            self.kind = "fjs" if not has_any else ("dfa" if not any_after_zom else "nfa")

    def match(self, value):
        """value: bytes"""
        n = len(value)
        if n < self.min_size or (self.max_size is not None and n > self.max_size):
            return False
        if not value.startswith(self.prefix) or not value[n - len(self.suffix):].startswith(self.suffix):
            return False
        mid = value[len(self.prefix):n - len(self.suffix)]
        if self.kind == "fjs":
            return self._fjs(mid)
        if self.kind == "dfa":
            return self._dfa(mid)
        if self.kind == "nfa":
            return self._nfa(mid)
        return True

    # FjsMatcher.Fjs.match (M/likematcher/FjsMatcher.java:188-211)
    def _fjs(self, mid):
        start = 0
        for it in self.middle:
            if it[0] != "lit":
                continue
            if start == len(mid):
                return False
            term = _units_to_utf8(it[1])
            at = mid.find(term, start)
            if at < 0:
                return False
            start = at + len(term)
        return not self.exact or start == len(mid)

    # DenseDfaMatcher.makeNfa (M/likematcher/DenseDfaMatcher.java:141-212): transitions (from, predicate, to) over bytes
    def _byte_nfa(self):
        trans, count = [], [1]

        def add():
            count[0] += 1
            return count[0] - 1

        def utf8_char(frm, to):
            s1, s2, s3 = add(), add(), add()
            trans.extend([(frm, lambda b: b >> 7 == 0, to), (frm, lambda b: b >> 3 == 0b11110, s1), (frm, lambda b: b >> 4 == 0b1110, s2),
                          (frm, lambda b: b >> 5 == 0b110, s3), (s1, lambda b: b >> 6 == 0b10, s2), (s2, lambda b: b >> 6 == 0b10, s3),
                          (s3, lambda b: b >> 6 == 0b10, to)])

        state = 0
        for it in self.middle:
            if it[0] == "lit":
                for byte in _units_to_utf8(it[1]):
                    nxt = add()
                    trans.append((state, (lambda v: lambda b: b == v)(byte), nxt))
                    state = nxt
            elif it[0] == "any":
                for _ in range(it[1]):
                    nxt = add()
                    utf8_char(state, nxt)
                    state = nxt
            else:
                utf8_char(state, state)
        return trans, state

    def _dfa(self, mid):
        trans, accept = self._byte_nfa()
        states = {0}
        for b in mid:
            states = {to for frm, pred, to in trans if frm in states and pred(b)}
            if not states:
                return False
            if not self.exact and accept in states:
                return True
        return accept in states

    # NfaMatcher (M/likematcher/NfaMatcher.java:33-164)
    def _nfa(self, mid):
        match, loopback = [], []
        for it in self.middle:
            if it[0] == "zom":
                loopback.append(len(match))
            else:
                match += it[1] if it[0] == "lit" else [ANY] * it[1]
        accept_state = len(match)
        match.append(NONE)
        loop = set(loopback)
        current, accept, i, limit = {0}, False, 0, len(mid)
        while i < limit:
            h = mid[i]
            cp = None
            if h < 0x80:
                cp, i = h, i + 1
            elif h & 0xE0 == 0xC0:
                if i + 1 < limit:
                    cp, i = ((h & 0x1F) << 6) | (mid[i + 1] & 0x3F), i + 2
            elif h & 0xF0 == 0xE0:
                if i + 2 < limit:
                    cp, i = ((h & 0x0F) << 12) | ((mid[i + 1] & 0x3F) << 6) | (mid[i + 2] & 0x3F), i + 3
            elif h & 0xF8 == 0xF0:
                if i + 3 < limit:
                    cp = ((h & 0x07) << 18) | ((mid[i + 1] & 0x3F) << 12) | ((mid[i + 2] & 0x3F) << 6) | (mid[i + 3] & 0x3F)
                    i += 4
            if cp is None:
                return False
            nxt = set()
            for s in current:
                if s in loop:
                    nxt.add(s)
                if match[s] == ANY or match[s] == cp:
                    nxt.add(s + 1)
            if not nxt:
                return False
            accept = accept_state in nxt
            if not self.exact and accept:
                return True
            current = nxt
        return accept


def like(value, pattern, escape=None):
    """value LIKE pattern [ESCAPE escape]; value: bytes or str (taken as UTF-8); raises InvalidPattern where the reference throws"""
    return Matcher(pattern, escape).match(value.encode() if isinstance(value, str) else bytes(value))
