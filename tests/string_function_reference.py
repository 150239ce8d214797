"""An exact Python restatement of the string functions FilterAndProject evaluates on the GPU, over bytes.

M = core/trino-main/src/main/java/io/trino/operator/scalar.  Code points are counted as airlift's SliceUtf8 counts them: every byte that
is not a continuation byte (10xxxxxx).  On bytes that are not UTF-8 the reference documents no result; the functions here restate the
device's deterministic choice (see device_lib.cuh), marked "no parity".
"""

MAX_CONCAT_BYTES = 1 << 20      # DEFAULT_MAX_PAGE_SIZE_IN_BYTES (spi/block/PageBuilderStatus.java:22), ConcatFunction.MAX_OUTPUT_LENGTH
INT_MIN, INT_MAX = -(1 << 31), (1 << 31) - 1

# Character.isWhitespace: SPACE_SEPARATOR but U+00A0, U+2007, U+202F; LINE_SEPARATOR; PARAGRAPH_SEPARATOR; U+0009-U+000D; U+001C-U+001F
WHITESPACE = frozenset([0x20, 0x1680, 0x2028, 0x2029, 0x205F, 0x3000] + list(range(0x09, 0x0E)) + list(range(0x1C, 0x20)) +
                       [c for c in range(0x2000, 0x200B) if c != 0x2007])


class ConcatTooLarge(Exception):
    """INVALID_FUNCTION_ARGUMENT "Concatenated string is too large" (ConcatFunction.java:82-88)"""


class SliceOutOfBounds(Exception):
    """Slice.slice's IndexOutOfBoundsException: substring(utf8, start, length) where Java's int sum startCodePoint + lengthCodePoints wraps
    (StringFunctions.java:366) - an internal error of the reference, not a SQL result"""


def _cont(b):
    return (b & 0xC0) == 0x80


def _saturated_cast(v):
    """Ints.saturatedCast"""
    return max(INT_MIN, min(INT_MAX, v))


def _wrap_int(v):
    return (v + (1 << 31)) % (1 << 32) - (1 << 31)


def count_code_points(s):
    """SliceUtf8.countCodePoints"""
    return sum(1 for b in s if not _cont(b))


def offset_of_code_point(s, position, count):
    """SliceUtf8.offsetOfCodePoint(utf8, position, codePointCount): -1 when the string ends first"""
    if len(s) - position <= count:
        return -1
    i = position
    for _ in range(count):
        i += 1
        while i < len(s) and _cont(s[i]):
            i += 1
        if i >= len(s):
            return -1
    return i


def length(s):
    """StringFunctions.length (M/StringFunctions.java:95-102)"""
    return count_code_points(s)


def substring(s, start, length=None, java_int_wrap=True):
    """StringFunctions.substring(utf8, start) (M/StringFunctions.java:284-320) and substring(utf8, start, length) (:331-378).
    java_int_wrap=False: the device's result where the reference fails in Slice.slice (the suffix)"""
    if start == 0 or (length is not None and length <= 0) or len(s) == 0:
        return b""
    sc = _saturated_cast(start)
    lc = _saturated_cast(length) if length is not None else 0
    if sc > 0:
        b = offset_of_code_point(s, 0, sc - 1)
        if b < 0:
            return b""
        e = len(s)
        if length is not None:
            e = offset_of_code_point(s, b, lc)
            if e < 0:
                e = len(s)
        return s[b:e]
    cps = count_code_points(s)
    sc += cps
    if sc < 0:
        return b""
    b = offset_of_code_point(s, 0, sc)
    if b < 0:                    # no parity: bytes that are not UTF-8
        return b""
    e = len(s)
    if length is not None:
        total = _wrap_int(sc + lc) if java_int_wrap else sc + lc
        if total < cps:
            if java_int_wrap and sc + lc >= cps:
                raise SliceOutOfBounds("startCodePoint + lengthCodePoints wraps")
            e = offset_of_code_point(s, b, lc)
            if e < 0:
                e = len(s)
    return s[b:e]


def _lead_len(h):
    return 1 if h < 0x80 else 2 if (h & 0xE0) == 0xC0 else 3 if (h & 0xF0) == 0xE0 else 4 if (h & 0xF8) == 0xF0 else 0


def _decode(s, at, n):
    """the code point of the well-formed n-byte sequence at s[at], or -1"""
    h = s[at]
    if n == 1:
        return h if h < 0x80 else -1
    if _lead_len(h) != n:
        return -1
    c = h & (0x7F >> n)
    for k in range(1, n):
        if not _cont(s[at + k]):
            return -1
        c = (c << 6) | (s[at + k] & 0x3F)
    return c


def _trim(s, left, right):
    """SliceUtf8.leftTrim / rightTrim / trim (M/StringFunctions.java:484-527): whitespace code points off either end.  A sequence that
    is not UTF-8 stops the trim (no parity)"""
    b, e = 0, len(s)
    while left and b < e:
        n = _lead_len(s[b])
        if n == 0 or b + n > e:
            break
        c = _decode(s, b, n)
        if c < 0 or c not in WHITESPACE:
            break
        b += n
    while right and e > b:
        q = e - 1
        while q > b and q > e - 4 and _cont(s[q]):
            q -= 1
        n = e - q
        if _lead_len(s[q]) != n:
            break
        c = _decode(s, q, n)
        if c < 0 or c not in WHITESPACE:
            break
        e = q
    return s[b:e]


def ltrim(s):
    return _trim(s, True, False)


def rtrim(s):
    return _trim(s, False, True)


def trim(s):
    return _trim(s, True, True)


def concat(*pieces):
    """ConcatFunction.concat (ConcatFunction.java:78-95): NULL when a piece is NULL (FAIL_ON_NULL, checked before the call, so an
    oversized piece beside a NULL raises nothing); the running total past MAX_CONCAT_BYTES raises"""
    if any(p is None for p in pieces):
        return None
    total = 0
    for p in pieces:
        total += len(p)
        if total > MAX_CONCAT_BYTES:
            raise ConcatTooLarge("Concatenated string is too large")
    return b"".join(pieces)


FUNCTIONS = {"length": length, "substr": substring, "ltrim": ltrim, "rtrim": rtrim, "trim": trim, "concat": concat}
