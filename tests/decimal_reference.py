"""Exact restatement, on Python ints, of the reference's DECIMAL operators, casts and type rules (M/type/DecimalOperators.java,
M/type/DecimalCasts.java, M/type/DecimalToDecimalCasts.java over S/type/Int128Math.java, S/type/Decimals.java and
S/type/DecimalConversions.java), method by method: the short method where every type is short (precision <= 18), 64-bit wraparound where
the reference does not check, HALF_UP where it rounds.  Values are unscaled ints; types are (precision, scale).

apply() returns the result value or raises DecimalError with the status the device raises."""
from fractions import Fraction

from trino_b200 import abi

P38 = 10 ** 38
MAX_UNSCALED = P38 - 1


class DecimalError(Exception):
    def __init__(self, status):
        super().__init__(status)
        self.status = status


def _overflow():
    return DecimalError(abi.ERR_NUMERIC_VALUE_OUT_OF_RANGE)


def _invalid_cast():
    return DecimalError(abi.ERR_INVALID_CAST_ARGUMENT)


def wrap64(x):
    x &= (1 << 64) - 1
    return x - (1 << 64) if x >= 1 << 63 else x


def wrap128(x):
    x &= (1 << 128) - 1
    return x - (1 << 128) if x >= 1 << 127 else x


def is_long(t):
    return t is not None and t[0] > 18


def java_div(a, b):
    """Java long division (truncates toward zero)"""
    q = abs(a) // abs(b)
    return wrap64(q if (a >= 0) == (b >= 0) else -q)


def java_rem(a, b):
    return wrap64(a - java_div(a, b) * b)


# ---- type rules ---------------------------------------------------------------------------------------------------------------------
def decimal_result_type(op, a, b=None, legacy=False):
    """the result DECIMAL(p, s) of +, -, *, / (M/type/DecimalOperators.java:71-540): with legacy=False the default rules (modelled on
    SQL Server: the exact precision, capped at 38 by giving up scale down to 6), with legacy=True the rules of
    deprecated.legacy-arithmetic-decimal-operators (M/FeaturesConfig.java:535)"""
    ap, as_ = a
    bp, bs = b if b is not None else (0, 0)
    if op in (abi.EX_MOV, abi.EX_NEG):
        return a
    if legacy:
        if op in (abi.EX_ADD, abi.EX_SUB):
            scale = max(as_, bs)
            return min(38, scale + max(ap - as_, bp - bs) + 1), scale
        if op == abi.EX_MUL:
            return min(38, ap + bp), as_ + bs
        if op == abi.EX_DIV:
            return min(38, ap + bs + max(bs - as_, 0)), max(as_, bs)
        raise ValueError(op)
    if op in (abi.EX_ADD, abi.EX_SUB):
        whole = max(ap - as_, bp - bs)          # digits left of the point
        frac = max(as_, bs)
        precision = min(38, whole + frac + 1)
        return precision, min(frac, precision - whole)
    if op == abi.EX_MUL:
        exact_p, exact_s = ap + bp + 1, as_ + bs
    elif op == abi.EX_DIV:
        exact_s = max(6, as_ + bp + 1)
        exact_p = ap - as_ + bs + exact_s
    else:
        raise ValueError(op)
    if exact_p <= 38:
        return exact_p, exact_s
    whole = exact_p - exact_s
    return 38, min(exact_s, 6 if whole > 32 else 38 - whole)


# ---- Int128Math -------------------------------------------------------------------------------------------------------------------
def multiply(a, b):
    """Int128Math.multiply: ArithmeticException when the product's magnitude reaches 2^127"""
    if abs(a) * abs(b) >= 1 << 127:
        raise ArithmeticError
    return a * b


def add128(a, b):
    r = a + b
    if not -(1 << 127) <= r < 1 << 127:
        raise ArithmeticError
    return r


def scale_down_round_up(x, k):
    if k == 0:
        return x
    d = 10 ** k
    q, r = divmod(abs(x), d)
    if 2 * r >= d:
        q += 1
    return -q if x < 0 else q


def rescale(x, k):
    """Int128Math.rescale: up by 10^k (checked, k <= 38), or down HALF_UP"""
    if k > 0:
        if k > 38:
            raise ArithmeticError
        return multiply(x, 10 ** k)
    return scale_down_round_up(x, -k)


def divide_round_up(a, k, b):
    """Int128Math.divideRoundUp(a, k, b, 0): the quotient must fit 128 bits; the increment and the sign wrap as in the reference"""
    if k >= 38:
        raise ArithmeticError
    n = abs(a) * 10 ** max(k, 0)
    d = abs(b)
    q, r = divmod(n, d)
    if q >= 1 << 128:
        raise ArithmeticError
    if ((2 * r) & ((1 << 128) - 1)) >= d:
        q = (q + 1) & ((1 << 128) - 1)
    if (a < 0) != (b < 0):
        q = (-q) & ((1 << 128) - 1)
    return wrap128(q)


def overflows(x):
    return x > MAX_UNSCALED or x < -MAX_UNSCALED


def exceeds_precision(x, p):
    return abs(x) >= 10 ** p


def to_long_exact(x):
    if not -(1 << 63) <= x < 1 << 63:
        raise ArithmeticError
    return x


# ---- operators -------------------------------------------------------------------------------------------------------------------
def add_sub(op, a, at, b, bt, rt):
    sign = 1 if op == abi.EX_ADD else -1
    ar, br = max(0, bt[1] - at[1]), max(0, at[1] - bt[1])
    if not (is_long(at) or is_long(bt) or is_long(rt)):
        return wrap64(a * 10 ** ar + sign * b * 10 ** br)       # addShortShortShort / subtractShortShortShort, unchecked
    try:
        rescale_amount, left = (br, False) if ar == 0 else (ar, True)
        x, y = (rescale(a, rescale_amount), b) if left else (a, rescale(b, rescale_amount))
        s = add128(x, sign * y)
        r = rescale(s, rt[1] - max(at[1], bt[1]))
    except ArithmeticError:
        raise _overflow()
    if overflows(r):
        raise _overflow()
    return r


def mul(a, at, b, bt, rt):
    if not (is_long(at) or is_long(bt)):
        return wrap64(a * b) if not is_long(rt) else a * b      # multiplyShortShortShort (unchecked) / multiplyShortShortLong (exact)
    try:
        r = rescale(multiply(a, b), rt[1] - (at[1] + bt[1]))
    except ArithmeticError:
        raise _overflow()
    if overflows(r):
        raise _overflow()
    return r


def div(a, at, b, bt, rt):
    k = rt[1] - at[1] + bt[1]
    if b == 0:
        raise DecimalError(abi.ERR_DIVISION_BY_ZERO)
    if not (is_long(at) or is_long(bt) or is_long(rt)):
        # divideShortShortShort on Java longs
        if a == 0:
            return 0
        sg = (1 if a > 0 else -1) * (1 if b > 0 else -1)
        ua, ub = wrap64(abs(a)), wrap64(abs(b))
        rs = wrap64(ua * 10 ** k)
        q = java_div(rs, ub)
        rem = wrap64(rs - q * ub)
        if ((rem * 2) & ((1 << 64) - 1)) >= (ub & ((1 << 64) - 1)):
            q = wrap64(q + 1)
        return wrap64(sg * q)
    try:
        q = divide_round_up(a, k, b)
        if not is_long(rt):
            return to_long_exact(q)
    except ArithmeticError:
        raise _overflow()
    if overflows(q):
        raise _overflow()
    return q


def neg(a, at):
    if not is_long(at):
        return wrap64(-a)
    if a == -(1 << 127):
        raise _overflow()
    return -a


def compare(op, a, b):
    return {abi.EX_EQ: a == b, abi.EX_NE: a != b, abi.EX_LT: a < b, abi.EX_LE: a <= b, abi.EX_GT: a > b, abi.EX_GE: a >= b}[op]


# ---- casts -------------------------------------------------------------------------------------------------------------------------
def bigint_to_decimal(v, rt):
    p, s = rt
    if not is_long(rt):
        d = v * 10 ** s
        if not -(1 << 63) <= d < 1 << 63:                      # multiplyExact
            raise _invalid_cast()
        if wrap64(abs(d)) >= 10 ** p:                           # Math.abs wraps at Long.MIN_VALUE
            raise _invalid_cast()
        return d
    try:
        r = multiply(10 ** s, v)
    except ArithmeticError:
        raise _invalid_cast()
    if exceeds_precision(r, p):
        raise _invalid_cast()
    return r


def decimal_to_bigint(v, at):
    t = 10 ** at[1]
    if not is_long(at):
        if v >= 0:
            return java_div(wrap64(v + t // 2), t)
        return wrap64(-java_div(wrap64(-v + t // 2), t))
    try:
        return to_long_exact(rescale(v, -at[1]))
    except ArithmeticError:
        raise _invalid_cast()


def decimal_to_double(v, at):
    if not is_long(at):
        return float(v) / float(10 ** at[1])                    # two roundings, as (double) decimal / tenToScale
    return float(Fraction(v, 10 ** at[1]))                      # the double nearest the exact value


def decimal_to_decimal(v, at, rt):
    (sp, ss), (rp, rs) = at, rt
    if not is_long(at) and not is_long(rt):
        f = 10 ** abs(rs - ss)
        if rs >= ss:
            r = wrap64(v * f)
        else:
            r = java_div(v, f)
            m = java_rem(v, f)
            if v >= 0 and m >= f // 2:
                r += 1
            elif v < 0 and m <= -(f // 2):
                r -= 1
        if wrap64(abs(r)) >= 10 ** rp:
            raise _invalid_cast()
        return r
    if at == rt:
        return v
    try:
        r = rescale(v, rs - ss)
    except ArithmeticError:
        raise _invalid_cast()
    if exceeds_precision(r, rp):
        raise _invalid_cast()
    return wrap64(r) if not is_long(rt) else r


def apply(op, vtype, sig, a, b=None, c=None):
    """one non-NULL DECIMAL instruction: sig = (a, b, c, result) types"""
    at, bt, ct, rt = sig
    if op in (abi.EX_ADD, abi.EX_SUB):
        return add_sub(op, a, at, b, bt, rt)
    if op == abi.EX_MUL:
        return mul(a, at, b, bt, rt)
    if op == abi.EX_DIV:
        return div(a, at, b, bt, rt)
    if op == abi.EX_NEG:
        return neg(a, at)
    if op == abi.EX_MOV:
        return a
    if op in (abi.EX_EQ, abi.EX_NE, abi.EX_LT, abi.EX_LE, abi.EX_GT, abi.EX_GE):
        return compare(op, a, b)
    if op == abi.EX_BETWEEN:
        return b <= a <= c
    if op == abi.EX_CAST_TO_DECIMAL:
        return bigint_to_decimal(a, rt) if vtype == abi.V_BIGINT else decimal_to_decimal(a, at, rt)
    if op == abi.EX_CAST_DECIMAL_TO_BIGINT:
        return decimal_to_bigint(a, at)
    if op == abi.EX_CAST_DECIMAL_TO_DOUBLE:
        return decimal_to_double(a, at)
    raise ValueError(op)
