// device_lib.cuh — device-side building blocks shared by the ahead-of-time kernels (nvcc) and the kernels
// specialised at run time with NVRTC (jit.cu embeds this file verbatim as the prelude of every generated
// translation unit).  It therefore includes NOTHING and defines its own fixed-width integer names under NVRTC.
//
// Contents: column refs, validity/loads, the reference's hash mixers, the per-operation semantics of the
// expression evaluator (one function, folded at compile time when op/type are constants), accumulator
// arithmetic, and the bodies of the fused aggregation kernels (small-group, global, general) as templates over a row program.
#ifndef TG_DEVICE_LIB_CUH
#define TG_DEVICE_LIB_CUH

#ifdef __CUDACC_RTC__
typedef signed char int8_t;
typedef short int16_t;
typedef int int32_t;
typedef long long int64_t;
typedef unsigned char uint8_t;
typedef unsigned short uint16_t;
typedef unsigned int uint32_t;
typedef unsigned long long uint64_t;
#define LLONG_MIN (-9223372036854775807LL - 1)
#endif

#define TGD_MAX_CHANNELS 32

// compact POD view of a fixed-width column
struct ColRef {
    const void* data;
    const uint8_t* validity;   // Arrow bitmap or null
    int32_t type;
    int32_t elem;
};

struct DColumns {
    ColRef cols[TGD_MAX_CHANNELS];
};

// expression opcodes / value types / operand kinds: numerically identical to include/trino_gpu.h
enum {
    TGD_EX_MOV = 0, TGD_EX_ADD = 1, TGD_EX_SUB = 2, TGD_EX_MUL = 3, TGD_EX_DIV = 4, TGD_EX_MOD = 5, TGD_EX_NEG = 6,
    TGD_EX_EQ = 10, TGD_EX_NE = 11, TGD_EX_LT = 12, TGD_EX_LE = 13, TGD_EX_GT = 14, TGD_EX_GE = 15,
    TGD_EX_AND = 20, TGD_EX_OR = 21, TGD_EX_NOT = 22, TGD_EX_IS_NULL = 23, TGD_EX_IS_NOT_NULL = 24, TGD_EX_BETWEEN = 25,
    TGD_EX_CAST_BIGINT_TO_DOUBLE = 30, TGD_EX_CAST_DOUBLE_TO_BIGINT = 31, TGD_EX_CAST_TO_DECIMAL = 32, TGD_EX_CAST_DECIMAL_TO_BIGINT = 33,
    TGD_EX_CAST_DECIMAL_TO_DOUBLE = 34, TGD_EX_IN = 40, TGD_EX_LIKE = 41,
    TGD_EX_LENGTH = 50, TGD_EX_SUBSTR = 51, TGD_EX_LTRIM = 52, TGD_EX_RTRIM = 53, TGD_EX_TRIM = 54, TGD_EX_CONCAT = 55,
    TGD_EX_IF = 60, TGD_EX_COALESCE = 61
};
// TGD_V_DECIMAL_LONG is internal: the output-column type of a long DECIMAL projection (16-byte cells: high word, low word)
enum { TGD_V_BIGINT = 0, TGD_V_DOUBLE = 1, TGD_V_BOOLEAN = 2, TGD_V_VARCHAR = 3, TGD_V_DECIMAL = 4, TGD_V_DECIMAL_LONG = 5 };
// TG_ERR_BIT_CONCAT_TOO_LARGE: a concatenation past 1 MiB (INVALID_FUNCTION_ARGUMENT).  The interpreter keeps 4 bits of error per temp and
// holds it there as TG_ERR_CODE_CONCAT (15, never a single bit); vm_temp_error turns it back into the bit.
enum { TG_ERR_BIT_OVERFLOW = 1, TG_ERR_BIT_DIV_ZERO = 2, TG_ERR_BIT_INVALID_CAST = 4, TG_ERR_BIT_DECIMAL_OVERFLOW = 8, TG_ERR_BIT_CONCAT_TOO_LARGE = 16 };
#define TG_ERR_CODE_CONCAT 15u
#define TGD_MAX_CONCAT_BYTES (1 << 20)    // DEFAULT_MAX_PAGE_SIZE_IN_BYTES (S/block/PageBuilderStatus.java:22)

// The reference's method for one DECIMAL instruction, fixed at create from its signature (expr.cu decimal_method).  la / lb / lc / lr:
// operand a / b / c and the result are long decimals (a BIGINT operand or a non-DECIMAL result: 0).  k0..k2, m0, m1: see vm_apply_dec.
// hi: the high words of long constant operands a, b, c.
struct DDec {
    int8_t is_dec, la, lb, lc, lr, pad0, pad1, pad2;
    int32_t k0, k1, k2, pad3;
    long long m0, m1;
    long long hi[3];
};

enum AccKind {
    ACC_ROWS = 0, ACC_NONNULL = 1, ACC_SUM_F64 = 2, ACC_SUM_I64_LO = 3, ACC_SUM_I64_HI = 4,
    ACC_MIN_F64 = 5, ACC_MAX_F64 = 6, ACC_MIN_I64 = 7, ACC_MAX_I64 = 8, ACC_SUM_F64_FROM_I64 = 9,
    // VarianceState {count, mean, m2} as three consecutive words (count, mean bits, m2 bits): the first word's kind names the input
    // (a DOUBLE value, a BIGINT-family value, or an intermediate state row), the other two are ACC_VAR_MEAN / ACC_VAR_M2
    ACC_VAR_F64 = 10, ACC_VAR_I64 = 11, ACC_VAR_STATE = 12, ACC_VAR_MEAN = 13, ACC_VAR_M2 = 14
};

#define TGD_EMPTY_KEY 0x8000000000000000ULL
#define TGD_NO_ROW 0x7FFFFFFFFFFFFFFFLL
#define TGD_S_THREADS 256

// per-CTA partial results of the small-group aggregation kernel
struct SmallOut {
    unsigned long long* blk_keys;    // [grid][L]
    long long* blk_first;            // [grid][L+2]
    unsigned long long* blk_acc;     // [grid][L+2][A]
    int* overflow;
    unsigned int* err;
};

#define TGD_MAX_STR_OUTS 8
#define TGD_MAX_PIECES 8          // pieces of one concatenation
#define TGD_MAX_PIECE_SLOTS 16    // captured pieces of one program
#define TGD_SRC_NONE (-2147483647 - 1)

// computed projection outputs of the filter/project kernels
struct OutCols {
    int32_t count;
    int32_t temp[TGD_MAX_CHANNELS];
    int32_t vtype[TGD_MAX_CHANNELS];
    void* data[TGD_MAX_CHANNELS];
    uint8_t* nullmap[TGD_MAX_CHANNELS];   // 1 byte per row, 1 = NULL
    // pass-through projections copied by the fused (chunked) projection kernel; nullmap == nullptr: the input has no NULLs
    int32_t pass_count;
    void* pass_data[TGD_MAX_CHANNELS];
    uint8_t* pass_nullmap[TGD_MAX_CHANNELS];
    // VARCHAR projections (DProgram::str_out[k]): per output row and piece an (int32 begin, int32 len) descriptor into the piece's
    // source, [row][piece]; the byte assembly kernel turns them into a UTF8 column
    int32_t str_count;
    void* str_desc[TGD_MAX_STR_OUTS];
    uint8_t* str_nullmap[TGD_MAX_STR_OUTS];
};

// ---- VARCHAR operands of FilterAndProject programs ------------------------------------------------------------------------
// The UTF8 channels a program's string operations read, in slots: slot k is channel DProgram::str_channel[k].  Kept apart from
// ColRef / DColumns, which every kernel of the library takes by value.
#define TGD_MAX_STR_CHANNELS 8
struct StrCols {
    const int32_t* offsets[TGD_MAX_STR_CHANNELS];
    const uint8_t* bytes[TGD_MAX_STR_CHANNELS];
};

// A constant LIKE pattern as LikeMatcher.compile(pattern, escape, optimize = true) leaves it (M/likematcher/LikeMatcher.java:58-153):
// length bounds, a constant prefix and suffix, and a matcher for the middle.  FJS: literal terms found in order (bytewise);
// DFA: the byte-level automaton of DenseDfaMatcher (`_` and `%` consume whole, well-formed UTF-8 sequences); NFA: NfaMatcher, whose `_`
// consumes one decoded code point and whose literals are UTF-16 code units.  DFA and NFA run as one 64-bit mask of positions:
// position p is followed by `_` (any_mask), by a literal (lit_pos / lit_val), and may carry a `%` loop (loop_mask); `accept` is the last.
enum { TGD_LIKE_NONE = 0, TGD_LIKE_FJS = 1, TGD_LIKE_DFA = 2, TGD_LIKE_NFA = 3 };
#define TGD_LIKE_BYTES 1024
#define TGD_LIKE_TERMS 32
#define TGD_LIKE_LITS 64
struct DLike {
    int32_t min_size, max_size;                // max_size < 0: unbounded
    int32_t prefix_len, suffix_len;            // bytes[0, prefix_len) and bytes[prefix_len, prefix_len + suffix_len)
    int32_t kind;                              // TGD_LIKE_*
    int32_t exact;                             // the middle must match to its end
    int32_t num_terms;                         // FJS
    int32_t accept;                            // DFA / NFA
    int32_t num_lits;
    int32_t pad;
    unsigned long long any_mask, loop_mask;
    int32_t term_off[TGD_LIKE_TERMS], term_len[TGD_LIKE_TERMS];
    int32_t lit_pos[TGD_LIKE_LITS], lit_val[TGD_LIKE_LITS];
    uint8_t bytes[TGD_LIKE_BYTES];
};

#if defined(__CUDACC__)

struct StrRef {
    const uint8_t* p;
    int32_t len;
};

__device__ __forceinline__ StrRef tg_str(const StrCols& s, int slot, int64_t row)
{
    const int32_t b = s.offsets[slot][row], e = s.offsets[slot][row + 1];
    return StrRef{s.bytes[slot] + b, e - b};
}

// the n (<= 8) bytes at p as a little-endian word, zero above them.  Only the aligned 8-byte words that hold one of the n bytes are
// read (one, or two joined by a shift), so a string at the very end of its buffer is never read past the word it ends in.
__device__ __forceinline__ unsigned long long tg_ld_bytes(const uint8_t* p, int n)
{
    if (n <= 0) return 0ULL;
    const unsigned long long a = (unsigned long long)p;
    const unsigned long long* w = (const unsigned long long*)(a & ~7ULL);
    const int sh = (int)(a & 7ULL);
    unsigned long long v = __ldg(w) >> (sh * 8);
    if (sh + n > 8) v |= __ldg(w + 1) << ((8 - sh) * 8);
    return n >= 8 ? v : v & ((1ULL << (n * 8)) - 1ULL);
}

__device__ __forceinline__ unsigned long long tg_bswap64(unsigned long long x)
{
    const unsigned int lo = (unsigned int)x, hi = (unsigned int)(x >> 32);
    return ((unsigned long long)__byte_perm(lo, 0, 0x0123) << 32) | __byte_perm(hi, 0, 0x0123);
}

__device__ __forceinline__ bool tg_str_eq(StrRef a, StrRef b)
{
    if (a.len != b.len) return false;
    for (int i = 0; i < a.len; i += 8) {
        const int n = a.len - i < 8 ? a.len - i : 8;
        if (tg_ld_bytes(a.p + i, n) != tg_ld_bytes(b.p + i, n)) return false;
    }
    return true;
}

// Slice.compareTo: unsigned bytes, lexicographic, a proper prefix first.  Byte-swapped 8-byte words compare as unsigned integers.
__device__ __forceinline__ int tg_str_cmp(StrRef a, StrRef b)
{
    const int m = a.len < b.len ? a.len : b.len;
    for (int i = 0; i < m; i += 8) {
        const int n = m - i < 8 ? m - i : 8;
        const unsigned long long x = tg_bswap64(tg_ld_bytes(a.p + i, n)), y = tg_bswap64(tg_ld_bytes(b.p + i, n));
        if (x != y) return x < y ? -1 : 1;
    }
    return a.len < b.len ? -1 : a.len > b.len ? 1 : 0;
}

__device__ __forceinline__ bool tg_str_cmp_op(int op, StrRef a, StrRef b)
{
    if (op == TGD_EX_EQ) return tg_str_eq(a, b);
    if (op == TGD_EX_NE) return !tg_str_eq(a, b);
    const int c = tg_str_cmp(a, b);
    switch (op) {
        case TGD_EX_LT: return c < 0;
        case TGD_EX_LE: return c <= 0;
        case TGD_EX_GT: return c > 0;
        default: return c >= 0;
    }
}

// ---- string functions (M/operator/scalar/StringFunctions.java over airlift's SliceUtf8) -----------------------------------------------
// Code points are counted as SliceUtf8.countCodePoints counts them: every byte that is not a continuation byte (10xxxxxx).  On bytes that
// are not UTF-8 the results are deterministic and stay inside the string, with no parity claimed.
__device__ __forceinline__ bool tg_utf8_cont(uint8_t b) { return (b & 0xC0) == 0x80; }

__device__ __forceinline__ long long tg_utf8_count(StrRef s)
{
    long long n = 0;
    int i = 0;
    for (; i + 8 <= s.len; i += 8) {
        const unsigned long long w = tg_ld_bytes(s.p + i, 8);
        // a continuation byte has bit 7 set and bit 6 clear
        n += 8 - __popcll(w & ~(w << 1) & 0x8080808080808080ULL);
    }
    for (; i < s.len; i++) n += tg_utf8_cont(s.p[i]) ? 0 : 1;
    return n;
}

// SliceUtf8.offsetOfCodePoint(s, position, count): the byte offset of the count-th code point after `position`, or -1 when the string ends
// first.  A code point starts at a byte that is not a continuation byte.
__device__ __forceinline__ int tg_utf8_offset(StrRef s, int position, int count)
{
    if ((long long)s.len - position <= count) return -1;
    int i = position;
    for (int k = 0; k < count; k++) {
        i++;
        while (i < s.len && tg_utf8_cont(s.p[i])) i++;
        if (i >= s.len) return -1;
    }
    return i;
}

__device__ __forceinline__ int tg_sat_int(long long v) { return v > 2147483647LL ? 2147483647 : v < -2147483648LL ? (-2147483647 - 1) : (int)v; }

// StringFunctions.substring(utf8, start) (has_len = false, :284-320) and substring(utf8, start, length) (:331-378).  Where Java's
// startCodePoint + lengthCodePoints wraps (a negative start with a length near INT_MAX) the reference fails inside Slice.slice; this
// returns the suffix, as the unwrapped sum would.
__device__ __forceinline__ StrRef tg_substr(StrRef s, long long start, bool has_len, long long length)
{
    const StrRef empty{s.p, 0};
    if (start == 0 || (has_len && length <= 0) || s.len == 0) return empty;
    int sc = tg_sat_int(start);
    const int lc = has_len ? tg_sat_int(length) : 0;
    int b, e = s.len;
    if (sc > 0) {
        b = tg_utf8_offset(s, 0, sc - 1);
        if (b < 0) return empty;
        if (has_len) {
            e = tg_utf8_offset(s, b, lc);
            if (e < 0) e = s.len;
        }
    }
    else {
        const long long cps = tg_utf8_count(s);
        const long long st = (long long)sc + cps;
        if (st < 0) return empty;
        b = tg_utf8_offset(s, 0, (int)st);
        if (b < 0) return empty;
        if (has_len && st + lc < cps) {
            e = tg_utf8_offset(s, b, lc);
            if (e < 0) e = s.len;
        }
    }
    return StrRef{s.p + b, e - b};
}

// Character.isWhitespace: the space separators but U+00A0, U+2007 and U+202F, the line and paragraph separators, U+0009-U+000D and
// U+001C-U+001F
__device__ __forceinline__ bool tg_is_whitespace(unsigned int c)
{
    if (c <= 0x20) return c == 0x20 || (c >= 0x09 && c <= 0x0D) || (c >= 0x1C && c <= 0x1F);
    if (c < 0x1680) return false;
    return c == 0x1680 || (c >= 0x2000 && c <= 0x200A && c != 0x2007) || c == 0x2028 || c == 0x2029 || c == 0x205F || c == 0x3000;
}

// the code point of the well-formed sequence of n bytes at p (n = 1..4), or -1 when it is not one
__device__ __forceinline__ int tg_utf8_decode(const uint8_t* p, int n)
{
    const unsigned int h = p[0];
    if (n == 1) return h < 0x80 ? (int)h : -1;
    const unsigned int want = n == 2 ? 0xC0u : n == 3 ? 0xE0u : 0xF0u, mask = n == 2 ? 0xE0u : n == 3 ? 0xF0u : 0xF8u;
    if ((h & mask) != want) return -1;
    unsigned int c = h & (0x7Fu >> n);
    for (int k = 1; k < n; k++) {
        if (!tg_utf8_cont(p[k])) return -1;
        c = (c << 6) | (p[k] & 0x3Fu);
    }
    return (int)c;
}

__device__ __forceinline__ int tg_utf8_lead_len(uint8_t h) { return h < 0x80 ? 1 : (h & 0xE0) == 0xC0 ? 2 : (h & 0xF0) == 0xE0 ? 3 : (h & 0xF8) == 0xF0 ? 4 : 0; }

// SliceUtf8.leftTrim / rightTrim / trim: whitespace code points off either end; a sequence that is not UTF-8 stops the trim
__device__ __forceinline__ StrRef tg_trim(StrRef s, bool left, bool right)
{
    int b = 0, e = s.len;
    if (left) {
        while (b < e) {
            const int n = tg_utf8_lead_len(s.p[b]);
            if (n == 0 || b + n > e) break;
            const int c = tg_utf8_decode(s.p + b, n);
            if (c < 0 || !tg_is_whitespace((unsigned int)c)) break;
            b += n;
        }
    }
    if (right) {
        while (e > b) {
            int q = e - 1;
            while (q > b && q > e - 4 && tg_utf8_cont(s.p[q])) q--;
            const int n = e - q;
            if (tg_utf8_lead_len(s.p[q]) != n) break;
            const int c = tg_utf8_decode(s.p + q, n);
            if (c < 0 || !tg_is_whitespace((unsigned int)c)) break;
            e = q;
        }
    }
    return StrRef{s.p + b, e - b};
}

// The error of a call over operands a, b, c (BytecodeUtils.java:303-306): the operands' errors in order, stopping at the first NULL one,
// then its own
__device__ __forceinline__ uint32_t vm_error_call(bool an, uint32_t ea, bool bn, uint32_t eb, uint32_t ec, bool any_null, uint32_t own)
{
    if (ea || an) return ea;
    if (eb || bn) return eb;
    if (ec) return ec;
    return any_null ? 0u : own;
}

__device__ __forceinline__ bool tg_bytes_eq(const uint8_t* p, const uint8_t* q, int n)
{
    for (int i = 0; i < n; i++)
        if (p[i] != q[i]) return false;
    return true;
}

// FjsMatcher: every term, in order, at its leftmost occurrence after the previous one
__device__ __forceinline__ bool tg_like_fjs(const DLike& L, const uint8_t* p, int len)
{
    int start = 0;
    for (int t = 0; t < L.num_terms; t++) {
        const uint8_t* term = L.bytes + L.term_off[t];
        const int tl = L.term_len[t];
        if (start == len) return false;
        int at = -1;
        for (int i = start; i + tl <= len; i++)
            if (p[i] == term[0] && tg_bytes_eq(p + i + 1, term + 1, tl - 1)) { at = i; break; }
        if (at < 0) return false;
        start = at + tl;
    }
    return !L.exact || start == len;
}

// positions followed by a literal equal to v
__device__ __forceinline__ unsigned long long tg_like_lits(const DLike& L, int v)
{
    unsigned long long m = 0;
    for (int k = 0; k < L.num_lits; k++)
        if (L.lit_val[k] == v) m |= 1ULL << L.lit_pos[k];
    return m;
}

// DenseDfaMatcher's language, simulated over bytes: D = positions reached, P1..P3 = positions reached once 1..3 more continuation bytes
// (10xxxxxx) complete the UTF-8 sequence a `_` or a `%` is consuming
__device__ __forceinline__ bool tg_like_dfa(const DLike& L, const uint8_t* p, int len)
{
    const unsigned long long acc = 1ULL << L.accept;
    unsigned long long D = 1, P1 = 0, P2 = 0, P3 = 0;
    for (int i = 0; i < len; i++) {
        const int b = p[i];
        const unsigned long long step = ((D & L.any_mask) << 1) | (D & L.loop_mask);
        unsigned long long nd = (D & tg_like_lits(L, b)) << 1, n1 = 0, n2 = 0, n3 = 0;
        if (b < 0x80) nd |= step;
        else if (b < 0xC0) { nd |= P1; n1 = P2; n2 = P3; }
        else if (b < 0xE0) n1 = step;
        else if (b < 0xF0) n2 = step;
        else if (b < 0xF8) n3 = step;
        D = nd; P1 = n1; P2 = n2; P3 = n3;
        if ((D | P1 | P2 | P3) == 0) return false;
        if (!L.exact && (D & acc)) return true;
    }
    return (D & acc) != 0;
}

// NfaMatcher: code points decoded as it decodes them (lead byte and length only; a truncated or stray byte fails the match)
__device__ __forceinline__ bool tg_like_nfa(const DLike& L, const uint8_t* p, int len)
{
    const unsigned long long acc = 1ULL << L.accept;
    unsigned long long D = 1;
    int i = 0;
    while (i < len) {
        const int h = p[i];
        int cp;
        if (h < 0x80) { cp = h; i += 1; }
        else if ((h & 0xE0) == 0xC0 && i + 1 < len) { cp = ((h & 0x1F) << 6) | (p[i + 1] & 0x3F); i += 2; }
        else if ((h & 0xF0) == 0xE0 && i + 2 < len) { cp = ((h & 0x0F) << 12) | ((p[i + 1] & 0x3F) << 6) | (p[i + 2] & 0x3F); i += 3; }
        else if ((h & 0xF8) == 0xF0 && i + 3 < len) {
            cp = ((h & 0x07) << 18) | ((p[i + 1] & 0x3F) << 12) | ((p[i + 2] & 0x3F) << 6) | (p[i + 3] & 0x3F);
            i += 4;
        }
        else return false;
        D = ((D & (L.any_mask | tg_like_lits(L, cp))) << 1) | (D & L.loop_mask);
        if (D == 0) return false;
        if (!L.exact && (D & acc)) return true;
    }
    return (D & acc) != 0;
}

__device__ __forceinline__ bool tg_like_middle(const DLike& L, const uint8_t* p, int len)
{
    switch (L.kind) {
        case TGD_LIKE_FJS: return tg_like_fjs(L, p, len);
        case TGD_LIKE_DFA: return tg_like_dfa(L, p, len);
        case TGD_LIKE_NFA: return tg_like_nfa(L, p, len);
        default: return true;
    }
}

// LikeMatcher.match (M/likematcher/LikeMatcher.java:160-183)
__device__ __forceinline__ bool tg_like(const DLike& L, StrRef s)
{
    if (s.len < L.min_size || (L.max_size >= 0 && s.len > L.max_size)) return false;
    if (!tg_bytes_eq(s.p, L.bytes, L.prefix_len)) return false;
    if (!tg_bytes_eq(s.p + s.len - L.suffix_len, L.bytes + L.prefix_len, L.suffix_len)) return false;
    return tg_like_middle(L, s.p + L.prefix_len, s.len - L.prefix_len - L.suffix_len);
}

__device__ __forceinline__ bool tg_valid(const uint8_t* validity, int64_t i)
{
    return validity == nullptr || ((validity[i >> 3] >> (i & 7)) & 1);
}

// sign-extending load of any fixed-width integer column element / raw bits of FLOAT64
__device__ __forceinline__ int64_t tg_load_i64(const ColRef& c, int64_t i)
{
    switch (c.elem) {
        case 8: return ((const int64_t*)c.data)[i];
        case 4: return ((const int32_t*)c.data)[i];
        case 2: return ((const int16_t*)c.data)[i];
        default: return ((const int8_t*)c.data)[i];
    }
}

template <int ELEM>
__device__ __forceinline__ int64_t tg_load_elem(const void* data, int64_t i)
{
    if (ELEM == 8) return ((const int64_t*)data)[i];
    if (ELEM == 4) return ((const int32_t*)data)[i];
    if (ELEM == 2) return ((const int16_t*)data)[i];
    return ((const int8_t*)data)[i];
}

__device__ __forceinline__ uint64_t tgd_murmur3_mix(uint64_t x)
{
    x ^= x >> 33; x *= 0xff51afd7ed558ccdULL; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ULL; x ^= x >> 33;
    return x;
}

// ---- expression semantics ---------------------------------------------------------------------------
struct Value {
    int64_t bits;
    bool is_null;
};

__device__ __forceinline__ bool vm_cmp(int op, int vtype, int64_t a, int64_t b)
{
    if (vtype == TGD_V_DOUBLE) {
        double x = __longlong_as_double(a), y = __longlong_as_double(b);
        switch (op) {
            case TGD_EX_EQ: return x == y;
            case TGD_EX_NE: return !(x == y);
            case TGD_EX_LT: return x < y;
            case TGD_EX_LE: return x <= y;
            case TGD_EX_GT: return x > y;
            default: return x >= y;
        }
    }
    switch (op) {
        case TGD_EX_EQ: return a == b;
        case TGD_EX_NE: return a != b;
        case TGD_EX_LT: return a < b;
        case TGD_EX_LE: return a <= b;
        case TGD_EX_GT: return a > b;
        default: return a >= b;
    }
}

// One operation of the evaluator (everything except IN, whose constant list lives with the caller).
// SQL three-valued logic; checked BIGINT arithmetic (Math.*Exact); IEEE DOUBLE arithmetic through the
// *_rn intrinsics, which are never contracted into FMAs.
__device__ __forceinline__ Value vm_apply(int op, int vtype, Value a, Value b, Value c, uint32_t* err)
{
    Value res;
    int64_t r = 0;
    bool rn = false;
    const bool dbl = vtype == TGD_V_DOUBLE;
    switch (op) {
        case TGD_EX_MOV: r = a.bits; rn = a.is_null; break;
        case TGD_EX_ADD: case TGD_EX_SUB: case TGD_EX_MUL: case TGD_EX_DIV: case TGD_EX_MOD: {
            rn = a.is_null || b.is_null;
            if (rn) break;
            if (dbl) {
                double x = __longlong_as_double(a.bits), y = __longlong_as_double(b.bits), z;
                if (op == TGD_EX_ADD) z = __dadd_rn(x, y);
                else if (op == TGD_EX_SUB) z = __dsub_rn(x, y);
                else if (op == TGD_EX_MUL) z = __dmul_rn(x, y);
                else if (op == TGD_EX_DIV) z = __ddiv_rn(x, y);
                else z = fmod(x, y);
                r = __double_as_longlong(z);
            }
            else {
                long long x = a.bits, y = b.bits, z = 0;
                if (op == TGD_EX_ADD) {
                    z = (long long)((unsigned long long)x + (unsigned long long)y);
                    if (((x ^ z) & (y ^ z)) < 0) *err |= TG_ERR_BIT_OVERFLOW;
                }
                else if (op == TGD_EX_SUB) {
                    z = (long long)((unsigned long long)x - (unsigned long long)y);
                    if (((x ^ y) & (x ^ z)) < 0) *err |= TG_ERR_BIT_OVERFLOW;
                }
                else if (op == TGD_EX_MUL) {
                    z = (long long)((unsigned long long)x * (unsigned long long)y);
                    long long hi = __mul64hi(x, y);
                    if (hi != (z >> 63)) *err |= TG_ERR_BIT_OVERFLOW;
                }
                else {
                    if (y == 0) { *err |= TG_ERR_BIT_DIV_ZERO; }
                    else if (y == -1) {
                        if (op == TGD_EX_DIV) {
                            if (x == LLONG_MIN) *err |= TG_ERR_BIT_OVERFLOW;
                            else z = -x;
                        }
                        else z = 0;
                    }
                    else z = op == TGD_EX_DIV ? x / y : x % y;
                }
                r = z;
            }
            break;
        }
        case TGD_EX_NEG:
            rn = a.is_null;
            if (rn) break;
            if (dbl) r = a.bits ^ (long long)0x8000000000000000ULL;
            else {
                if (a.bits == LLONG_MIN) *err |= TG_ERR_BIT_OVERFLOW;
                r = (long long)(0ULL - (unsigned long long)a.bits);
            }
            break;
        case TGD_EX_EQ: case TGD_EX_NE: case TGD_EX_LT: case TGD_EX_LE: case TGD_EX_GT: case TGD_EX_GE:
            rn = a.is_null || b.is_null;
            if (!rn) r = vm_cmp(op, vtype, a.bits, b.bits) ? 1 : 0;
            break;
        case TGD_EX_AND: {
            bool af = !a.is_null && a.bits == 0, bf = !b.is_null && b.bits == 0;
            if (af || bf) { r = 0; rn = false; }
            else if (a.is_null || b.is_null) rn = true;
            else r = 1;
            break;
        }
        case TGD_EX_OR: {
            bool at = !a.is_null && a.bits != 0, bt = !b.is_null && b.bits != 0;
            if (at || bt) { r = 1; rn = false; }
            else if (a.is_null || b.is_null) rn = true;
            else r = 0;
            break;
        }
        case TGD_EX_NOT: rn = a.is_null; r = a.bits == 0 ? 1 : 0; break;
        case TGD_EX_IS_NULL: r = a.is_null ? 1 : 0; break;
        case TGD_EX_IS_NOT_NULL: r = a.is_null ? 0 : 1; break;
        case TGD_EX_BETWEEN: {
            // value BETWEEN min AND max  ==  value >= min AND value <= max (Kleene AND)
            bool n1 = a.is_null || b.is_null, n2 = a.is_null || c.is_null;
            bool v1 = !n1 && vm_cmp(TGD_EX_GE, vtype, a.bits, b.bits);
            bool v2 = !n2 && vm_cmp(TGD_EX_LE, vtype, a.bits, c.bits);
            bool f1 = !n1 && !v1, f2 = !n2 && !v2;
            if (f1 || f2) r = 0;
            else if (n1 || n2) rn = true;
            else r = 1;
            break;
        }
        case TGD_EX_CAST_BIGINT_TO_DOUBLE:
            rn = a.is_null;
            r = __double_as_longlong((double)a.bits);
            break;
        case TGD_EX_CAST_DOUBLE_TO_BIGINT: {
            rn = a.is_null;
            if (rn) break;
            double x = __longlong_as_double(a.bits);
            // DoubleMath.roundToLong(x, HALF_UP): NaN / out of range is INVALID_CAST_ARGUMENT (M/type/DoubleOperators.java:159-167)
            if (!(x >= -9.2233720368547758e18 && x < 9.2233720368547758e18)) *err |= TG_ERR_BIT_INVALID_CAST;
            else r = llround(x);
            break;
        }
        // both operands were evaluated; the select keeps one (its value and NULL flag)
        case TGD_EX_IF: {
            const bool t = !a.is_null && a.bits != 0;
            r = t ? b.bits : c.bits;
            rn = t ? b.is_null : c.is_null;
            break;
        }
        case TGD_EX_COALESCE: r = a.is_null ? b.bits : a.bits; rn = a.is_null && b.is_null; break;
        default: break;
    }
    res.bits = r;
    res.is_null = rn;
    return res;
}

// The error the result of one instruction carries (one TG_ERR_BIT_* or 0): the first error, in the reference's evaluation order,
// of the operands it evaluates, otherwise its own (`own`, what vm_apply raised).  ea / eb / ec are the errors the operands carry
// (a column or constant never carries one).  Only the errors carried by the filter and by the outputs are raised, so an operand
// the reference never evaluates raises nothing:
//   AND / OR: the left operand's error; none when the left operand is FALSE / TRUE (AndCodeGenerator.java:56-75,
//             OrCodeGenerator.java:69-70); otherwise the right operand's
//   BETWEEN:  the value's error; none when the value is NULL; min's; none when min <= value is FALSE; max's
//             (BetweenCodeGenerator.java:62-80)
//   calls:    the operands' errors in order, stopping at the first NULL operand (BytecodeUtils.java:303-306), then their own
//   IS [NOT] NULL, MOV: the operand's
//   IF:       the condition's; then the THEN operand's when the condition is TRUE, otherwise the ELSE operand's
//             (IfCodeGenerator.java:47-62: a NULL condition counts as FALSE)
//   COALESCE: the first operand's; none when it is non-NULL, otherwise the second's (CoalesceCodeGenerator.java:45-75)
__device__ __forceinline__ uint32_t vm_error(int op, int vtype, Value a, uint32_t ea, Value b, uint32_t eb, Value c, uint32_t ec, uint32_t own)
{
    if (ea) return ea;
    switch (op) {
        case TGD_EX_AND: return (!a.is_null && a.bits == 0) ? 0 : eb;
        case TGD_EX_OR: return (!a.is_null && a.bits != 0) ? 0 : eb;
        case TGD_EX_IF: return (!a.is_null && a.bits != 0) ? eb : ec;
        case TGD_EX_COALESCE: return a.is_null ? eb : 0;
        case TGD_EX_BETWEEN:
            if (a.is_null) return 0;
            if (eb) return eb;
            if (!b.is_null && !vm_cmp(TGD_EX_LE, vtype, b.bits, a.bits)) return 0;
            return ec;
        case TGD_EX_ADD: case TGD_EX_SUB: case TGD_EX_MUL: case TGD_EX_DIV: case TGD_EX_MOD:
        case TGD_EX_EQ: case TGD_EX_NE: case TGD_EX_LT: case TGD_EX_LE: case TGD_EX_GT: case TGD_EX_GE:
            if (a.is_null) return 0;
            return eb ? eb : own;
        default: return own;   // one operand
    }
}

#endif  // __CUDACC__

// ---- DECIMAL: 128-bit two's-complement arithmetic over (high, low) 64-bit words --------------------------------------------------------
// Int128Math (S/type/Int128Math.java) and Decimals.overflows (S/type/Decimals.java:314-335) restated.  Written over word pairs so that NVRTC
// needs no 128-bit integer type; host and device share them (the host computes the constants of a program with them).
#if defined(__CUDACC__)
#define TGD_HD __host__ __device__ __forceinline__
#else
#define TGD_HD inline
#endif

struct U128 {
    unsigned long long hi, lo;
};

TGD_HD unsigned long long tgd_umulhi(unsigned long long a, unsigned long long b)
{
#if defined(__CUDA_ARCH__)
    return __umul64hi(a, b);
#else
    return (unsigned long long)(((unsigned __int128)a * b) >> 64);
#endif
}

TGD_HD int tgd_clz64(unsigned long long x)
{
#if defined(__CUDA_ARCH__)
    return __clzll((long long)x);
#else
    return x ? __builtin_clzll(x) : 64;
#endif
}

TGD_HD U128 u128_sx(long long v) { return U128{(unsigned long long)(v >> 63), (unsigned long long)v}; }
TGD_HD bool u128_is_neg(U128 x) { return (long long)x.hi < 0; }
TGD_HD bool u128_is_zero(U128 x) { return (x.hi | x.lo) == 0; }
TGD_HD U128 u128_negate(U128 x) { return U128{~x.hi + (x.lo == 0 ? 1ULL : 0ULL), 0ULL - x.lo}; }
TGD_HD U128 u128_add(U128 a, U128 b)
{
    const unsigned long long lo = a.lo + b.lo;
    return U128{a.hi + b.hi + (lo < a.lo ? 1ULL : 0ULL), lo};
}
TGD_HD U128 u128_sub(U128 a, U128 b) { return U128{a.hi - b.hi - (a.lo < b.lo ? 1ULL : 0ULL), a.lo - b.lo}; }
TGD_HD int u128_cmp(U128 a, U128 b)     // signed
{
    if (a.hi != b.hi) return (long long)a.hi < (long long)b.hi ? -1 : 1;
    return a.lo < b.lo ? -1 : a.lo > b.lo ? 1 : 0;
}
TGD_HD int u128_ucmp(U128 a, U128 b)
{
    if (a.hi != b.hi) return a.hi < b.hi ? -1 : 1;
    return a.lo < b.lo ? -1 : a.lo > b.lo ? 1 : 0;
}
TGD_HD U128 u128_abs(U128 x) { return u128_is_neg(x) ? u128_negate(x) : x; }    // the magnitude, as an unsigned value
TGD_HD int u128_bits(U128 x) { return x.hi ? 128 - tgd_clz64(x.hi) : 64 - tgd_clz64(x.lo); }
TGD_HD U128 u128_shr(U128 x, int s)     // logical, 0 <= s < 128
{
    if (s == 0) return x;
    if (s >= 64) return U128{0ULL, x.hi >> (s - 64)};
    return U128{x.hi >> s, (x.lo >> s) | (x.hi << (64 - s))};
}
TGD_HD U128 u128_shl(U128 x, int s)     // 0 <= s < 128
{
    if (s == 0) return x;
    if (s >= 64) return U128{x.lo << (s - 64), 0ULL};
    return U128{(x.hi << s) | (x.lo >> (64 - s)), x.lo << s};
}
TGD_HD bool u128_bit(U128 x, int i) { return i >= 64 ? ((x.hi >> (i - 64)) & 1ULL) != 0 : ((x.lo >> i) & 1ULL) != 0; }
TGD_HD U128 u128_low_bits(U128 x, int n)     // bits [0, n), 0 <= n < 128
{
    if (n >= 64) return U128{n == 64 ? 0ULL : x.hi & ((1ULL << (n - 64)) - 1ULL), x.lo};
    return U128{0ULL, n == 0 ? 0ULL : x.lo & ((1ULL << n) - 1ULL)};
}
// x << s over 256 bits (hi:lo), 0 <= s < 256
TGD_HD void u128_shl_wide(U128 x, int s, U128* hi, U128* lo)
{
    if (s >= 128) { *hi = u128_shl(x, s - 128); *lo = U128{0ULL, 0ULL}; return; }
    *lo = u128_shl(x, s);
    *hi = s == 0 ? U128{0ULL, 0ULL} : u128_shr(x, 128 - s);
}

// 10^k, 0 <= k <= 38 (folds to immediates when k is a constant)
TGD_HD U128 tgd_pow10(int k)
{
    U128 r{0ULL, 1ULL};
    for (int i = 0; i < k; i++) r = U128{r.hi * 10ULL + tgd_umulhi(r.lo, 10ULL), r.lo * 10ULL};
    return r;
}

// magnitudes a * b; true when the product is 2^127 or more (Int128Math.multiply's overflow rule: the signed result would not fit)
TGD_HD bool u128_umul_ovf(U128 a, U128 b, U128* r)
{
    const unsigned long long h0 = tgd_umulhi(a.lo, b.lo);
    bool ovf = (a.hi != 0 && b.hi != 0) || tgd_umulhi(a.lo, b.hi) != 0 || tgd_umulhi(a.hi, b.lo) != 0;
    const unsigned long long s1 = h0 + a.lo * b.hi;
    ovf = ovf || s1 < h0;
    const unsigned long long s2 = s1 + a.hi * b.lo;
    ovf = ovf || s2 < s1 || (s2 >> 63) != 0;
    *r = U128{s2, a.lo * b.lo};
    return ovf;
}

// checked signed multiply (Int128Math.multiply)
TGD_HD bool u128_mul_ovf(U128 a, U128 b, U128* r)
{
    const bool neg = u128_is_neg(a) != u128_is_neg(b);
    U128 m;
    const bool ovf = u128_umul_ovf(u128_abs(a), u128_abs(b), &m);
    *r = neg ? u128_negate(m) : m;
    return ovf;
}

// x * 10^k, checked (Int128Math.shiftLeftBy10: overflow past 127 bits, or k > 38)
TGD_HD bool u128_scale_up_ovf(U128 x, int k, U128* r)
{
    if (k > 38) { *r = x; return true; }
    return u128_mul_ovf(x, tgd_pow10(k), r);
}

// unsigned (nh:nl) / d, 256 by 128 bits; false when the quotient does not fit 128 bits (Int128Math.pack).  A 128-bit dividend over a
// divisor below 2^32 takes four digit steps; anything else shift-and-subtract from the dividend's top bit.
TGD_HD bool u256_divmod(U128 nh, U128 nl, U128 d, U128* q, U128* rem)
{
    if ((nh.hi | nh.lo) == 0 && d.hi == 0 && (d.lo >> 32) == 0) {
        // a 128-bit dividend and a divisor below 2^32 (decimal(12,2) / decimal(12,2) and the like): four 64-by-32-bit digit steps
        const unsigned long long dv = d.lo;
        const unsigned long long n3 = nl.hi >> 32, n2 = nl.hi & 0xFFFFFFFFULL, n1 = nl.lo >> 32, n0 = nl.lo & 0xFFFFFFFFULL;
        const unsigned long long q3 = n3 / dv, r3 = n3 % dv;
        const unsigned long long t2 = (r3 << 32) | n2, q2 = t2 / dv, r2 = t2 % dv;
        const unsigned long long t1 = (r2 << 32) | n1, q1 = t1 / dv, r1 = t1 % dv;
        const unsigned long long t0 = (r1 << 32) | n0, q0 = t0 / dv, r0 = t0 % dv;
        *q = U128{(q3 << 32) | q2, (q1 << 32) | q0};
        *rem = U128{0ULL, r0};
        return true;
    }
    const int nb = nh.hi | nh.lo ? 128 + u128_bits(nh) : u128_bits(nl);
    U128 r{0ULL, 0ULL}, qt{0ULL, 0ULL};
    bool fits = true;
    for (int i = nb - 1; i >= 0; i--) {
        const U128& w = i >= 128 ? nh : nl;
        const int j = i & 127;
        const unsigned long long bit = j >= 64 ? (w.hi >> (j - 64)) & 1ULL : (w.lo >> j) & 1ULL;
        const bool carry = (r.hi >> 63) != 0;
        r = U128{(r.hi << 1) | (r.lo >> 63), (r.lo << 1) | bit};
        if (carry || u128_ucmp(r, d) >= 0) {
            r = u128_sub(r, d);
            if (i >= 128) fits = false;
            else if (j >= 64) qt.hi |= 1ULL << (j - 64);
            else qt.lo |= 1ULL << j;
        }
    }
    *q = qt;
    *rem = r;
    return fits;
}

// full unsigned 128 x 128 -> 256 product (hi:lo)
TGD_HD void u128_umul_full(U128 a, U128 b, U128* hi, U128* lo)
{
    // 64-bit limbs: a = a1:a0, b = b1:b0
    const unsigned long long p00l = a.lo * b.lo, p00h = tgd_umulhi(a.lo, b.lo);
    const unsigned long long p01l = a.lo * b.hi, p01h = tgd_umulhi(a.lo, b.hi);
    const unsigned long long p10l = a.hi * b.lo, p10h = tgd_umulhi(a.hi, b.lo);
    const unsigned long long p11l = a.hi * b.hi, p11h = tgd_umulhi(a.hi, b.hi);
    unsigned long long w1 = p00h, c1 = 0;
    w1 += p01l; c1 += w1 < p01l;
    w1 += p10l; c1 += w1 < p10l;
    unsigned long long w2 = p11l, c2 = 0;
    w2 += p01h; c2 += w2 < p01h;
    w2 += p10h; c2 += w2 < p10h;
    w2 += c1; c2 += w2 < c1;
    *lo = U128{w1, p00l};
    *hi = U128{p11h + c2, w2};
}

// x / 10^k rounded HALF_UP on the magnitude (Int128Math.scaleDownRoundUp), 0 <= k
TGD_HD U128 u128_scale_down_round_up(U128 x, int k)
{
    if (k == 0) return x;
    if (k > 38) return U128{0ULL, 0ULL};     // |x| < 2^127 < 10^39 / 2
    const bool neg = u128_is_neg(x);
    const U128 d = tgd_pow10(k);
    U128 q, r;
    u256_divmod(U128{0ULL, 0ULL}, u128_abs(x), d, &q, &r);
    if (u128_ucmp(r, u128_sub(d, r)) >= 0) q = u128_add(q, U128{0ULL, 1ULL});
    return neg ? u128_negate(q) : q;
}

// Int128Math.rescale: k > 0 scales up (checked), k < 0 scales down HALF_UP
TGD_HD bool u128_rescale_ovf(U128 x, int k, U128* r)
{
    if (k >= 0) return k == 0 ? (*r = x, false) : u128_scale_up_ovf(x, k, r);
    *r = u128_scale_down_round_up(x, -k);
    return false;
}

// Decimals.overflows: outside +-(10^38 - 1)
TGD_HD bool u128_dec_overflows(U128 x)
{
    const U128 max{0x4b3b4ca85a86c47aULL, 0x098a223fffffffffULL};
    return u128_cmp(x, max) > 0 || u128_cmp(x, u128_negate(max)) < 0;
}

// |x| >= 10^p (Decimals.overflows(Int128, precision))
TGD_HD bool u128_exceeds_precision(U128 x, int p) { return u128_ucmp(u128_abs(x), tgd_pow10(p)) >= 0; }

// Int128Math.divideRoundUp(dividend, k, divisor, 0): |dividend| * 10^k / |divisor| HALF_UP, the sign restored; true on overflow
// (k >= 38 or a quotient past 128 bits).  The increment and the negation wrap as the reference's do.
TGD_HD bool u128_divide_round_up_ovf(U128 a, int k, U128 b, U128* r)
{
    if (k >= 38) return true;
    const bool neg = u128_is_neg(a) != u128_is_neg(b);
    const U128 d = u128_abs(b);
    U128 nh, nl, q, rem;
    u128_umul_full(u128_abs(a), tgd_pow10(k), &nh, &nl);
    if (!u256_divmod(nh, nl, d, &q, &rem)) return true;
    const U128 rem2{(rem.hi << 1) | (rem.lo >> 63), rem.lo << 1};
    if (u128_ucmp(rem2, d) >= 0) q = u128_add(q, U128{0ULL, 1ULL});
    *r = neg ? u128_negate(q) : q;
    return false;
}

#if defined(__CUDACC__)

// x / 10^s correctly rounded to the nearest double (DecimalConversions.longDecimalToDouble: its fast path and its parseDouble fallback
// both give the double nearest the exact value).  The magnitude is shifted left until the quotient holds at least 66 bits; the quotient
// rounds to 53 bits half-even with the remainder as sticky bit.
__device__ __forceinline__ double tgd_u128_div_pow10_to_double(U128 x, int s)
{
    if (u128_is_zero(x)) return 0.0;
    const bool neg = u128_is_neg(x);
    const U128 n = u128_abs(x), d = tgd_pow10(s);
    int sh = 66 + u128_bits(d) - u128_bits(n);     // <= 66 + 127 - 1
    if (sh < 0) sh = 0;
    U128 th, tl;     // n << sh over 256 bits
    u128_shl_wide(n, sh, &th, &tl);
    U128 q, rem;
    u256_divmod(th, tl, d, &q, &rem);     // q has 66..128 bits
    const int drop = u128_bits(q) - 53;
    unsigned long long mant = u128_shr(q, drop).lo;
    const bool round_bit = u128_bit(q, drop - 1);
    const bool sticky = !u128_is_zero(rem) || !u128_is_zero(u128_low_bits(q, drop - 1));
    int e = drop - sh;
    if (round_bit && (sticky || (mant & 1ULL))) {
        mant++;
        if (mant == (1ULL << 53)) { mant >>= 1; e++; }
    }
    const double v = scalbn((double)mant, e);
    return neg ? -v : v;
}

struct DVal {
    U128 v;
    bool is_null;
};

__device__ __forceinline__ long long tgd_mulhi_s(long long a, long long b) { return __mul64hi(a, b); }

// One DECIMAL instruction (d.is_dec) except IN: the operands as 128-bit values (a short decimal or a BIGINT sign-extended).  The
// result's low word is a short decimal, BIGINT, DOUBLE (bits) or BOOLEAN result; a long decimal uses both words.  The method is the
// reference's for the signature, fixed in `d` (expr.cu decimal_method):
//   ADD / SUB   short: a * m0 +- b * m1 (unchecked); long: k0 = rescale, k1 = rescale the left operand, k2 = result rescale
//   MUL         short: a * b (unchecked); short x short -> long: exact; long: checked, then rescale by k2
//   DIV         k0 = rescale factor; short / short -> short: divideShortShortShort with m0 = 10^k0; otherwise divideRoundUp
//   CAST_TO_DECIMAL      k0 = result precision, k1 = result scale - operand scale (DECIMAL operand) or the result scale (BIGINT),
//                        k2 = 1 when the types are identical; m0 = 10^|k1| and m1 = 10^|k1| / 2 for the short paths
//   CAST_DECIMAL_TO_*    k1 = the operand's scale, m0 = 10^k1 (short)
__device__ __forceinline__ DVal vm_apply_dec(int op, int vtype, const DDec& d, DVal a, DVal b, DVal c, uint32_t* err)
{
    DVal r;
    r.v = U128{0ULL, 0ULL};
    r.is_null = false;
    const bool shortest = !d.la && !d.lb && !d.lr;
    switch (op) {
        case TGD_EX_MOV: r = a; break;
        case TGD_EX_ADD: case TGD_EX_SUB: {
            r.is_null = a.is_null || b.is_null;
            if (r.is_null) break;
            if (shortest) {
                const unsigned long long x = a.v.lo * (unsigned long long)d.m0, y = b.v.lo * (unsigned long long)d.m1;
                r.v = u128_sx((long long)(op == TGD_EX_ADD ? x + y : x - y));
                break;
            }
            U128 x = a.v, y = b.v, s;
            bool ovf = false;
            if (d.k0) ovf = d.k1 ? u128_scale_up_ovf(a.v, d.k0, &x) : u128_scale_up_ovf(b.v, d.k0, &y);
            if (op == TGD_EX_ADD) {
                s = u128_add(x, y);
                ovf = ovf || (((s.hi ^ x.hi) & (s.hi ^ y.hi)) >> 63) != 0;
            }
            else {
                s = u128_sub(x, y);
                ovf = ovf || (((x.hi ^ y.hi) & (x.hi ^ s.hi)) >> 63) != 0;
            }
            if (!ovf) ovf = u128_rescale_ovf(s, d.k2, &r.v);
            if (ovf || u128_dec_overflows(r.v)) *err |= TG_ERR_BIT_DECIMAL_OVERFLOW;
            break;
        }
        case TGD_EX_MUL: {
            r.is_null = a.is_null || b.is_null;
            if (r.is_null) break;
            if (shortest) { r.v = u128_sx((long long)(a.v.lo * b.v.lo)); break; }
            if (!d.la && !d.lb) {
                r.v = U128{(unsigned long long)tgd_mulhi_s((long long)a.v.lo, (long long)b.v.lo), a.v.lo * b.v.lo};
                break;
            }
            U128 p;
            bool ovf = u128_mul_ovf(a.v, b.v, &p);
            if (!ovf) ovf = u128_rescale_ovf(p, d.k2, &r.v);
            if (ovf || u128_dec_overflows(r.v)) *err |= TG_ERR_BIT_DECIMAL_OVERFLOW;
            break;
        }
        case TGD_EX_DIV: {
            r.is_null = a.is_null || b.is_null;
            if (r.is_null) break;
            if (u128_is_zero(b.v)) { *err |= TG_ERR_BIT_DIV_ZERO; break; }
            if (shortest) {
                // divideShortShortShort, 64-bit wraparound included
                const long long x = (long long)a.v.lo, y = (long long)b.v.lo;
                if (x == 0) break;
                const long long sg = (x > 0 ? 1 : -1) * (y > 0 ? 1 : -1);
                const long long ux = x < 0 ? (long long)(0ULL - (unsigned long long)x) : x, uy = y < 0 ? (long long)(0ULL - (unsigned long long)y) : y;
                const long long rs = (long long)((unsigned long long)ux * (unsigned long long)d.m0);
                const long long q = rs / uy;     // (uy is never -1)
                const long long rem = (long long)((unsigned long long)rs - (unsigned long long)q * (unsigned long long)uy);
                const long long q2 = (unsigned long long)rem * 2ULL >= (unsigned long long)uy ? (long long)((unsigned long long)q + 1ULL) : q;
                r.v = u128_sx((long long)((unsigned long long)sg * (unsigned long long)q2));
                break;
            }
            U128 q;
            bool ovf = u128_divide_round_up_ovf(a.v, d.k0, b.v, &q);
            if (!ovf) ovf = d.lr ? u128_dec_overflows(q) : q.hi != (unsigned long long)((long long)q.lo >> 63);
            if (ovf) *err |= TG_ERR_BIT_DECIMAL_OVERFLOW;
            else r.v = q;
            break;
        }
        case TGD_EX_NEG:
            r.is_null = a.is_null;
            if (r.is_null) break;
            if (!d.la) r.v = u128_sx((long long)(0ULL - a.v.lo));
            else {
                if (a.v.hi == 0x8000000000000000ULL && a.v.lo == 0ULL) *err |= TG_ERR_BIT_DECIMAL_OVERFLOW;
                r.v = u128_negate(a.v);
            }
            break;
        case TGD_EX_EQ: case TGD_EX_NE: case TGD_EX_LT: case TGD_EX_LE: case TGD_EX_GT: case TGD_EX_GE: {
            r.is_null = a.is_null || b.is_null;
            if (r.is_null) break;
            const int k = d.la ? u128_cmp(a.v, b.v) : ((long long)a.v.lo < (long long)b.v.lo ? -1 : (long long)a.v.lo > (long long)b.v.lo ? 1 : 0);
            const bool t = op == TGD_EX_EQ ? k == 0 : op == TGD_EX_NE ? k != 0 : op == TGD_EX_LT ? k < 0 : op == TGD_EX_LE ? k <= 0 : op == TGD_EX_GT ? k > 0 : k >= 0;
            r.v.lo = t ? 1ULL : 0ULL;
            break;
        }
        case TGD_EX_BETWEEN: {
            const bool n1 = a.is_null || b.is_null, n2 = a.is_null || c.is_null;
            const bool f1 = !n1 && u128_cmp(a.v, b.v) < 0, f2 = !n2 && u128_cmp(a.v, c.v) > 0;
            r.is_null = !(f1 || f2) && (n1 || n2);
            r.v.lo = (f1 || f2 || r.is_null) ? 0ULL : 1ULL;
            break;
        }
        case TGD_EX_IS_NULL: r.v.lo = a.is_null ? 1ULL : 0ULL; break;
        case TGD_EX_IS_NOT_NULL: r.v.lo = a.is_null ? 0ULL : 1ULL; break;
        case TGD_EX_CAST_TO_DECIMAL: {
            r.is_null = a.is_null;
            if (r.is_null) break;
            bool bad = false;
            if (vtype != TGD_V_DECIMAL) {
                if (!d.lr) {
                    // bigintToShortDecimal: multiplyExact, then |v| >= 10^p (Math.abs wraps at Long.MIN_VALUE as the reference's does)
                    const long long x = (long long)a.v.lo, v = (long long)((unsigned long long)x * (unsigned long long)d.m0);
                    bad = tgd_mulhi_s(x, d.m0) != (v >> 63);
                    const long long av = v < 0 ? (long long)(0ULL - (unsigned long long)v) : v;
                    bad = bad || av >= (long long)tgd_pow10(d.k0).lo;
                    r.v = u128_sx(v);
                }
                else {
                    bad = u128_mul_ovf(tgd_pow10(d.k1), a.v, &r.v);
                    bad = bad || u128_exceeds_precision(r.v, d.k0);
                }
            }
            else if (d.k2) r = a;
            else if (!d.la && !d.lr) {
                // shortToShortCast
                const long long x = (long long)a.v.lo;
                long long v;
                if (d.k1 >= 0) v = (long long)((unsigned long long)x * (unsigned long long)d.m0);
                else {
                    v = x / d.m0;
                    const long long rm = x % d.m0;
                    if (x >= 0) { if (rm >= d.m1) v++; }
                    else if (rm <= -d.m1) v--;
                }
                const long long av = v < 0 ? (long long)(0ULL - (unsigned long long)v) : v;
                bad = av >= (long long)tgd_pow10(d.k0).lo;
                r.v = u128_sx(v);
            }
            else {
                bad = u128_rescale_ovf(a.v, d.k1, &r.v) || u128_exceeds_precision(r.v, d.k0);
                if (!d.lr) r.v = u128_sx((long long)r.v.lo);
            }
            if (bad) { *err |= TG_ERR_BIT_INVALID_CAST; r.v = U128{0ULL, 0ULL}; }
            break;
        }
        case TGD_EX_CAST_DECIMAL_TO_BIGINT:
            r.is_null = a.is_null;
            if (r.is_null) break;
            if (!d.la) {
                const unsigned long long x = a.v.lo, h = (unsigned long long)d.m0 / 2ULL;
                r.v = u128_sx((long long)x >= 0 ? (long long)(x + h) / d.m0 : (long long)(0ULL - (unsigned long long)((long long)(0ULL - x + h) / d.m0)));
            }
            else {
                const U128 q = u128_scale_down_round_up(a.v, d.k1);
                if (q.hi != (unsigned long long)((long long)q.lo >> 63)) *err |= TG_ERR_BIT_INVALID_CAST;
                else r.v = q;
            }
            break;
        case TGD_EX_CAST_DECIMAL_TO_DOUBLE:
            r.is_null = a.is_null;
            if (r.is_null) break;
            r.v.lo = (unsigned long long)__double_as_longlong(d.la ? tgd_u128_div_pow10_to_double(a.v, d.k1)
                                                                   : __ddiv_rn((double)(long long)a.v.lo, (double)d.m0));
            break;
        // a is the BOOLEAN condition (la = 0); b, c and the result are one DECIMAL type, so both words are selected as they are
        case TGD_EX_IF: r = (!a.is_null && a.v.lo != 0ULL) ? b : c; break;
        case TGD_EX_COALESCE: r = a.is_null ? b : a; break;
        default: break;
    }
    if (!d.lr && op != TGD_EX_MOV) r.v.hi = (unsigned long long)((long long)r.v.lo >> 63);
    return r;
}

// vm_error for a DECIMAL instruction: the same rules, BETWEEN's "min <= value" compared as 128-bit values
__device__ __forceinline__ uint32_t vm_error_dec(int op, DVal a, uint32_t ea, DVal b, uint32_t eb, uint32_t ec, uint32_t own)
{
    if (ea) return ea;
    switch (op) {
        case TGD_EX_BETWEEN:
            if (a.is_null) return 0;
            if (eb) return eb;
            if (!b.is_null && u128_cmp(b.v, a.v) > 0) return 0;
            return ec;
        case TGD_EX_IF: return (!a.is_null && a.v.lo != 0ULL) ? eb : ec;
        case TGD_EX_COALESCE: return a.is_null ? eb : 0;
        case TGD_EX_ADD: case TGD_EX_SUB: case TGD_EX_MUL: case TGD_EX_DIV:
        case TGD_EX_EQ: case TGD_EX_NE: case TGD_EX_LT: case TGD_EX_LE: case TGD_EX_GT: case TGD_EX_GE:
            if (a.is_null) return 0;
            return eb ? eb : own;
        default: return own;
    }
}

// ---- accumulators -------------------------------------------------------------------------------------
// order-preserving encodings so MIN/MAX are plain integer min/max.  min(DOUBLE) compares with COMPARISON_UNORDERED_LAST
// (NaN is the largest value, S/type/DoubleType.java:231-235), max(DOUBLE) with COMPARISON_UNORDERED_FIRST (NaN is the
// smallest, :237-252; M/operator/aggregation/MaxAggregationFunction.java:49): max({1.0, NaN}) = 1.0, max({NaN}) = NaN.
__host__ __device__ __forceinline__ unsigned long long f64_order_key(long long bits)
{
    unsigned long long u = (unsigned long long)bits;
    if ((u & 0x7FFFFFFFFFFFFFFFULL) > 0x7FF0000000000000ULL) u = 0x7FF8000000000000ULL;
    return (u >> 63) ? ~u : (u | 0x8000000000000000ULL);
}
// key for MAX: NaN ranks below every other value (key 1: above the "no row yet" initial 0, below -Infinity's key)
__host__ __device__ __forceinline__ unsigned long long f64_order_key_max(long long bits)
{
    unsigned long long u = (unsigned long long)bits;
    if ((u & 0x7FFFFFFFFFFFFFFFULL) > 0x7FF0000000000000ULL) return 1ULL;
    return (u >> 63) ? ~u : (u | 0x8000000000000000ULL);
}
__host__ __device__ __forceinline__ long long f64_from_order_key(unsigned long long k)
{
    if (k == 1ULL) return 0x7FF8000000000000LL;      // MAX's NaN (never produced by f64_order_key)
    return (long long)((k >> 63) ? (k & 0x7FFFFFFFFFFFFFFFULL) : ~k);
}
__host__ __device__ __forceinline__ unsigned long long i64_order_key(long long v) { return (unsigned long long)v ^ 0x8000000000000000ULL; }

__host__ __device__ __forceinline__ unsigned long long acc_init(int kind)
{
    return (kind == ACC_MIN_F64 || kind == ACC_MIN_I64) ? 0xFFFFFFFFFFFFFFFFULL : 0ULL;
}

__device__ __forceinline__ unsigned long long acc_combine(int kind, unsigned long long a, unsigned long long b)
{
    switch (kind) {
        case ACC_SUM_F64: case ACC_SUM_F64_FROM_I64:
            return (unsigned long long)__double_as_longlong(__dadd_rn(__longlong_as_double((long long)a), __longlong_as_double((long long)b)));
        case ACC_MIN_F64: case ACC_MIN_I64: return a < b ? a : b;
        case ACC_MAX_F64: case ACC_MAX_I64: return a > b ? a : b;
        default: return a + b;   // counts and the two halves of the 128-bit integer sum (carry handled by caller)
    }
}

// VarianceState.update (M/operator/aggregation/state/VarianceState.java:35-41), Welford's step on (count, mean bits, m2 bits)
__device__ __forceinline__ void acc_var_step(unsigned long long& n, unsigned long long& mean_bits, unsigned long long& m2_bits, double x)
{
    const long long c = (long long)n + 1;
    double mean = __longlong_as_double((long long)mean_bits), m2 = __longlong_as_double((long long)m2_bits);
    const double delta = __dsub_rn(x, mean);
    mean = __dadd_rn(mean, __ddiv_rn(delta, __ll2double_rn(c)));
    m2 = __dadd_rn(m2, __dmul_rn(delta, __dsub_rn(x, mean)));
    n = (unsigned long long)c;
    mean_bits = (unsigned long long)__double_as_longlong(mean);
    m2_bits = (unsigned long long)__double_as_longlong(m2);
}

// one accumulator update by one row on a thread-private accumulator word; `hi_off` = distance to the HI half
__device__ __forceinline__ void acc_update_private(int kind, unsigned long long* p, long long hi_off, long long bits)
{
    switch (kind) {
        case ACC_ROWS: case ACC_NONNULL: *p += 1; break;
        case ACC_SUM_F64: *p = (unsigned long long)__double_as_longlong(__dadd_rn(__longlong_as_double((long long)*p), __longlong_as_double(bits))); break;
        case ACC_SUM_F64_FROM_I64: *p = (unsigned long long)__double_as_longlong(__dadd_rn(__longlong_as_double((long long)*p), (double)bits)); break;
        case ACC_SUM_I64_LO: {
            unsigned long long old = *p, add = (unsigned long long)bits, nw = old + add;
            *p = nw;
            p[hi_off] += (unsigned long long)((bits < 0 ? -1LL : 0LL) + (nw < old ? 1LL : 0LL));
            break;
        }
        case ACC_MIN_F64: { unsigned long long k = f64_order_key(bits); if (k < *p) *p = k; break; }
        case ACC_MAX_F64: { unsigned long long k = f64_order_key_max(bits); if (k > *p) *p = k; break; }
        case ACC_MIN_I64: { unsigned long long k = i64_order_key(bits); if (k < *p) *p = k; break; }
        case ACC_MAX_I64: { unsigned long long k = i64_order_key(bits); if (k > *p) *p = k; break; }
        case ACC_VAR_F64: case ACC_VAR_I64: {
            unsigned long long n = *p, mean = p[hi_off], m2 = p[2 * hi_off];
            acc_var_step(n, mean, m2, kind == ACC_VAR_F64 ? __longlong_as_double(bits) : __ll2double_rn(bits));
            *p = n;
            p[hi_off] = mean;
            p[2 * hi_off] = m2;
            break;
        }
        default: break;
    }
}

// VarianceState.merge (VarianceState.java:43-59), Chan's combination of (n, mean, m2) with (nb, mb, qb), in place.  An empty side leaves
// the other unchanged.  The new mean is written mean + delta * nb / n (not the reference's (n * mean + nb * mb) / n): it stays exact when
// the two means agree, so a group of identical values keeps m2 == +0.0 however its rows were split.
__device__ __forceinline__ void tgd_var_merge(unsigned long long& n, unsigned long long& mean, unsigned long long& m2,
                                              unsigned long long nb, unsigned long long mb, unsigned long long qb)
{
    if ((long long)nb == 0) return;
    if ((long long)n == 0) { n = nb; mean = mb; m2 = qb; return; }
    const long long na = (long long)n, nt = na + (long long)nb;
    const double ma = __longlong_as_double((long long)mean), dn = __ll2double_rn(nt), dnb = __ll2double_rn((long long)nb);
    const double delta = __dsub_rn(__longlong_as_double((long long)mb), ma);
    const double m = __dadd_rn(ma, __ddiv_rn(__dmul_rn(delta, dnb), dn));
    const double cross = __ddiv_rn(__dmul_rn(__dmul_rn(__dmul_rn(delta, delta), dnb), __ll2double_rn(na)), dn);
    const double q = __dadd_rn(__dadd_rn(__longlong_as_double((long long)m2), __longlong_as_double((long long)qb)), cross);
    n = (unsigned long long)nt;
    mean = (unsigned long long)__double_as_longlong(m);
    m2 = (unsigned long long)__double_as_longlong(q);
}

// one intermediate state row (count, mean bits, m2 bits) merged into a thread-private variance accumulator; `hi_off` = word distance
__device__ __forceinline__ void acc_var_merge_private(unsigned long long* p, long long hi_off, long long count, long long mean_bits, long long m2_bits)
{
    unsigned long long n = *p, mean = p[hi_off], m2 = p[2 * hi_off];
    tgd_var_merge(n, mean, m2, (unsigned long long)count, (unsigned long long)mean_bits, (unsigned long long)m2_bits);
    *p = n;
    p[hi_off] = mean;
    p[2 * hi_off] = m2;
}

__host__ __device__ __forceinline__ bool acc_is_var(int kind) { return kind == ACC_VAR_F64 || kind == ACC_VAR_I64 || kind == ACC_VAR_STATE; }

// ---- small-group fused aggregation: kernel body as a template over a row program ------------------------
// A row program P provides
//   static constexpr int L (key slots per CTA, power of two), A (accumulator words per group), R (rows per thread
//   in flight per loop trip)
//   struct P::Regs                      raw column values of one row
//   __device__ static int acc_kind(int a)
//   __device__ void load(cols, row, Regs&)                 all global loads of a row, nothing else
//   __device__ bool row(const Regs&, &key, &special, &err) filter + projections + key packing; false = row rejected;
//        `special` = 0 (NULL key) / 1 (key equal to the EMPTY sentinel) / -1
//   __device__ void accumulate(acc_ptr /* &acc[(slot*A)*T + tid] */, T)   applies every accumulator for that row
// The loads of R rows are issued back to back before the first row is consumed (memory-level parallelism), then the
// rows are folded one by one into the thread-private accumulators.
// Shared memory: tkeys[L] | lfirst[L+2] | acc[(L+2)*A*T].
template <class P>
__device__ __forceinline__ void agg_small_body(P& prog, const DColumns& cols, int64_t n, SmallOut out, unsigned long long* smem_u64)
{
    constexpr int L = P::L, A = P::A, T = TGD_S_THREADS;
    unsigned long long* tkeys = smem_u64;
    long long* lfirst = (long long*)(tkeys + L);
    unsigned long long* acc = (unsigned long long*)(lfirst + L + 2);
    const int tid = threadIdx.x;

    for (int i = tid; i < L; i += T) tkeys[i] = TGD_EMPTY_KEY;
    for (int i = tid; i < L + 2; i += T) lfirst[i] = TGD_NO_ROW;
    // the two special groups (NULL key, sentinel-valued key) exist for single-key plans only: a packed multi-column key never takes them,
    // and without their accumulator sets a CTA needs a third less shared memory (Q1: 73.8 -> 49.2 KB, 4 CTAs per SM instead of 3)
    constexpr int SETS = P::SPECIALS ? L + 2 : L;
    for (int s = 0; s < SETS; s++)
        for (int a = 0; a < A; a++) acc[((size_t)s * A + a) * T + tid] = acc_init(P::acc_kind(a));
    __shared__ int s_overflow;
    if (tid == 0) s_overflow = 0;
    __syncthreads();

    unsigned long long seen = 0;
    uint32_t err = 0;
    constexpr int R = P::R;
    const int64_t stride = (int64_t)gridDim.x * T;
    bool stop = false;
    // VEC: a thread owns R = 4 CONSECUTIVE rows per trip (16-byte loads, a warp reads 128 consecutive rows of every column);
    // otherwise its R rows are a grid stride apart.  Either way the rows of one thread ascend.
    static_assert(!P::VEC || R == 4, "the vector loader handles four rows");
    const int64_t first = P::VEC ? ((int64_t)blockIdx.x * T + tid) * R : (int64_t)blockIdx.x * T + tid;
    const int64_t row_step = P::VEC ? 1 : stride;
    for (int64_t base = first; base < n && !stop; base += stride * R) {
        if (*((volatile int*)&s_overflow)) break;   // some thread of this CTA ran out of key slots: the pass is void
        typename P::Regs regs[R];
        if (P::VEC && base + R <= n) prog.load4(cols, base, regs);
        else {
#pragma unroll
            for (int j = 0; j < R; j++) {
                int64_t row = base + (int64_t)j * row_step;
                if (row < n) prog.load(cols, row, regs[j]);
            }
        }
#pragma unroll
        for (int j = 0; j < R; j++) {
            int64_t row = base + (int64_t)j * row_step;
            if (row >= n || stop) continue;
            unsigned long long pk = 0;
            int special = -1;
            if (!prog.row(regs[j], &pk, &special, &err)) continue;
            int slot;
            if (special >= 0) slot = L + special;
            else {
                int h = (int)(tgd_murmur3_mix(pk) & (unsigned long long)(L - 1));
                slot = -1;
                for (int probe = 0; probe < L; probe++) {
                    unsigned long long cur = tkeys[h];
                    if (cur == TGD_EMPTY_KEY) cur = atomicCAS(&tkeys[h], TGD_EMPTY_KEY, pk);
                    if (cur == TGD_EMPTY_KEY || cur == pk) { slot = h; break; }
                    h = (h + 1) & (L - 1);
                }
                if (slot < 0) { s_overflow = 1; stop = true; continue; }   // more distinct keys in this CTA than L: host switches to path G
            }
            if (!((seen >> slot) & 1)) {
                seen |= 1ULL << slot;
                atomicMin(&lfirst[slot], (long long)row);   // rows of one thread ascend: its first hit is its minimum
            }
            prog.accumulate(&acc[((size_t)slot * A) * T + tid], T);
        }
    }
    if (err) atomicOr(out.err, err);
    __syncthreads();
    if (s_overflow) {
        if (tid == 0) *out.overflow = 1;
        return;
    }

    // fixed-order reduction of the T private copies of every (slot, acc): lane-sequential then xor tree
    const int warp = tid >> 5, lane = tid & 31, nwarps = T >> 5;
    const size_t b = blockIdx.x;
    for (int pair = warp; pair < (L + 2) * A; pair += nwarps) {
        int s = pair / A, a = pair % A;
        int kind = P::acc_kind(a);
        if (kind == ACC_SUM_I64_HI || kind == ACC_VAR_MEAN || kind == ACC_VAR_M2) continue;   // reduced together with their first word
        if (lfirst[s] == TGD_NO_ROW) continue;
        const unsigned long long* p = &acc[((size_t)s * A + a) * T];
        if (acc_is_var(kind)) {
            unsigned long long n = 0, m = 0, q = 0;
            for (int t = lane; t < T; t += 32) tgd_var_merge(n, m, q, p[t], p[t + T], p[t + 2 * T]);
            for (int off = 16; off > 0; off >>= 1) {
                const unsigned long long on = __shfl_xor_sync(0xffffffffu, n, off), om = __shfl_xor_sync(0xffffffffu, m, off),
                                         oq = __shfl_xor_sync(0xffffffffu, q, off);
                tgd_var_merge(n, m, q, on, om, oq);
            }
            if (lane == 0) {
                out.blk_acc[(b * (L + 2) + s) * A + a] = n;
                out.blk_acc[(b * (L + 2) + s) * A + a + 1] = m;
                out.blk_acc[(b * (L + 2) + s) * A + a + 2] = q;
            }
        }
        else if (kind == ACC_SUM_I64_LO) {
            const unsigned long long* ph = p + T;
            unsigned long long lo = 0, hi = 0;
            for (int t = lane; t < T; t += 32) { unsigned long long o = lo; lo += p[t]; hi += ph[t] + (lo < o ? 1 : 0); }
            for (int off = 16; off > 0; off >>= 1) {
                unsigned long long ol = __shfl_xor_sync(0xffffffffu, lo, off), oh = __shfl_xor_sync(0xffffffffu, hi, off);
                unsigned long long o = lo; lo += ol; hi += oh + (lo < o ? 1 : 0);
            }
            if (lane == 0) {
                out.blk_acc[(b * (L + 2) + s) * A + a] = lo;
                out.blk_acc[(b * (L + 2) + s) * A + a + 1] = hi;
            }
        }
        else {
            unsigned long long r = acc_init(kind);
            for (int t = lane; t < T; t += 32) r = acc_combine(kind, r, p[t]);
            for (int off = 16; off > 0; off >>= 1) r = acc_combine(kind, r, __shfl_xor_sync(0xffffffffu, r, off));
            if (lane == 0) out.blk_acc[(b * (L + 2) + s) * A + a] = r;
        }
    }
    for (int s = tid; s < L + 2; s += T) {
        out.blk_first[b * (L + 2) + s] = lfirst[s];
        if (s < L) out.blk_keys[b * L + s] = tkeys[s];
    }
}

// ---- global aggregation (no GROUP BY keys): kernel body as a template over the same row program -----------------------------
// Fixed-order CTA reduction of per-thread accumulator words: an xor-shuffle tree inside every warp (a 128-bit integer sum travels as
// its LO/HI pair with the carry, as in agg_small_body), then the warps folded in warp order through shared memory `wpart`
// ([warps][A]); thread a writes the CTA's word a to out[a].  `kind_of(a)` = accumulator kind of word a.
template <class KindOf>
__device__ __forceinline__ void tgd_cta_reduce(const unsigned long long* acc, int A, KindOf kind_of, unsigned long long* wpart, unsigned long long* out)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
#pragma unroll
    for (int a = 0; a < A; a++) {
        const int kind = kind_of(a);
        if (kind == ACC_SUM_I64_HI || kind == ACC_VAR_MEAN || kind == ACC_VAR_M2) continue;
        if (acc_is_var(kind)) {
            unsigned long long n = acc[a], m = acc[a + 1], q = acc[a + 2];
            for (int off = 16; off > 0; off >>= 1) {
                const unsigned long long on = __shfl_xor_sync(0xffffffffu, n, off), om = __shfl_xor_sync(0xffffffffu, m, off),
                                         oq = __shfl_xor_sync(0xffffffffu, q, off);
                tgd_var_merge(n, m, q, on, om, oq);
            }
            if (lane == 0) { wpart[warp * A + a] = n; wpart[warp * A + a + 1] = m; wpart[warp * A + a + 2] = q; }
        }
        else if (kind == ACC_SUM_I64_LO) {
            unsigned long long lo = acc[a], hi = acc[a + 1];
            for (int off = 16; off > 0; off >>= 1) {
                unsigned long long ol = __shfl_xor_sync(0xffffffffu, lo, off), oh = __shfl_xor_sync(0xffffffffu, hi, off);
                unsigned long long o = lo; lo += ol; hi += oh + (lo < o ? 1 : 0);
            }
            if (lane == 0) { wpart[warp * A + a] = lo; wpart[warp * A + a + 1] = hi; }
        }
        else {
            unsigned long long r = acc[a];
            for (int off = 16; off > 0; off >>= 1) r = acc_combine(kind, r, __shfl_xor_sync(0xffffffffu, r, off));
            if (lane == 0) wpart[warp * A + a] = r;
        }
    }
    __syncthreads();
    for (int a = threadIdx.x; a < A; a += blockDim.x) {
        const int kind = kind_of(a);
        if (kind == ACC_SUM_I64_HI || kind == ACC_VAR_MEAN || kind == ACC_VAR_M2) continue;
        if (acc_is_var(kind)) {
            unsigned long long n = 0, m = 0, q = 0;
            for (int w = 0; w < nwarps; w++) tgd_var_merge(n, m, q, wpart[w * A + a], wpart[w * A + a + 1], wpart[w * A + a + 2]);
            out[a] = n;
            out[a + 1] = m;
            out[a + 2] = q;
        }
        else if (kind == ACC_SUM_I64_LO) {
            unsigned long long lo = 0, hi = 0;
            for (int w = 0; w < nwarps; w++) { unsigned long long o = lo; lo += wpart[w * A + a]; hi += wpart[w * A + a + 1] + (lo < o ? 1 : 0); }
            out[a] = lo;
            out[a + 1] = hi;
        }
        else {
            unsigned long long r = acc_init(kind);
            for (int w = 0; w < nwarps; w++) r = acc_combine(kind, r, wpart[w * A + a]);
            out[a] = r;
        }
    }
}

// AggregationOperator's hot loop: every row of the page folds into ONE group, so the accumulators are per-thread registers
// (acc[P::A] at stride 1: the generated accumulate() indexes them with constants), with no table, no first-row stamps and no atomics
// in the row loop.  A thread owns 4 consecutive rows per trip of a grid-stride loop.  Deferred loads: the columns only the filter reads
// come first (load4_early / load_early); the other columns (projection and aggregate inputs) are read only when one of the thread's 4
// rows passed the filter - for an 8-byte column the 4 rows are one 32-byte sector, which a thread whose rows all fail never touches.
// Output: the CTA's accumulator words at part[blockIdx.x * A] (folded in CTA order by agg_global_fold_kernel) and the error bits.
// P supplies, besides the members agg_small_body uses: load_early / load_late / load4_early / load4_late (the two halves of load /
// load4) and filter(regs, &err) (the filter alone; its errors count on every row).
template <class P>
__device__ __forceinline__ void agg_global_body(P& prog, const DColumns& cols, int64_t n, unsigned long long* __restrict__ part, unsigned int* __restrict__ err_out)
{
    constexpr int A = P::A, R = 4, T = TGD_S_THREADS;
    static_assert(A >= 1, "at least one accumulator word");
    __shared__ unsigned long long wpart[(T / 32) * A];
    unsigned long long acc[A];
#pragma unroll
    for (int a = 0; a < A; a++) acc[a] = acc_init(P::acc_kind(a));
    uint32_t err = 0;
    const int64_t stride = (int64_t)gridDim.x * T * R;
    for (int64_t base = ((int64_t)blockIdx.x * T + threadIdx.x) * R; base < n; base += stride) {
        typename P::Regs regs[R];
        const bool vec = P::VEC && base + R <= n;
        if (vec) prog.load4_early(cols, base, regs);
        else {
#pragma unroll
            for (int j = 0; j < R; j++)
                if (base + j < n) prog.load_early(cols, base + j, regs[j]);
        }
        bool pass[R];
        bool any = false;
#pragma unroll
        for (int j = 0; j < R; j++) {
            pass[j] = base + j < n && prog.filter(regs[j], &err);
            any |= pass[j];
        }
        if (!any) continue;
        if (vec) prog.load4_late(cols, base, regs);
        else {
#pragma unroll
            for (int j = 0; j < R; j++)
                if (pass[j]) prog.load_late(cols, base + j, regs[j]);
        }
#pragma unroll
        for (int j = 0; j < R; j++) {
            if (!pass[j]) continue;
            unsigned long long pk = 0;
            int special = -1;
            if (prog.row(regs[j], &pk, &special, &err)) prog.accumulate(acc, 1);
        }
    }
    tgd_cta_reduce(acc, A, [](int a) { return P::acc_kind(a); }, wpart, part + (size_t)blockIdx.x * A);
    if (err) atomicOr(err_out, err);
}

// ---- general group-by, fused single pass (path G): kernel body as a template over the same row program ---------------------
// One AoS record per table slot: {key, first-row stamp, accumulator words ...} (W 8-byte words).  A row finds or claims its key's
// record, lowers the stamp and applies its accumulators with fire-and-forget reductions.  R rows are in flight per thread: all column
// loads of the R rows first, then the R record heads (independent random reads), then the resolves.  Claims are budgeted through
// TGD_TICKET_WAYS counters (tickets[way]; a way is picked by the lane) so that a page of mostly new keys does not serialise on one
// L2 address; a row that finds its way's budget exhausted goes to the deferred list and is replayed after the table has grown.
// tickets layout: [0, WAYS) claims per way, [WAYS] deferred rows, [WAYS + 1] special groups born.
// P supplies, besides load() / row(): accumulate_global(unsigned long long* acc) - reductions on the record's accumulator words.
#define TGD_TICKET_WAYS 64
#define TGD_G_ROWS 2      // rows in flight per thread with __launch_bounds__(256, 4)

// {a, b} = the two 64-bit words at p (16-byte aligned) in one L2 transaction, never served from the L1
__device__ __forceinline__ void tgd_ld_pair(const unsigned long long* p, unsigned long long& a, unsigned long long& b)
{
    asm volatile("ld.volatile.global.v2.u64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "l"(p) : "memory");
}

template <class P>
__device__ __forceinline__ void agg_general_body(P& prog, const DColumns& cols, long long n, const int* __restrict__ rows, long long first,
                                                 const int* __restrict__ stamp_rows, long long page_base, unsigned long long* __restrict__ recs, long long cap, int W,
                                                 int* __restrict__ tickets, int budget_per_way, int* __restrict__ deferred, unsigned int* __restrict__ err_out)
{
    constexpr int R = P::GR;          // rows in flight per thread (TGD_G_ROWS unless the generator says otherwise)
    const unsigned long long mask = (unsigned long long)cap - 1;
    const int way = ((threadIdx.x >> 5) + blockIdx.x * 8) & (TGD_TICKET_WAYS - 1);      // one ticket word per warp at a time
    const int lane = threadIdx.x & 31;
    unsigned int err = 0;
    int have = 0;                                                     // tickets in hand (the same number in every lane)
    const int batch = budget_per_way >= (32 << 8) ? 32 : (budget_per_way >> 8) > 0 ? (budget_per_way >> 8) : 1;
    const long long stride = (long long)gridDim.x * blockDim.x;
    // the loop is uniform per warp (every lane makes the same trips) so that the warp can re-converge explicitly between the phases:
    // measured on the first version, the divergent tail of the probe loop ran the stamp + accumulator code with ~7 of 32 lanes active
    for (long long wbase = (long long)blockIdx.x * blockDim.x + (threadIdx.x & ~31); wbase < n; wbase += stride * R) {
        typename P::Regs regs[R];
        long long row[R];
#pragma unroll
        for (int j = 0; j < R; j++) {
            long long i = wbase + lane + (long long)j * stride;
            row[j] = i < n ? (rows ? (long long)rows[i] : first + i) : -1;
            if (row[j] >= 0) prog.load(cols, row[j], regs[j]);
        }
        unsigned long long pk[R], pos[R], cur[R], nxt[R];
        long long slot[R];
        bool open[R];        // still looking for its slot
#pragma unroll
        for (int j = 0; j < R; j++) {
            pk[j] = 0;
            int sp = -1;
            if (row[j] >= 0 && !prog.row(regs[j], &pk[j], &sp, &err)) row[j] = -1;      // rejected by the fused filter
            pos[j] = tgd_murmur3_mix(pk[j]) & mask;
            slot[j] = (row[j] >= 0 && sp >= 0) ? cap + sp : -1;
            open[j] = row[j] >= 0 && sp < 0;
        }
        // one 16-byte load brings the home slot's key AND its first-row stamp; the successor's key is requested with it: a row that
        // has to move on finds the next key already on its way, and a row that stays (most do) never reads its stamp separately
        unsigned long long st0[R];
#pragma unroll
        for (int j = 0; j < R; j++) {
            cur[j] = 0; st0[j] = 0; nxt[j] = 0;
            if (open[j]) {
                tgd_ld_pair(recs + (size_t)pos[j] * W, cur[j], st0[j]);
                nxt[j] = *((volatile unsigned long long*)(recs + (size_t)((pos[j] + 1) & mask) * W));
            }
        }
        bool moved[R];
#pragma unroll
        for (int j = 0; j < R; j++) moved[j] = false;
        // lock-step probing: one step of every open row per trip, the warp stays converged.  Insertions need a ticket (the fill limit
        // of the table is a budget of tickets per way); a warp draws them in batches and keeps the remainder (`have`, warp-uniform), so
        // the returning atomicAdd sits on the critical path of one insertion in `batch`, not of every trip that inserts.
        while (true) {
            bool any = false;
#pragma unroll
            for (int j = 0; j < R; j++) {
                bool active = open[j];
                unsigned long long c = cur[j];
                const bool want = active && c == TGD_EMPTY_KEY;
                const unsigned int wmask = __ballot_sync(0xffffffffu, want);
                if (wmask) {
                    const int cnt = __popc(wmask), leader = __ffs(wmask) - 1;
                    if (cnt > have) {
                        int got = 0;
                        if (lane == leader) {
                            const int ask = cnt - have > batch ? cnt - have : batch;
                            const int base = atomicAdd(tickets + way, ask);
                            got = budget_per_way - base;
                            got = got < 0 ? 0 : (got > ask ? ask : got);
                            if (got < ask) atomicSub(tickets + way, ask - got);          // drawn beyond the budget: handed back at once
                        }
                        have += __shfl_sync(0xffffffffu, got, leader);
                    }
                    const bool granted = want && __popc(wmask & ((1u << lane) - 1)) < have;
                    have -= cnt < have ? cnt : have;
                    bool won = false;
                    if (granted) {
                        c = atomicCAS(recs + (size_t)pos[j] * W, TGD_EMPTY_KEY, pk[j]);
                        won = c == TGD_EMPTY_KEY;
                    }
                    have += __popc(__ballot_sync(0xffffffffu, granted && !won));          // lost the race for the slot: the ticket stays in hand
                    if (want && !granted) { open[j] = false; active = false; }              // no room: deferred below
                    if (won) { slot[j] = (long long)pos[j]; open[j] = false; active = false; }
                }
                if (active) {
                    if (c == pk[j]) { slot[j] = (long long)pos[j]; open[j] = false; }
                    else {
                        pos[j] = (pos[j] + 1) & mask;
                        cur[j] = nxt[j];
                        nxt[j] = *((volatile unsigned long long*)(recs + (size_t)((pos[j] + 1) & mask) * W));
                        moved[j] = true;
                        any = true;
                    }
                }
            }
            if (!__any_sync(0xffffffffu, any)) break;
        }
        __syncwarp();
        // stamps: read the R stamps first, lower the ones that need it
        long long stamp[R], seen[R];
#pragma unroll
        for (int j = 0; j < R; j++) {
            stamp[j] = 0;
            seen[j] = 0;
            if (row[j] >= 0 && slot[j] >= 0) {
                stamp[j] = page_base + (stamp_rows ? (long long)stamp_rows[row[j]] : row[j]);
                // (a stamp read together with the key may be stale, i.e. too high: stamps only ever go down, so the worst case is one
                //  atomicMin that changes nothing)
                seen[j] = (!moved[j] && slot[j] < cap) ? (long long)st0[j] : *((volatile long long*)(recs + (size_t)slot[j] * W + 1));
            }
        }
#pragma unroll
        for (int j = 0; j < R; j++) {
            if (row[j] < 0) continue;
            if (slot[j] < 0) { deferred[atomicAdd(tickets + TGD_TICKET_WAYS, 1)] = (int)row[j]; continue; }
            if (seen[j] > stamp[j]) {
                long long old = atomicMin((long long*)(recs + (size_t)slot[j] * W + 1), stamp[j]);
                if (old == TGD_NO_ROW && slot[j] >= cap) atomicAdd(tickets + TGD_TICKET_WAYS + 1, 1);   // a special (NULL / sentinel key) group came to life
            }
        }
        __syncwarp();
#pragma unroll
        for (int j = 0; j < R; j++) {
            if (row[j] < 0 || slot[j] < 0) continue;
            unsigned long long pk2;
            int sp2;
            prog.row(regs[j], &pk2, &sp2, &err);          // re-establish this row's values (registers only) for the accumulators
            prog.accumulate_global(recs + (size_t)slot[j] * W + 2);
        }
    }
    if (lane == 0 && have > 0) atomicSub(tickets + way, have);        // tickets drawn and not used
    if (err) atomicOr(err_out, err);
}

// ---- FilterAndProject in two passes without a selection vector -------------------------------------------------------------
// Every CTA owns a contiguous chunk of rows.  Pass 1 evaluates the filter (flags, 1 byte per row) and counts the selected rows
// of the chunk; a scan of the chunk counts gives every chunk its first output row.  Pass 2 ranks the selected rows of a tile
// (ballot + a scan over the tile's (iteration, warp) cells), evaluates the projections and copies the pass-through channels
// straight to output row chunk_off + rank: output order = input order (PageProcessor.java:302-336).
// P supplies: static bool filter(cols, strs, row, err*), static void row(cols, strs, row, j, out, err*, nulls_seen*).
constexpr int FPC_R = 4;          // tile = FPC_R x 256 rows
constexpr int FPC_T = 256;

template <class P>
__device__ __forceinline__ void fp_filter_chunks_body(const DColumns& cols, const StrCols& strs, long long n, long long chunk, unsigned char* __restrict__ flags,
                                                      unsigned int* __restrict__ chunk_counts, unsigned int* __restrict__ err_out)
{
    __shared__ unsigned int warp_sel[FPC_T / 32];
    const long long begin = (long long)blockIdx.x * chunk, end = begin + chunk < n ? begin + chunk : n;
    unsigned int err = 0, mine = 0;
    for (long long row = begin + threadIdx.x; row < end; row += FPC_T) {
        bool s = P::filter(cols, strs, row, &err);
        flags[row] = s ? 1 : 0;
        mine += s ? 1u : 0u;
    }
    for (int off = 16; off > 0; off >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, off);
    if ((threadIdx.x & 31) == 0) warp_sel[threadIdx.x >> 5] = mine;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned int total = 0;
        for (int w = 0; w < FPC_T / 32; w++) total += warp_sel[w];
        chunk_counts[blockIdx.x] = total;
    }
    if (err) atomicOr(err_out, err);
}

template <class P>
__device__ __forceinline__ void fp_project_chunks_body(const DColumns& cols, const StrCols& strs, const unsigned char* __restrict__ flags, long long n, long long chunk,
                                                       const long long* __restrict__ chunk_off, const OutCols& out, unsigned int* __restrict__ err_out,
                                                       unsigned int* __restrict__ any_null)
{
    constexpr int NW = FPC_T / 32;
    __shared__ unsigned int cells[FPC_R * NW];     // selected rows per (iteration, warp), then their exclusive prefix
    __shared__ unsigned int tile_total;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long begin = (long long)blockIdx.x * chunk, end = begin + chunk < n ? begin + chunk : n;
    long long running = chunk_off[blockIdx.x];
    unsigned int err = 0, nulls_seen = 0;
    for (long long tile = begin; tile < end; tile += (long long)FPC_R * FPC_T) {
        bool sel[FPC_R];
        unsigned int rank[FPC_R];
#pragma unroll
        for (int i = 0; i < FPC_R; i++) {
            long long row = tile + (long long)i * FPC_T + threadIdx.x;
            sel[i] = row < end && flags[row] != 0;
            unsigned int b = __ballot_sync(0xffffffffu, sel[i]);
            rank[i] = __popc(b & ((1u << lane) - 1));
            if (lane == 0) cells[i * NW + warp] = __popc(b);
        }
        __syncthreads();
        if (warp == 0) {
            static_assert(FPC_R * NW == 32, "one cell per lane");
            unsigned int v = cells[lane], incl = v;
            for (int off = 1; off < 32; off <<= 1) {
                unsigned int u = __shfl_up_sync(0xffffffffu, incl, off);
                if (lane >= off) incl += u;
            }
            cells[lane] = incl - v;
            if (lane == 31) tile_total = incl;
        }
        __syncthreads();
#pragma unroll
        for (int i = 0; i < FPC_R; i++) {
            if (!sel[i]) continue;
            long long row = tile + (long long)i * FPC_T + threadIdx.x;
            P::row(cols, strs, row, running + cells[i * NW + warp] + rank[i], out, &err, &nulls_seen);
        }
        running += tile_total;
        __syncthreads();
    }
    if (err) atomicOr(err_out, err);
    if (nulls_seen) atomicOr(any_null, nulls_seen);
}

#endif  // __CUDACC__
#endif  // TG_DEVICE_LIB_CUH
