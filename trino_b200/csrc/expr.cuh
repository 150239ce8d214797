// expr.cuh — device-side evaluator of tgpu_expr_program (the GPU stand-in for the bytecode that
// ExpressionCompiler.compilePageProcessor emits, M/sql/gen/ExpressionCompiler.java:50-85).
//
// Semantics reproduced:
//   - SQL three-valued logic, NULL-propagating arithmetic/comparison, Kleene AND/OR
//     (M/sql/gen/columnar/AndFilterEvaluator.java, OrFilterEvaluator.java; filters reject NULL:
//      M/sql/gen/columnar/ColumnarFilter.java:27-30)
//   - BIGINT arithmetic is checked (Math.addExact/subtractExact/multiplyExact/negateExact,
//     M/type/BigintOperators.java:52-110) -> NUMERIC_VALUE_OUT_OF_RANGE / DIVISION_BY_ZERO; CAST(DOUBLE AS BIGINT) out of
//     range -> INVALID_CAST_ARGUMENT
//   - an error is raised only where the reference evaluates the operation that raises it: AND / OR short-circuit,
//     a NULL argument skips the remaining ones (vm_error in device_lib.cuh)
//   - DOUBLE arithmetic is IEEE-754 binary64 with NO fused multiply-add (M/type/DoubleOperators.java:66-86):
//     every operation goes through __dadd_rn/__dmul_rn/__ddiv_rn which the compiler never contracts.
//
// Execution model: one thread evaluates one row; the <= TGPU_MAX_TEMPS temporaries of a row live in shared
// memory ([temp][thread], conflict-free 64-bit accesses) so the instruction stream can index them
// dynamically; null flags of the temporaries are one register bitmask.
#pragma once
#include "common.cuh"

namespace tg {

struct DOperand {
    int32_t kind;
    int32_t index;
    int64_t imm;
};

struct DInsn {
    int32_t op, vtype, dst, pad;
    DOperand a, b, c;
};

// The source of a VARCHAR view: >= 0 a UTF8 channel, < 0 (but TGD_SRC_NONE) pool constant -(src + 1), TGD_SRC_NONE a NULL operand
// One CONCAT instruction: its result's pieces (piece slots and their sources); a_slot / b_slot: the slot operand a / b is captured in
// (-1: the operand is a CONCAT temp, whose pieces come first / last); inner: the result is read by a later CONCAT, so it carries its
// operands' errors only and that CONCAT checks the length over all pieces (the variadic call's one check)
struct DCat {
    int8_t n, inner, a_slot, b_slot;
    int8_t slot[TGD_MAX_PIECES];
    int32_t src[TGD_MAX_PIECES];
};
// One VARCHAR projection: its temp and pieces (slot -1: the view in the temp itself)
struct DStrOut {
    int32_t temp, n;
    int32_t slot[TGD_MAX_PIECES];
    int32_t src[TGD_MAX_PIECES];
};

struct DProgram {
    int32_t num_insns;
    int32_t num_filter_insns;   // instructions [0, num_filter_insns) compute the filter
    int32_t filter_temp;        // -1: no filter
    int32_t num_in_lists;
    int32_t in_offset[8];
    int32_t in_count[8];
    int64_t in_values[128];
    DInsn insns[TGPU_MAX_INSNS];
    // VARCHAR operands (FilterAndProject only): the UTF8 channels string operations read (slot k = channel str_channel[k];
    // str_slot[channel] = its slot or -1), the constant pool and the compiled LIKE patterns
    int32_t num_str_channels;
    int32_t str_channel[TGD_MAX_STR_CHANNELS];
    int8_t str_slot[TGPU_MAX_CHANNELS];
    int32_t num_strings;
    int32_t str_off[TGPU_MAX_STRINGS];
    int32_t str_len[TGPU_MAX_STRINGS];
    int32_t num_likes;
    int32_t str_pad;
    uint8_t str_bytes[TGPU_MAX_STRING_BYTES];
    DLike likes[TGPU_MAX_LIKE_PATTERNS];
    // DECIMAL operands (FilterAndProject only): the reference's method of each DECIMAL instruction (dec[i].is_dec), the high words of
    // long DECIMAL IN-list values, and what each temp holds after the program ran (temp_dec: 0 not a decimal, 1 short, 2 long).
    // long_temps: the temps that ever hold a long decimal (they get a high word)
    int32_t has_dec;
    uint32_t long_temps;
    int8_t temp_dec[TGPU_MAX_TEMPS];
    DDec dec[TGPU_MAX_INSNS];
    int64_t in_hi[128];
    // string functions (FilterAndProject only; has_strfn = 0: none).  A VARCHAR TEMP operand's imm names the source of the view the
    // temp holds (DStrSrc encoding).  A view temp holds (begin - source base) in its low and the length in its high 32 bits; a CONCAT
    // temp holds the total length, its pieces live in piece slots.  cat[i]: CONCAT instruction i; str_out[k]: the k-th VARCHAR projection
    int32_t has_strfn;
    int32_t num_piece_slots;
    int32_t num_str_outs;
    int32_t strfn_pad;
    DCat cat[TGPU_MAX_INSNS];
    DStrOut str_out[TGD_MAX_STR_OUTS];
};

// the program has an instruction over VARCHAR operands (or a LIKE)
bool expr_uses_strings(const DProgram& prog);
// the program has an instruction over DECIMAL operands or with a DECIMAL result
inline bool expr_uses_decimals(const DProgram& prog) { return prog.has_dec != 0; }


#if defined(__CUDACC__)

// Channels below `split` are read at `split_row`, the others at `row`: a join filter reads the build channels of the join-sources
// layout at the build position and the probe channels at the probe row.  split = 0 (the default) reads every channel at `row`.
__device__ __forceinline__ Value vm_fetch(const DOperand& o, const DColumns& cols, int64_t row, const int64_t* temps, int tstride, uint32_t nullbits,
                                          int split = 0, int64_t split_row = 0)
{
    Value v;
    switch (o.kind) {
        case TGPU_OPND_COLUMN: {
            const ColRef& c = cols.cols[o.index];
            const int64_t r = o.index < split ? split_row : row;
            v.is_null = !tg_valid(c.validity, r);
            v.bits = tg_load_i64(c, r);
            break;
        }
        case TGPU_OPND_TEMP:
            v.bits = temps[o.index * tstride];
            v.is_null = (nullbits >> o.index) & 1;
            break;
        case TGPU_OPND_CONST:
            v.bits = o.imm;
            v.is_null = false;
            break;
        default:   // TGPU_OPND_NULL / NONE
            v.bits = 0;
            v.is_null = true;
            break;
    }
    return v;
}

// error carried by operand o: temps carry one (4 bits per temp in `errs`), columns and constants none
__device__ __forceinline__ uint32_t vm_carried(const DOperand& o, uint32_t errs)
{
    return o.kind == TGPU_OPND_TEMP ? (errs >> (4 * o.index)) & 0xFu : 0u;
}

__device__ __forceinline__ uint32_t vm_temp_error(uint32_t errs, int t)
{
    const uint32_t e = (errs >> (4 * t)) & 0xFu;
    return e == TG_ERR_CODE_CONCAT ? (uint32_t)TG_ERR_BIT_CONCAT_TOO_LARGE : e;
}

// the first byte of a VARCHAR source (DCat::src encoding): a UTF8 channel's byte buffer or a pool constant
__device__ __forceinline__ const uint8_t* vm_src_base(const DProgram* __restrict__ prog, const StrCols& strs, int32_t src)
{
    if (src == TGD_SRC_NONE) return nullptr;
    if (src >= 0) return strs.bytes[prog->str_slot[src]];
    return prog->str_bytes + prog->str_off[-(src + 1)];
}

__device__ __forceinline__ int32_t vm_opnd_src(const DOperand& o)
{
    if (o.kind == TGPU_OPND_COLUMN) return o.index;
    if (o.kind == TGPU_OPND_CONST) return (int32_t)(-(o.imm + 1));
    if (o.kind == TGPU_OPND_TEMP) return (int32_t)o.imm;
    return TGD_SRC_NONE;
}

// A VARCHAR operand: a UTF8 channel (through `strs`), a pool constant, NULL, or a temp holding a view (begin - source base, length)
__device__ __forceinline__ StrRef vm_fetch_str(const DProgram* __restrict__ prog, const DOperand& o, const DColumns& cols, const StrCols& strs, int64_t row,
                                               bool* is_null, const int64_t* temps = nullptr, int tstride = 0, uint32_t nullbits = 0)
{
    if (o.kind == TGPU_OPND_COLUMN) {
        *is_null = !tg_valid(cols.cols[o.index].validity, row);
        if (*is_null) return StrRef{nullptr, 0};
        return tg_str(strs, prog->str_slot[o.index], row);
    }
    if (o.kind == TGPU_OPND_CONST) {
        *is_null = false;
        return StrRef{prog->str_bytes + prog->str_off[o.imm], prog->str_len[o.imm]};
    }
    if (o.kind == TGPU_OPND_TEMP) {
        *is_null = (nullbits >> o.index) & 1;
        if (*is_null) return StrRef{nullptr, 0};
        const int64_t v = temps[o.index * tstride];
        return StrRef{vm_src_base(prog, strs, (int32_t)o.imm) + (uint32_t)v, (int32_t)(v >> 32)};
    }
    *is_null = true;
    return StrRef{nullptr, 0};
}

// One string predicate: BOOLEAN result, NULL as for the numeric operations
__device__ __forceinline__ Value vm_apply_str(const DProgram* __restrict__ prog, const DInsn& in, const DColumns& cols, const StrCols& strs, int64_t row,
                                              const int64_t* temps = nullptr, int tstride = 0, uint32_t nullbits = 0)
{
    Value r;
    r.bits = 0;
    bool an, bn = true, cn = true;
    const StrRef a = vm_fetch_str(prog, in.a, cols, strs, row, &an, temps, tstride, nullbits);
    switch (in.op) {
        case TGPU_EX_IS_NULL: r.is_null = false; r.bits = an ? 1 : 0; return r;
        case TGPU_EX_IS_NOT_NULL: r.is_null = false; r.bits = an ? 0 : 1; return r;
        case TGPU_EX_LIKE:
            r.is_null = an;
            if (!an) r.bits = tg_like(prog->likes[in.b.imm], a) ? 1 : 0;
            return r;
        case TGPU_EX_IN: {
            r.is_null = an;
            if (an) return r;
            const int li = (int)in.b.imm;
            bool hit = false;
            for (int k = 0; k < prog->in_count[li] && !hit; k++) {
                const int64_t sidx = prog->in_values[prog->in_offset[li] + k];
                hit = tg_str_eq(a, StrRef{prog->str_bytes + prog->str_off[sidx], prog->str_len[sidx]});
            }
            r.bits = hit ? 1 : 0;
            return r;
        }
        case TGPU_EX_BETWEEN: {
            const StrRef b = vm_fetch_str(prog, in.b, cols, strs, row, &bn, temps, tstride, nullbits);
            const StrRef c = vm_fetch_str(prog, in.c, cols, strs, row, &cn, temps, tstride, nullbits);
            const bool n1 = an || bn, n2 = an || cn;
            const bool f1 = !n1 && tg_str_cmp(a, b) < 0, f2 = !n2 && tg_str_cmp(a, c) > 0;
            r.is_null = !(f1 || f2) && (n1 || n2);
            r.bits = (f1 || f2 || r.is_null) ? 0 : 1;
            return r;
        }
        default: {
            const StrRef b = vm_fetch_str(prog, in.b, cols, strs, row, &bn, temps, tstride, nullbits);
            r.is_null = an || bn;
            if (!r.is_null) r.bits = tg_str_cmp_op(in.op, a, b) ? 1 : 0;
            return r;
        }
    }
}

// The error a string predicate's result carries: its VARCHAR temp operands' (a view carries the error of a substr's start or length),
// by vm_error's rules
__device__ __forceinline__ uint32_t vm_error_str_pred(const DProgram* __restrict__ prog, const DInsn& in, const DColumns& cols, const StrCols& strs, int64_t row,
                                                      const int64_t* temps, int tstride, uint32_t nullbits, uint32_t te)
{
    const uint32_t ea = vm_carried(in.a, te);
    if (in.op == TGPU_EX_IS_NULL || in.op == TGPU_EX_IS_NOT_NULL || in.op == TGPU_EX_LIKE || in.op == TGPU_EX_IN) return ea;
    bool an, bn;
    const StrRef a = vm_fetch_str(prog, in.a, cols, strs, row, &an, temps, tstride, nullbits);
    if (ea || an) return ea;
    const uint32_t eb = vm_carried(in.b, te);
    if (in.op != TGPU_EX_BETWEEN || eb) return eb;
    const StrRef b = vm_fetch_str(prog, in.b, cols, strs, row, &bn, temps, tstride, nullbits);
    if (!bn && tg_str_cmp(b, a) > 0) return 0;
    return vm_carried(in.c, te);
}

// One instruction over VARCHAR operands in the interpreter: predicates, LENGTH, the views SUBSTR and the trims write (begin - source base
// in the low word, length in the high word), and CONCAT, which captures its new pieces in `pieces` and writes the total length
__device__ __forceinline__ void vm_step_str(const DProgram* __restrict__ prog, int pc, const DInsn& in, const DColumns& cols, const StrCols& strs, int64_t row,
                                            int64_t* temps, int tstride, uint32_t* nullbits, uint32_t* te, int64_t* pieces)
{
    int64_t r = 0;
    bool rn;
    uint32_t e;
    const uint32_t nb = *nullbits;
    switch (in.op) {
        case TGPU_EX_LENGTH: case TGPU_EX_SUBSTR: case TGPU_EX_LTRIM: case TGPU_EX_RTRIM: case TGPU_EX_TRIM: {
            bool an;
            const StrRef a = vm_fetch_str(prog, in.a, cols, strs, row, &an, temps, tstride, nb);
            const uint32_t ea = vm_carried(in.a, *te);
            if (in.op == TGPU_EX_LENGTH) {
                rn = an;
                e = ea;
                if (!an) r = tg_utf8_count(a);
                break;
            }
            StrRef v = a;
            if (in.op == TGPU_EX_SUBSTR) {
                const bool has_len = in.c.kind != TGPU_OPND_NONE;
                const Value b = vm_fetch(in.b, cols, row, temps, tstride, nb);
                Value c;
                c.bits = 0;
                c.is_null = false;
                if (has_len) c = vm_fetch(in.c, cols, row, temps, tstride, nb);
                rn = an || b.is_null || c.is_null;
                e = vm_error_call(an, ea, b.is_null, vm_carried(in.b, *te), has_len ? vm_carried(in.c, *te) : 0u, rn, 0u);
                if (!rn) v = tg_substr(a, b.bits, has_len, c.bits);
            }
            else {
                rn = an;
                e = ea;
                if (!rn) v = tg_trim(a, in.op != TGPU_EX_RTRIM, in.op != TGPU_EX_LTRIM);
            }
            if (!rn) r = (int64_t)(uint32_t)(v.p - vm_src_base(prog, strs, vm_opnd_src(in.a))) | ((int64_t)v.len << 32);
            break;
        }
        case TGPU_EX_CONCAT: {
            const DCat& k = prog->cat[pc];
            bool an, bn;
            StrRef a = StrRef{nullptr, 0}, b = StrRef{nullptr, 0};
            if (k.a_slot >= 0) a = vm_fetch_str(prog, in.a, cols, strs, row, &an, temps, tstride, nb);
            else an = (nb >> in.a.index) & 1;
            if (k.b_slot >= 0) b = vm_fetch_str(prog, in.b, cols, strs, row, &bn, temps, tstride, nb);
            else bn = (nb >> in.b.index) & 1;
            rn = an || bn;
            if (!rn) {
                if (k.a_slot >= 0) pieces[k.a_slot] = (int64_t)(uint32_t)(a.p - vm_src_base(prog, strs, vm_opnd_src(in.a))) | ((int64_t)a.len << 32);
                if (k.b_slot >= 0) pieces[k.b_slot] = (int64_t)(uint32_t)(b.p - vm_src_base(prog, strs, vm_opnd_src(in.b))) | ((int64_t)b.len << 32);
                for (int q = 0; q < k.n; q++) r += pieces[k.slot[q]] >> 32;
            }
            e = vm_error_call(an, vm_carried(in.a, *te), bn, vm_carried(in.b, *te), 0u, rn, !k.inner && r > TGD_MAX_CONCAT_BYTES ? TG_ERR_CODE_CONCAT : 0u);
            break;
        }
        default: {
            const Value v = vm_apply_str(prog, in, cols, strs, row, temps, tstride, nb);
            r = v.bits;
            rn = v.is_null;
            e = vm_error_str_pred(prog, in, cols, strs, row, temps, tstride, nb, *te);
            break;
        }
    }
    temps[in.dst * tstride] = r;
    *nullbits = (nb & ~(1u << in.dst)) | ((rn ? 1u : 0u) << in.dst);
    *te = (*te & ~(0xFu << (4 * in.dst))) | (e << (4 * in.dst));
}

// A DECIMAL operand (or the BIGINT operand of a cast to DECIMAL) as a 128-bit value: `lng` = a long decimal (a TGPU_INT128 channel's
// (high, low) cell, a temp's high-word lane `thi`, or a constant whose high word is `khi`); anything else is sign-extended
__device__ __forceinline__ DVal vm_fetch_dec(const DOperand& o, bool lng, long long khi, const DColumns& cols, int64_t row, const int64_t* temps,
                                             const int64_t* thi, int tstride, uint32_t nullbits)
{
    DVal v;
    v.v = U128{0ULL, 0ULL};
    v.is_null = true;
    switch (o.kind) {
        case TGPU_OPND_COLUMN: {
            const ColRef& c = cols.cols[o.index];
            v.is_null = !tg_valid(c.validity, row);
            if (lng) v.v = U128{(unsigned long long)((const int64_t*)c.data)[2 * row], (unsigned long long)((const int64_t*)c.data)[2 * row + 1]};
            else v.v = u128_sx(tg_load_i64(c, row));
            break;
        }
        case TGPU_OPND_TEMP:
            v.is_null = (nullbits >> o.index) & 1;
            v.v = lng ? U128{(unsigned long long)thi[o.index * tstride], (unsigned long long)temps[o.index * tstride]} : u128_sx(temps[o.index * tstride]);
            break;
        case TGPU_OPND_CONST:
            v.is_null = false;
            v.v = lng ? U128{(unsigned long long)khi, (unsigned long long)o.imm} : u128_sx(o.imm);
            break;
        default: break;
    }
    return v;
}

// One DECIMAL instruction of the interpreter: result value in temps / thi, NULL flag and error as the numeric ones
__device__ __forceinline__ void vm_step_dec(const DProgram* __restrict__ prog, const DInsn& in, const DDec& d, const DColumns& cols, int64_t row,
                                            int64_t* temps, int64_t* thi, int tstride, uint32_t* nullbits, uint32_t* te)
{
    const DVal a = vm_fetch_dec(in.a, d.la, d.hi[0], cols, row, temps, thi, tstride, *nullbits);
    DVal r;
    uint32_t e;
    if (in.op == TGPU_EX_IN) {
        r.is_null = a.is_null;
        r.v = U128{0ULL, 0ULL};
        const int li = (int)in.b.imm;
        bool hit = false;
        for (int k = 0; k < prog->in_count[li]; k++) {
            const int at = prog->in_offset[li] + k;
            const U128 x = d.la ? U128{(unsigned long long)prog->in_hi[at], (unsigned long long)prog->in_values[at]} : u128_sx(prog->in_values[at]);
            hit |= x.hi == a.v.hi && x.lo == a.v.lo;
        }
        r.v.lo = hit && !a.is_null ? 1ULL : 0ULL;
        e = vm_carried(in.a, *te);
    }
    else {
        const DVal b = vm_fetch_dec(in.b, d.lb, d.hi[1], cols, row, temps, thi, tstride, *nullbits);
        const DVal c = vm_fetch_dec(in.c, d.lc, d.hi[2], cols, row, temps, thi, tstride, *nullbits);
        uint32_t own = 0;
        r = vm_apply_dec(in.op, in.vtype, d, a, b, c, &own);
        e = vm_error_dec(in.op, a, vm_carried(in.a, *te), b, vm_carried(in.b, *te), vm_carried(in.c, *te), own);
    }
    temps[in.dst * tstride] = (int64_t)r.v.lo;
    thi[in.dst * tstride] = (int64_t)r.v.hi;
    *nullbits = (*nullbits & ~(1u << in.dst)) | ((r.is_null ? 1u : 0u) << in.dst);
    *te = (*te & ~(0xFu << (4 * in.dst))) | (e << (4 * in.dst));
}

// Runs instructions [first, last) for one row.  `temps` points at this thread's column of the shared
// [temp][thread] array (stride tstride).  Returns the updated null bitmask; *errs holds the TG_ERR_BIT_* each temp
// carries (4 bits per temp, see vm_error): the caller raises those of the temps it reads.  `split` / `split_row`: see vm_fetch.
// STR: the program may hold string operations (FilterAndProject), read through `strs`; `pieces`: the thread's concatenation piece slots.  DEC: the program may hold DECIMAL operations
// (FilterAndProject), whose temps keep their high words in `thi` (same layout as `temps`)
template <bool STR = false, bool DEC = false>
__device__ __forceinline__ uint32_t vm_run(const DProgram* __restrict__ prog, int first, int last, const DColumns& cols, int64_t row,
                                           int64_t* temps, int tstride, uint32_t nullbits, uint32_t* errs, int split = 0, int64_t split_row = 0,
                                           const StrCols* strs = nullptr, int64_t* thi = nullptr, int64_t* pieces = nullptr)
{
    uint32_t te = *errs;
    for (int pc = first; pc < last; pc++) {
        const DInsn& in = prog->insns[pc];
        if (DEC && prog->dec[pc].is_dec) {
            vm_step_dec(prog, in, prog->dec[pc], cols, row, temps, thi, tstride, &nullbits, &te);
            continue;
        }
        if (STR && in.vtype == TGPU_V_VARCHAR) {
            vm_step_str(prog, pc, in, cols, *strs, row, temps, tstride, &nullbits, &te, pieces);
            continue;
        }
        Value a = vm_fetch(in.a, cols, row, temps, tstride, nullbits, split, split_row);
        Value b = vm_fetch(in.b, cols, row, temps, tstride, nullbits, split, split_row);
        Value c;
        c.bits = 0; c.is_null = true;
        uint32_t own = 0, ec = 0;
        int64_t r;
        bool rn;
        if (in.op == TGPU_EX_IN) {
            rn = a.is_null;
            r = 0;
            if (!rn) {
                int li = (int)in.b.imm;
                int off = prog->in_offset[li], cnt = prog->in_count[li];
                bool hit = false;
                for (int k = 0; k < cnt; k++) {
                    int64_t v = prog->in_values[off + k];
                    hit |= in.vtype == TGPU_V_DOUBLE ? (__longlong_as_double(a.bits) == __longlong_as_double(v)) : (a.bits == v);
                }
                r = hit ? 1 : 0;
            }
        }
        else {
            if (in.op == TGPU_EX_BETWEEN || in.op == TGPU_EX_IF) {
                c = vm_fetch(in.c, cols, row, temps, tstride, nullbits, split, split_row);
                ec = vm_carried(in.c, te);
            }
            Value res = vm_apply(in.op, in.vtype, a, b, c, &own);
            r = res.bits;
            rn = res.is_null;
        }
        uint32_t e = vm_error(in.op, in.vtype, a, vm_carried(in.a, te), b, in.op == TGPU_EX_IN ? 0u : vm_carried(in.b, te), c, ec, own);
        temps[in.dst * tstride] = r;
        nullbits = (nullbits & ~(1u << in.dst)) | ((rn ? 1u : 0u) << in.dst);
        te = (te & ~(0xFu << (4 * in.dst))) | (e << (4 * in.dst));
    }
    *errs = te;
    return nullbits;
}

#endif  // __CUDACC__

// host side: validate + flatten a tgpu_expr_program into a DProgram (defined in expr.cu)
int expr_compile(tgpu_ctx* ctx, const tgpu_expr_program* program, DProgram* out, int32_t* max_channel);

// NVRTC code generation shared by the operators that specialise a program (defined in expr.cu): printf-style append, and the
// straight-line code of instructions [first, last) over locals c<k> / c<k>n (channel k's value and NULL flag) and t<i> / tn<i> / te<i>
// (temp i's value, NULL flag and carried error bits), which the caller declares
void fp_appendf(std::string& s, const char* fmt, ...);
void fp_emit_insns(std::string& s, const DProgram& prog, int first, int last);
// the declarations of every temp's locals (with the high words of long DECIMAL temps and the views of string functions)
void fp_emit_temps(std::string& s, const DProgram& prog);
// used[k] = true for every channel k that instructions [first, last) read as an operand
void fp_mark_columns(const DProgram& prog, int first, int last, bool* used);
// fail with the error one set of TG_ERR_BIT_* bits stands for (TGPU_OK when none is set)
int expr_raise(tgpu_ctx* ctx, int64_t errbits);

}  // namespace tg
