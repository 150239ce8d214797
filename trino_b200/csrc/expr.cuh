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

__device__ __forceinline__ uint32_t vm_temp_error(uint32_t errs, int t) { return (errs >> (4 * t)) & 0xFu; }

// Runs instructions [first, last) for one row.  `temps` points at this thread's column of the shared
// [temp][thread] array (stride tstride).  Returns the updated null bitmask; *errs holds the TG_ERR_BIT_* each temp
// carries (4 bits per temp, see vm_error): the caller raises those of the temps it reads.  `split` / `split_row`: see vm_fetch.
// A VARCHAR operand: a UTF8 channel (through `strs`), a pool constant or NULL
__device__ __forceinline__ StrRef vm_fetch_str(const DProgram* __restrict__ prog, const DOperand& o, const DColumns& cols, const StrCols& strs, int64_t row,
                                               bool* is_null)
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
    *is_null = true;
    return StrRef{nullptr, 0};
}

// One string operation: BOOLEAN result, NULL as for the numeric operations, never an error (its operands are never temps)
__device__ __forceinline__ Value vm_apply_str(const DProgram* __restrict__ prog, const DInsn& in, const DColumns& cols, const StrCols& strs, int64_t row)
{
    Value r;
    r.bits = 0;
    bool an, bn = true, cn = true;
    const StrRef a = vm_fetch_str(prog, in.a, cols, strs, row, &an);
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
            const StrRef b = vm_fetch_str(prog, in.b, cols, strs, row, &bn);
            const StrRef c = vm_fetch_str(prog, in.c, cols, strs, row, &cn);
            const bool n1 = an || bn, n2 = an || cn;
            const bool f1 = !n1 && tg_str_cmp(a, b) < 0, f2 = !n2 && tg_str_cmp(a, c) > 0;
            r.is_null = !(f1 || f2) && (n1 || n2);
            r.bits = (f1 || f2 || r.is_null) ? 0 : 1;
            return r;
        }
        default: {
            const StrRef b = vm_fetch_str(prog, in.b, cols, strs, row, &bn);
            r.is_null = an || bn;
            if (!r.is_null) r.bits = tg_str_cmp_op(in.op, a, b) ? 1 : 0;
            return r;
        }
    }
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

// STR: the program may hold string operations (FilterAndProject), read through `strs`.  DEC: the program may hold DECIMAL operations
// (FilterAndProject), whose temps keep their high words in `thi` (same layout as `temps`)
template <bool STR = false, bool DEC = false>
__device__ __forceinline__ uint32_t vm_run(const DProgram* __restrict__ prog, int first, int last, const DColumns& cols, int64_t row,
                                           int64_t* temps, int tstride, uint32_t nullbits, uint32_t* errs, int split = 0, int64_t split_row = 0,
                                           const StrCols* strs = nullptr, int64_t* thi = nullptr)
{
    uint32_t te = *errs;
    for (int pc = first; pc < last; pc++) {
        const DInsn& in = prog->insns[pc];
        if (DEC && prog->dec[pc].is_dec) {
            vm_step_dec(prog, in, prog->dec[pc], cols, row, temps, thi, tstride, &nullbits, &te);
            continue;
        }
        if (STR && in.vtype == TGPU_V_VARCHAR) {
            const Value v = vm_apply_str(prog, in, cols, *strs, row);
            temps[in.dst * tstride] = v.bits;
            nullbits = (nullbits & ~(1u << in.dst)) | ((v.is_null ? 1u : 0u) << in.dst);
            te &= ~(0xFu << (4 * in.dst));
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
            if (in.op == TGPU_EX_BETWEEN) {
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
// fail with the error one set of TG_ERR_BIT_* bits stands for (TGPU_OK when none is set)
int expr_raise(tgpu_ctx* ctx, int64_t errbits);

}  // namespace tg
