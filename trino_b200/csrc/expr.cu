// expr.cu — FilterAndProjectOperator / PageProcessor on the GPU.
//
// Reference: PageProcessor.createWorkProcessor (M/operator/project/PageProcessor.java:105-142): evaluate
// the filter to SelectedPositions, then every projection over the selected positions
// (ProjectSelectedPositions.processBatch :302-336); FilterAndProjectOperator
// (M/operator/FilterAndProjectOperator.java:60-95) wraps it.  Output rows keep input order.
#include "expr.cuh"
#include "jit.cuh"

namespace tg {

int expr_compile(tgpu_ctx* ctx, const tgpu_expr_program* p, DProgram* out, int32_t* max_channel)
{
    memset(out, 0, sizeof(*out));
    *max_channel = -1;
    if (!p) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "expression program is null");
    if (p->num_insns < 0 || p->num_insns > TGPU_MAX_INSNS) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "expression program has %d instructions (max %d)", p->num_insns, TGPU_MAX_INSNS);
    if (p->num_filter_insns < 0 || p->num_filter_insns > p->num_insns) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "num_filter_insns out of range");
    if (p->filter_temp >= TGPU_MAX_TEMPS) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "filter_temp out of range");
    if (p->num_in_lists > 8) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "more than 8 IN lists");
    out->num_insns = p->num_insns;
    out->num_filter_insns = p->filter_temp >= 0 ? p->num_filter_insns : 0;
    out->filter_temp = p->filter_temp;
    out->num_in_lists = p->num_in_lists;
    int off = 0;
    for (int i = 0; i < p->num_in_lists; i++) {
        if (off + p->in_lists[i].count > 128) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "IN lists hold more than 128 constants");
        out->in_offset[i] = off;
        out->in_count[i] = p->in_lists[i].count;
        for (int k = 0; k < p->in_lists[i].count; k++) out->in_values[off + k] = p->in_lists[i].values[k];
        off += p->in_lists[i].count;
    }
    auto conv = [&](const tgpu_operand& o, DOperand* d) -> int {
        d->kind = o.kind;
        d->index = o.index;
        d->imm = o.imm.i64;
        if (o.kind == TGPU_OPND_COLUMN) {
            if (o.index < 0 || o.index >= TGPU_MAX_CHANNELS) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "operand channel %d out of range", o.index);
            if (o.index > *max_channel) *max_channel = o.index;
        }
        else if (o.kind == TGPU_OPND_TEMP) {
            if (o.index < 0 || o.index >= TGPU_MAX_TEMPS) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "operand temp %d out of range", o.index);
        }
        else if (o.kind < 0 || o.kind > TGPU_OPND_NULL) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "bad operand kind %d", o.kind);
        return TGPU_OK;
    };
    for (int i = 0; i < p->num_insns; i++) {
        const tgpu_expr_insn& s = p->insns[i];
        DInsn& d = out->insns[i];
        if (s.dst < 0 || s.dst >= TGPU_MAX_TEMPS) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: dst temp out of range", i);
        if (s.vtype < 0 || s.vtype > TGPU_V_BOOLEAN) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: bad vtype", i);
        switch (s.op) {
            case TGPU_EX_MOV: case TGPU_EX_ADD: case TGPU_EX_SUB: case TGPU_EX_MUL: case TGPU_EX_DIV: case TGPU_EX_MOD: case TGPU_EX_NEG:
            case TGPU_EX_EQ: case TGPU_EX_NE: case TGPU_EX_LT: case TGPU_EX_LE: case TGPU_EX_GT: case TGPU_EX_GE:
            case TGPU_EX_AND: case TGPU_EX_OR: case TGPU_EX_NOT: case TGPU_EX_IS_NULL: case TGPU_EX_IS_NOT_NULL: case TGPU_EX_BETWEEN:
            case TGPU_EX_CAST_BIGINT_TO_DOUBLE: case TGPU_EX_CAST_DOUBLE_TO_BIGINT:
                break;
            case TGPU_EX_IN:
                if (s.b.imm.i64 < 0 || s.b.imm.i64 >= p->num_in_lists) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "insn %d: IN list index out of range", i);
                break;
            default:
                return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "insn %d: unsupported op %d", i, s.op);
        }
        d.op = s.op;
        d.vtype = s.vtype;
        d.dst = s.dst;
        TG_TRY(conv(s.a, &d.a));
        TG_TRY(conv(s.b, &d.b));
        TG_TRY(conv(s.c, &d.c));
        if (s.op == TGPU_EX_IN) d.b.kind = TGPU_OPND_CONST;
    }
    return TGPU_OK;
}

int expr_raise(tgpu_ctx* ctx, int64_t errbits)
{
    if (errbits & TG_ERR_BIT_DIV_ZERO) return tg_fail(ctx, TGPU_ERR_DIVISION_BY_ZERO, "Division by zero");
    if (errbits & TG_ERR_BIT_OVERFLOW) return tg_fail(ctx, TGPU_ERR_NUMERIC_VALUE_OUT_OF_RANGE, "bigint arithmetic overflow");
    if (errbits & TG_ERR_BIT_INVALID_CAST) return tg_fail(ctx, TGPU_ERR_INVALID_CAST_ARGUMENT, "Unable to cast double to bigint");
    return TGPU_OK;
}

// ---- NVRTC code generation of programs -------------------------------------------------------------------------------
void fp_appendf(std::string& s, const char* fmt, ...)
{
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    s += buf;
}

static std::string fp_operand(const DOperand& o)
{
    char buf[128];
    switch (o.kind) {
        case TGPU_OPND_COLUMN: snprintf(buf, sizeof(buf), "Value{c%d, c%dn}", o.index, o.index); break;
        case TGPU_OPND_TEMP: snprintf(buf, sizeof(buf), "Value{t%d, tn%d}", o.index, o.index); break;
        case TGPU_OPND_CONST: snprintf(buf, sizeof(buf), "Value{(long long)0x%llxULL, false}", (unsigned long long)o.imm); break;
        default: snprintf(buf, sizeof(buf), "Value{0, true}"); break;
    }
    return buf;
}

// the error operand o carries (see vm_error): a temp's, never a column's or a constant's
static std::string fp_operand_error(const DOperand& o)
{
    return o.kind == TGPU_OPND_TEMP ? "te" + std::to_string(o.index) : "0u";
}

void fp_emit_insns(std::string& s, const DProgram& prog, int first, int last)
{
    for (int i = first; i < last; i++) {
        const DInsn& in = prog.insns[i];
        if (in.op == TGPU_EX_IN) {
            int li = (int)in.b.imm;
            fp_appendf(s, "    { Value a = %s; bool hit = false;\n", fp_operand(in.a).c_str());
            for (int k = 0; k < prog.in_count[li]; k++) {
                unsigned long long c = (unsigned long long)prog.in_values[prog.in_offset[li] + k];
                if (in.vtype == TGPU_V_DOUBLE) fp_appendf(s, "      hit |= __longlong_as_double(a.bits) == __longlong_as_double((long long)0x%llxULL);\n", c);
                else fp_appendf(s, "      hit |= a.bits == (long long)0x%llxULL;\n", c);
            }
            fp_appendf(s, "      t%d = hit ? 1 : 0; tn%d = a.is_null; te%d = %s; }\n", in.dst, in.dst, in.dst, fp_operand_error(in.a).c_str());
        }
        else {
            // operands are read into locals first: dst may be one of them, and vm_error needs their values
            fp_appendf(s, "    { Value a = %s, b = %s, c = %s; unsigned int e = 0; Value x = vm_apply(%d, %d, a, b, c, &e);\n", fp_operand(in.a).c_str(),
                       fp_operand(in.b).c_str(), fp_operand(in.c).c_str(), in.op, in.vtype);
            fp_appendf(s, "      e = vm_error(%d, %d, a, %s, b, %s, c, %s, e); t%d = x.bits; tn%d = x.is_null; te%d = e; }\n", in.op, in.vtype,
                       fp_operand_error(in.a).c_str(), fp_operand_error(in.b).c_str(), fp_operand_error(in.c).c_str(), in.dst, in.dst, in.dst);
        }
    }
}

}  // namespace tg

namespace {

using namespace tg;

constexpr int FP_THREADS = 256;

// ---- NVRTC specialisation of the two PageProcessor kernels ----------------------------------------------------------

// filter pass: one row per thread, writes 1/0 selection flags
__global__ void __launch_bounds__(FP_THREADS) fp_filter_kernel(const DProgram* __restrict__ prog, DColumns cols, int64_t n, uint8_t* __restrict__ flags,
                                                              unsigned int* __restrict__ err_out)
{
    __shared__ int64_t temps[TGPU_MAX_TEMPS * FP_THREADS];
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    uint32_t err = 0;
    for (; i < n; i += stride) {
        uint32_t te = 0;
        uint32_t nb = vm_run(prog, 0, prog->num_filter_insns, cols, i, temps + threadIdx.x, FP_THREADS, 0, &te);
        int ft = prog->filter_temp;
        err |= vm_temp_error(te, ft);
        bool sel = !((nb >> ft) & 1) && temps[ft * FP_THREADS + threadIdx.x] != 0;
        flags[i] = sel ? 1 : 0;
    }
    if (err) atomicOr(err_out, err);
}

// projection pass: output row j <- input row sel[j] (sel == nullptr: identity)
__global__ void __launch_bounds__(FP_THREADS) fp_project_kernel(const DProgram* __restrict__ prog, DColumns cols, const int32_t* __restrict__ sel, int64_t m,
                                                               OutCols out, unsigned int* __restrict__ err_out, unsigned int* __restrict__ any_null)
{
    __shared__ int64_t temps[TGPU_MAX_TEMPS * FP_THREADS];
    int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    uint32_t err = 0, nulls_seen = 0;
    for (; j < m; j += stride) {
        int64_t row = sel ? sel[j] : j;
        int64_t* t = temps + threadIdx.x;
        uint32_t te = 0;
        uint32_t nb = vm_run(prog, 0, prog->num_insns, cols, row, t, FP_THREADS, 0, &te);
        for (int c = 0; c < out.count; c++) {
            int tp = out.temp[c];
            err |= vm_temp_error(te, tp);
            bool isn = (nb >> tp) & 1;
            int64_t v = isn ? 0 : t[tp * FP_THREADS];
            if (out.vtype[c] == TGPU_V_BOOLEAN) ((int8_t*)out.data[c])[j] = (int8_t)v;
            else ((int64_t*)out.data[c])[j] = v;
            out.nullmap[c][j] = isn ? 1 : 0;
            if (isn) nulls_seen |= 1u << c;
        }
    }
    if (err) atomicOr(err_out, err);
    if (nulls_seen) atomicOr(any_null, nulls_seen);
}


// straight-line typed code for one program over channels of the given element sizes
static std::string gen_fp_source(const DProgram& prog, const int* elems, int num_channels, uint32_t nullable_mask, const std::vector<int>& pass_channels)
{
    std::string s;
    bool used[TGPU_MAX_CHANNELS] = {false};
    for (int i = 0; i < prog.num_insns; i++) {
        const DOperand* ops[3] = {&prog.insns[i].a, &prog.insns[i].b, &prog.insns[i].c};
        for (auto* o : ops)
            if (o->kind == TGPU_OPND_COLUMN) used[o->index] = true;
    }
    std::string loads, temps;
    for (int c = 0; c < num_channels && c < TGPU_MAX_CHANNELS; c++) {
        if (!used[c]) continue;
        fp_appendf(loads, "    const long long c%d = tg_load_elem<%d>(cols.cols[%d].data, row);", c, elems[c], c);
        if ((nullable_mask >> c) & 1) fp_appendf(loads, " const bool c%dn = !tg_valid(cols.cols[%d].validity, row);\n", c, c);
        else fp_appendf(loads, " const bool c%dn = false;\n", c);
    }
    for (int t = 0; t < TGPU_MAX_TEMPS; t++) fp_appendf(temps, "    long long t%d = 0; bool tn%d = true; unsigned int te%d = 0;\n", t, t, t);
    // value, NULL flag and carried error of the temp behind each computed output column (the only errors a projection raises)
    std::string output_switch = "    for (int c = 0; c < out.count; c++) {\n      long long v = 0; bool isn = true; unsigned int e = 0;\n      switch (out.temp[c]) {\n";
    for (int t = 0; t < TGPU_MAX_TEMPS; t++) fp_appendf(output_switch, "        case %d: v = t%d; isn = tn%d; e = te%d; break;\n", t, t, t, t);
    output_switch += "      }\n      err |= e;\n      if (isn) v = 0;\n";
    // filter kernel
    s += "extern \"C\" __global__ void __launch_bounds__(256) tg_fp_filter_jit(DColumns cols, long long n, unsigned char* flags, unsigned int* err_out) {\n";
    s += "  unsigned int err = 0;\n  long long stride = (long long)gridDim.x * blockDim.x;\n";
    s += "  for (long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x; row < n; row += stride) {\n";
    s += loads + temps;
    fp_emit_insns(s, prog, 0, prog.num_filter_insns);
    if (prog.filter_temp >= 0) fp_appendf(s, "    err |= te%d;\n    flags[row] = (!tn%d && t%d != 0) ? 1 : 0;\n", prog.filter_temp, prog.filter_temp, prog.filter_temp);
    else s += "    flags[row] = 1;\n";
    s += "  }\n  if (err) atomicOr(err_out, err);\n}\n";
    // projection kernel
    s += "extern \"C\" __global__ void __launch_bounds__(256) tg_fp_project_jit(DColumns cols, const int* sel, long long m, OutCols out, unsigned int* err_out, unsigned int* any_null) {\n";
    s += "  unsigned int err = 0, nulls_seen = 0;\n  long long stride = (long long)gridDim.x * blockDim.x;\n";
    s += "  for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < m; j += stride) {\n";
    s += "    const long long row = sel ? sel[j] : j;\n";
    s += loads + temps;
    fp_emit_insns(s, prog, 0, prog.num_insns);
    s += output_switch;
    s += "      if (out.vtype[c] == TGD_V_BOOLEAN) ((signed char*)out.data[c])[j] = (signed char)v; else ((long long*)out.data[c])[j] = v;\n";
    s += "      out.nullmap[c][j] = isn ? 1 : 0;\n      if (isn) nulls_seen |= 1u << c;\n    }\n";
    s += "  }\n  if (err) atomicOr(err_out, err);\n  if (nulls_seen) atomicOr(any_null, nulls_seen);\n}\n";
    // chunked two-pass form (no selection vector): per-row functors + the two kernels around the bodies of device_lib.cuh
    bool chunkable = prog.filter_temp >= 0;
    for (int ch : pass_channels)
        if (ch < 0 || ch >= num_channels || elems[ch] == 0) chunkable = false;     // variable-width pass-through: not in this form
    if (!chunkable) return s;
    s += "struct FProg {\n";
    s += "  static __device__ __forceinline__ bool filter(const DColumns& cols, long long row, unsigned int* errp) {\n    unsigned int err = 0;\n";
    s += loads + temps;
    fp_emit_insns(s, prog, 0, prog.num_filter_insns);
    fp_appendf(s, "    err |= te%d;\n    *errp |= err;\n    return !tn%d && t%d != 0;\n  }\n", prog.filter_temp, prog.filter_temp, prog.filter_temp);
    s += "  static __device__ __forceinline__ void row(const DColumns& cols, long long row, long long j, const OutCols& out, unsigned int* errp, unsigned int* nullsp) {\n";
    s += "    unsigned int err = 0, nulls_seen = 0;\n";
    s += loads + temps;
    fp_emit_insns(s, prog, 0, prog.num_insns);
    s += output_switch;
    s += "      if (out.vtype[c] == TGD_V_BOOLEAN) ((signed char*)out.data[c])[j] = (signed char)v; else ((long long*)out.data[c])[j] = v;\n";
    s += "      out.nullmap[c][j] = isn ? 1 : 0;\n      if (isn) nulls_seen |= 1u << c;\n    }\n";
    for (size_t k = 0; k < pass_channels.size(); k++) {
        int ch = pass_channels[k];
        const char* ty = elems[ch] == 16 ? "int4" : elems[ch] == 8 ? "long long" : elems[ch] == 4 ? "int" : elems[ch] == 2 ? "short" : "signed char";
        fp_appendf(s, "    ((%s*)out.pass_data[%d])[j] = ((const %s*)cols.cols[%d].data)[row];\n", ty, (int)k, ty, ch);
        if ((nullable_mask >> ch) & 1) fp_appendf(s, "    out.pass_nullmap[%d][j] = tg_valid(cols.cols[%d].validity, row) ? 0 : 1;\n", (int)k, ch);
    }
    s += "    *errp |= err;\n    *nullsp |= nulls_seen;\n  }\n};\n";
    s += "extern \"C\" __global__ void __launch_bounds__(256) tg_fp_filter_chunks_jit(DColumns cols, long long n, long long chunk, unsigned char* flags, "
         "unsigned int* counts, unsigned int* err_out) { fp_filter_chunks_body<FProg>(cols, n, chunk, flags, counts, err_out); }\n";
    s += "extern \"C\" __global__ void __launch_bounds__(256) tg_fp_project_chunks_jit(DColumns cols, const unsigned char* flags, long long n, long long chunk, "
         "const long long* chunk_off, OutCols out, unsigned int* err_out, unsigned int* any_null) "
         "{ fp_project_chunks_body<FProg>(cols, flags, n, chunk, chunk_off, out, err_out, any_null); }\n";
    return s;
}

// exclusive scan of the chunk counts of the chunked FilterAndProject form (one CTA)
__global__ void __launch_bounds__(256) fp_chunk_scan_kernel(const unsigned int* __restrict__ counts, int chunks, long long* __restrict__ chunk_off,
                                                            long long* __restrict__ total)
{
    __shared__ long long part[256];
    const int t = threadIdx.x;
    const int per = (chunks + 255) / 256;
    const int b0 = min(chunks, t * per), b1 = min(chunks, b0 + per);
    long long sum = 0;
    for (int b = b0; b < b1; b++) sum += counts[b];
    part[t] = sum;
    __syncthreads();
    for (int off = 1; off < 256; off <<= 1) {
        long long v = t >= off ? part[t - off] : 0;
        __syncthreads();
        part[t] += v;
        __syncthreads();
    }
    long long run = part[t] - sum;
    for (int b = b0; b < b1; b++) {
        chunk_off[b] = run;
        run += counts[b];
    }
    if (t == 255) *total = part[255];
}

struct FilterProjectOp : tgpu_op {
    DProgram host_prog;
    DevBuf d_prog;
    std::vector<tgpu_projection> projections;
    int32_t max_channel = -1;
    std::vector<OwnedPage*> pending;
    size_t next_out = 0;
    bool finishing = false;

    explicit FilterProjectOp(tgpu_ctx* c) : tgpu_op(c) {}
    ~FilterProjectOp() override { for (size_t i = next_out; i < pending.size(); i++) delete pending[i]; }

    bool needs_input() override { return !finishing && next_out >= pending.size(); }

    int add_input(const tgpu_page* page) override
    {
        for (size_t i = next_out; i < pending.size(); i++) delete pending[i];   // pages the caller never took
        pending.clear();
        next_out = 0;
        int64_t n = page->num_rows;
        if (n == 0) return TGPU_OK;
        if (n > (int64_t)INT32_MAX) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "page has more than 2^31-1 positions");
        DevPage in;
        TG_TRY(tg_ingest_page(ctx, page, &in));
        if (max_channel >= (int32_t)in.cols.size()) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "program reads channel %d, page has %zu", max_channel, in.cols.size());
        DColumns cols;
        memset(&cols, 0, sizeof(cols));
        for (size_t c = 0; c < in.cols.size() && c < TGPU_MAX_CHANNELS; c++) {
            if ((int32_t)c <= max_channel && in.cols[c].type == TGPU_UTF8) {
                // only pass-through is allowed for variable-width columns; computed operands were validated below
            }
            cols.cols[c] = tg_colref(in.cols[c]);
        }
        for (int i = 0; i < host_prog.num_insns; i++) {
            const DOperand* ops[3] = {&host_prog.insns[i].a, &host_prog.insns[i].b, &host_prog.insns[i].c};
            for (auto* o : ops)
                if (o->kind == TGPU_OPND_COLUMN && (in.cols[o->index].elem_size() == 0 || in.cols[o->index].elem_size() == 16 || in.cols[o->index].type == TGPU_FLOAT32))
                    return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "expressions over variable-width / 128-bit / REAL channel %d are not supported on the GPU path", o->index);
        }
        unsigned int* d_err = ctx->d_scratch->fp_flags;
        unsigned int* d_anynull = d_err + 1;
        TG_CUDA(ctx, cudaMemsetAsync(d_err, 0, 8, ctx->stream));
        const DProgram* dp = d_prog.as<DProgram>();
        int grid = tg_grid(ctx, n, FP_THREADS, 8);

        int64_t m = n;
        DevBuf sel;
        const int32_t* d_sel = nullptr;
        if (host_prog.filter_temp >= 0) {
            TG_TRY(jit_prepare(in));
            if (jit_project_chunks) {
                bool handled = false;
                TG_TRY(add_input_chunked(in, cols, n, d_err, d_anynull, &handled, &m));
                if (handled) return TGPU_OK;
                // every row passed the filter: fall through to the identity form (blocks pass through, no copies)
            }
        }
        if (host_prog.filter_temp >= 0 && !jit_project_chunks) {
            DevBuf flags;
            TG_TRY(flags.alloc(ctx, (size_t)n));
            TG_TRY(jit_prepare(in));
            if (jit_filter) {
                long long n_arg = n;
                unsigned char* f_arg = flags.as<unsigned char>();
                void* params[4] = {&cols, &n_arg, &f_arg, &d_err};
                TG_TRY(jit_launch(ctx, jit_filter, tg_grid(ctx, n, FP_THREADS, jit_blocks_per_sm(jit_filter, FP_THREADS, 0)), FP_THREADS, 0, params));
            }
            else TG_LAUNCH(ctx, fp_filter_kernel, grid, FP_THREADS, 0, dp, cols, n, flags.as<uint8_t>(), d_err);
            long long* d_count = &ctx->d_scratch->fp_count;
            TG_TRY(tg_flagged_positions(ctx, flags.as<uint8_t>(), n, &sel, d_count));
            TG_TRY(tg_read_i64(ctx, d_count, &m));
            int64_t errw = 0;
            TG_TRY(tg_read_i64(ctx, d_err, &errw));
            TG_TRY(raise(errw));
            if (m == 0) return TGPU_OK;
            if (m < n) d_sel = sel.as<int32_t>();
        }

        DevPage outp;
        outp.rows = m;
        outp.cols.resize(projections.size());
        ComputedCols cc;
        for (size_t pi = 0; pi < projections.size(); pi++) {
            const tgpu_projection& pr = projections[pi];
            if (pr.kind == 0) {
                if (pr.index < 0 || pr.index >= (int32_t)in.cols.size()) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "projection channel out of range");
                if (!d_sel) outp.cols[pi] = in.cols[pr.index];       // InputPageProjection on all positions: the block itself
                else TG_TRY(tg_gather_column(ctx, in.cols[pr.index], d_sel, m, false, &outp.cols[pi]));
            }
            else TG_TRY(add_computed(pr, m, (int)pi, &outp, &cc));
        }
        if (cc.oc.count > 0) {
            int pgrid = tg_grid(ctx, m, FP_THREADS, 8);
            TG_TRY(jit_prepare(in));
            if (jit_project) {
                long long m_arg = m;
                void* params[6] = {&cols, &d_sel, &m_arg, &cc.oc, &d_err, &d_anynull};
                TG_TRY(jit_launch(ctx, jit_project, tg_grid(ctx, m, FP_THREADS, jit_blocks_per_sm(jit_project, FP_THREADS, 0)), FP_THREADS, 0, params));
            }
            else TG_LAUNCH(ctx, fp_project_kernel, pgrid, FP_THREADS, 0, dp, cols, d_sel, m, cc.oc, d_err, d_anynull);
            TG_TRY(finish_computed(cc, d_err, &outp));
        }
        pending.push_back(tg_make_owned_page(std::move(outp)));
        return TGPU_OK;
    }

    // computed projection columns of one output page: their buffers as the project kernel sees them, and where they go
    struct ComputedCols {
        OutCols oc;
        std::vector<std::shared_ptr<DevBuf>> nullmaps;   // one byte per row, 1 = NULL
        std::vector<int> at;                             // output column of each computed column
        ComputedCols() { memset(&oc, 0, sizeof(oc)); }
    };

    // allocate output column `pi` (m rows) of computed projection `pr` and its byte null map
    int add_computed(const tgpu_projection& pr, int64_t m, int pi, DevPage* outp, ComputedCols* cc)
    {
        DevColumn& c = outp->cols[pi];
        c.type = pr.vtype == TGPU_V_DOUBLE ? TGPU_FLOAT64 : pr.vtype == TGPU_V_BOOLEAN ? TGPU_INT8 : TGPU_INT64;
        c.length = m;
        c.own_data = std::make_shared<DevBuf>();
        TG_TRY(c.own_data->alloc(ctx, (size_t)m * c.elem_size()));
        c.data = c.own_data->p;
        auto nm = std::make_shared<DevBuf>();
        TG_TRY(nm->alloc(ctx, (size_t)m));
        int k = cc->oc.count++;
        cc->oc.temp[k] = pr.index;
        cc->oc.vtype[k] = pr.vtype;
        cc->oc.data[k] = c.own_data->p;
        cc->oc.nullmap[k] = nm->as<uint8_t>();
        cc->nullmaps.push_back(std::move(nm));
        cc->at.push_back(pi);
        return TGPU_OK;
    }

    // after the project kernel: raise its error bits, then give validity to the computed columns that hold a NULL
    int finish_computed(const ComputedCols& cc, unsigned int* d_err, DevPage* outp)
    {
        int64_t word = 0;
        TG_TRY(tg_read_i64(ctx, d_err, &word));
        TG_TRY(raise(word & 0xFFFFFFFFLL));
        uint32_t any_null = (uint32_t)((uint64_t)word >> 32);
        for (int k = 0; k < cc.oc.count; k++)
            if ((any_null >> k) & 1) TG_TRY(attach_validity(cc.nullmaps[k]->as<uint8_t>(), &outp->cols[cc.at[k]]));
        return TGPU_OK;
    }

    // pack the byte null map of c's rows into its validity bitmap
    int attach_validity(const uint8_t* nullmap, DevColumn* c)
    {
        c->own_validity = std::make_shared<DevBuf>();
        TG_TRY(c->own_validity->alloc(ctx, (size_t)((c->length + 7) / 8)));
        TG_TRY(tg_pack_nullmap(ctx, nullmap, c->length, c->own_validity->as<uint8_t>()));
        c->validity = c->own_validity->as<uint8_t>();
        return TGPU_OK;
    }

    // chunked two-pass form: handled = false (and *m_out = n) when every row is selected
    int add_input_chunked(const DevPage& in, const DColumns& cols, int64_t n, unsigned int* d_err, unsigned int* d_anynull, bool* handled, int64_t* m_out)
    {
        *handled = false;
        const int64_t tile = (int64_t)FPC_R * FPC_T;
        int per_sm = std::min(jit_blocks_per_sm(jit_filter_chunks, FPC_T, 0), jit_blocks_per_sm(jit_project_chunks, FPC_T, 0));
        int64_t want = std::min<int64_t>(tg_div_up(n, tile), (int64_t)ctx->sm_count * per_sm);
        long long chunk = (long long)(tg_div_up(tg_div_up(n, want), tile) * tile);
        int chunks = (int)tg_div_up(n, chunk);
        DevBuf flags, counts, chunk_off, d_total;
        TG_TRY(flags.alloc(ctx, (size_t)n));
        TG_TRY(counts.alloc(ctx, (size_t)chunks * 4));
        TG_TRY(chunk_off.alloc(ctx, (size_t)chunks * 8));
        TG_TRY(d_total.alloc(ctx, 8));
        long long n_arg = n;
        {
            DColumns c = cols;
            unsigned char* f_arg = flags.as<unsigned char>();
            unsigned int* cnt_arg = counts.as<unsigned int>();
            void* params[6] = {&c, &n_arg, &chunk, &f_arg, &cnt_arg, &d_err};
            TG_TRY(jit_launch(ctx, jit_filter_chunks, chunks, FPC_T, 0, params));
        }
        TG_LAUNCH(ctx, fp_chunk_scan_kernel, 1, 256, 0, counts.as<unsigned int>(), chunks, chunk_off.as<long long>(), d_total.as<long long>());
        int64_t m = 0, errw = 0;
        TG_TRY(tg_read_i64(ctx, d_total.p, &m));
        TG_TRY(tg_read_i64(ctx, d_err, &errw));
        TG_TRY(raise(errw & 0xFFFFFFFFLL));
        *m_out = m;
        if (m == n) return TGPU_OK;
        *handled = true;
        if (m == 0) return TGPU_OK;
        DevPage outp;
        outp.rows = m;
        outp.cols.resize(projections.size());
        ComputedCols cc;
        OutCols& oc = cc.oc;
        std::vector<std::shared_ptr<DevBuf>> pass_nullmaps;
        std::vector<int> pass_at;
        for (size_t pi = 0; pi < projections.size(); pi++) {
            const tgpu_projection& pr = projections[pi];
            if (pr.kind == 0) {
                if (pr.index < 0 || pr.index >= (int32_t)in.cols.size()) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "projection channel out of range");
                const DevColumn& src = in.cols[pr.index];
                DevColumn& c = outp.cols[pi];
                c.type = src.type;
                c.length = m;
                c.own_data = std::make_shared<DevBuf>();
                TG_TRY(c.own_data->alloc(ctx, (size_t)m * src.elem_size()));
                c.data = c.own_data->p;
                int k = oc.pass_count++;
                oc.pass_data[k] = c.own_data->p;
                std::shared_ptr<DevBuf> nm;
                if (src.validity) {
                    nm = std::make_shared<DevBuf>();
                    TG_TRY(nm->alloc(ctx, (size_t)m));
                    oc.pass_nullmap[k] = nm->as<uint8_t>();
                }
                pass_nullmaps.push_back(nm);
                pass_at.push_back((int)pi);
            }
            else TG_TRY(add_computed(pr, m, (int)pi, &outp, &cc));
        }
        {
            DColumns c = cols;
            const unsigned char* f_arg = flags.as<unsigned char>();
            const long long* off_arg = chunk_off.as<long long>();
            void* params[8] = {&c, &f_arg, &n_arg, &chunk, &off_arg, &oc, &d_err, &d_anynull};
            TG_TRY(jit_launch(ctx, jit_project_chunks, chunks, FPC_T, 0, params));
        }
        TG_TRY(finish_computed(cc, d_err, &outp));
        for (int k = 0; k < oc.pass_count; k++)
            if (pass_nullmaps[k]) TG_TRY(attach_validity(pass_nullmaps[k]->as<uint8_t>(), &outp.cols[pass_at[k]]));
        pending.push_back(tg_make_owned_page(std::move(outp)));
        return TGPU_OK;
    }

    // kernels specialised for this program and this page's channel types / nullability (NVRTC, cached)
    void* jit_filter = nullptr;
    void* jit_project = nullptr;
    void* jit_filter_chunks = nullptr;      // chunked two-pass form (nullptr: not applicable to this program / page shape)
    void* jit_project_chunks = nullptr;
    std::string jit_key;
    std::vector<int> pass_channels() const
    {
        std::vector<int> v;
        for (auto& pr : projections)
            if (pr.kind == 0) v.push_back(pr.index);
        return v;
    }
    int jit_prepare(const DevPage& in)
    {
        if (!jit_available()) { jit_filter = jit_project = nullptr; return TGPU_OK; }
        int elems[TGPU_MAX_CHANNELS] = {0};
        uint32_t nullable = 0;
        std::string key;
        for (size_t c = 0; c < in.cols.size() && c < TGPU_MAX_CHANNELS; c++) {
            elems[c] = in.cols[c].elem_size();
            if (in.cols[c].validity) nullable |= 1u << c;
            key += (char)('0' + elems[c]);
        }
        key += ":" + std::to_string(nullable);
        if (key == jit_key && jit_filter) return TGPU_OK;
        std::vector<int> pass = pass_channels();
        std::string src = gen_fp_source(host_prog, elems, (int)in.cols.size(), nullable, pass);
        TG_TRY(jit_get_function(ctx, src, "tg_fp_filter_jit", &jit_filter));
        TG_TRY(jit_get_function(ctx, src, "tg_fp_project_jit", &jit_project));
        jit_filter_chunks = jit_project_chunks = nullptr;
        if (src.find("tg_fp_project_chunks_jit") != std::string::npos && pass.size() <= TGPU_MAX_CHANNELS && !getenv("TGPU_FP_SELECTION_VECTOR")) {
            TG_TRY(jit_get_function(ctx, src, "tg_fp_filter_chunks_jit", &jit_filter_chunks));
            TG_TRY(jit_get_function(ctx, src, "tg_fp_project_chunks_jit", &jit_project_chunks));
        }
        jit_key = key;
        return TGPU_OK;
    }

    int raise(int64_t errbits) { return expr_raise(ctx, errbits); }

    int get_output(OwnedPage** out) override
    {
        *out = nullptr;
        if (next_out < pending.size()) *out = pending[next_out++];
        return TGPU_OK;
    }
    int finish() override { finishing = true; return TGPU_OK; }
    bool is_finished() override { return finishing && next_out >= pending.size(); }
};

}  // namespace

extern "C" int tgpu_filter_project_create(tgpu_ctx* ctx, const tgpu_expr_program* program, tgpu_op** out)
{
    if (!ctx || !program || !out) return TGPU_ERR_INVALID_ARGUMENT;
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    std::unique_ptr<FilterProjectOp> op(new FilterProjectOp(ctx));
    TG_TRY(tg::expr_compile(ctx, program, &op->host_prog, &op->max_channel));
    if (program->num_projections > TGPU_MAX_CHANNELS) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "more than %d projections", TGPU_MAX_CHANNELS);
    for (int i = 0; i < program->num_projections; i++) {
        const tgpu_projection& p = program->projections[i];
        if (p.kind == 1 && (p.index < 0 || p.index >= TGPU_MAX_TEMPS)) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "projection temp out of range");
        op->projections.push_back(p);
    }
    TG_TRY(op->d_prog.alloc(ctx, sizeof(tg::DProgram)));
    TG_CUDA(ctx, cudaMemcpyAsync(op->d_prog.p, &op->host_prog, sizeof(tg::DProgram), cudaMemcpyHostToDevice, ctx->stream));
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    *out = op.release();
    return TGPU_OK;
}

extern "C" int tgpu_jit_selftest_filter_project(const tgpu_expr_program* program, const int32_t* channel_types, int32_t num_channels, uint32_t nullable_mask,
                                                int64_t* cubin_bytes, char* source_out, int64_t source_cap)
{
    if (!program || !channel_types || !cubin_bytes) return TGPU_ERR_INVALID_ARGUMENT;
    tgpu_ctx fake;
    tg::DProgram prog;
    int32_t max_channel = -1;
    int st = tg::expr_compile(&fake, program, &prog, &max_channel);
    if (st != TGPU_OK) return st;
    int elems[TGPU_MAX_CHANNELS] = {0};
    for (int c = 0; c < num_channels && c < TGPU_MAX_CHANNELS; c++) {
        DevColumn col;
        col.type = channel_types[c];
        elems[c] = col.elem_size();
    }
    std::vector<int> pass;
    for (int32_t i = 0; i < program->num_projections; i++)
        if (program->projections[i].kind == 0) pass.push_back(program->projections[i].index);
    std::string src = gen_fp_source(prog, elems, num_channels, nullable_mask, pass);
    if (source_out && source_cap > 0) { strncpy(source_out, src.c_str(), (size_t)source_cap - 1); source_out[source_cap - 1] = 0; }
    std::string cubin;
    st = tg::jit_compile_cubin(&fake, src, &cubin);
    if (st != TGPU_OK) { if (source_out && source_cap > 0) { strncpy(source_out, fake.err.c_str(), (size_t)source_cap - 1); source_out[source_cap - 1] = 0; } return st; }
    *cubin_bytes = (int64_t)cubin.size();
    return TGPU_OK;
}
