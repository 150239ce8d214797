// dynfilter.cu — DynamicPageFilter on the device: the probe-side half of dynamic filtering (SURVEY.md §8 f3).
//
// Reference: M/sql/gen/columnar/DynamicPageFilter.java:47-211.  The build side of a join publishes, per join key, the Domain of the
// values it holds (DynamicFilterSourceOperator / JoinDomainBuilder; here tgpu_lookup_key_domain reads it off the finished table); the
// probe-side scan turns the TupleDomain into one filter per column (:124-137) and drops rows that cannot match before they reach the
// join.  DynamicFilterEvaluator.evaluate (:160-178) applies the column filters one after another to the surviving positions and an
// EffectiveFilterProfiler (:181-210) switches a column's filter off once, after at least 2047 input positions, it lets through more
// than selectivityThreshold of them.
//
// Device form: ONE kernel evaluates every active column filter per row in the reference's order (short-circuit), counts per filter the
// rows that reached it and the rows that passed it (the profiler's two counters) and writes a selection flag; the selected rows are
// compacted with a stable select + per-column gather (output order = input order).  A Domain is `null allowed` + a value set: ALL,
// NONE, one inclusive range, or a sorted list of discrete values (binary search).
#include <algorithm>

#include "common.cuh"

namespace {

constexpr int DF_MAX = 16;

struct DDomain {
    ColRef col;
    int32_t null_allowed, kind, is_double, num_values;
    long long lo, hi;
    const long long* values;
};
struct DDomains {
    int32_t count;
    uint32_t active;        // bit i: filter i still evaluated (EffectiveFilterProfiler)
    DDomain d[DF_MAX];
};

__device__ __forceinline__ bool df_contains(const DDomain& d, int64_t row)
{
    if (!tg_valid(d.col.validity, row)) return d.null_allowed != 0;
    if (d.kind == TGPU_DOMAIN_ALL) return true;
    if (d.kind == TGPU_DOMAIN_NONE) return false;
    long long v = tg_load_i64(d.col, row);
    if (d.is_double) {
        double x = __longlong_as_double(v);
        return x >= __longlong_as_double(d.lo) && x <= __longlong_as_double(d.hi);     // RANGE only; NaN is in no range
    }
    if (v < d.lo || v > d.hi) return false;
    if (d.kind == TGPU_DOMAIN_RANGE) return true;
    int lo = 0, hi = d.num_values - 1;
    while (lo <= hi) {
        int mid = (lo + hi) >> 1;
        long long m = d.values[mid];
        if (m == v) return true;
        if (m < v) lo = mid + 1;
        else hi = mid - 1;
    }
    return false;
}

// counters: [2 * i] rows that reached filter i, [2 * i + 1] rows that passed it
__global__ void __launch_bounds__(256) df_flags_kernel(DDomains doms, int64_t n, uint8_t* __restrict__ flags, unsigned long long* __restrict__ counters)
{
    unsigned int in[DF_MAX], out[DF_MAX];
#pragma unroll
    for (int i = 0; i < DF_MAX; i++) { in[i] = 0; out[i] = 0; }
    int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; row < n; row += stride) {
        bool pass = true;
#pragma unroll
        for (int i = 0; i < DF_MAX; i++) {
            if (i >= doms.count || !pass) break;
            if (!((doms.active >> i) & 1)) continue;
            in[i]++;
            pass = df_contains(doms.d[i], row);
            out[i] += pass ? 1 : 0;
        }
        flags[row] = pass ? 1 : 0;
    }
#pragma unroll
    for (int i = 0; i < DF_MAX; i++) {
        if (i >= doms.count) break;
        unsigned int a = in[i], b = out[i];
        for (int off = 16; off > 0; off >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, off); b += __shfl_xor_sync(0xffffffffu, b, off); }
        if ((threadIdx.x & 31) == 0 && a) { atomicAdd(counters + 2 * i, (unsigned long long)a); atomicAdd(counters + 2 * i + 1, (unsigned long long)b); }
    }
}

struct HostDomain {
    tgpu_domain d;
    std::vector<int64_t> values;
    DevBuf d_values;
};

struct DynFilterOp : tgpu_op {
    std::vector<HostDomain> domains;
    double threshold = 1.0;
    // EffectiveFilterProfiler state (DynamicPageFilter.java:181-210)
    std::vector<int64_t> input_positions, output_positions;
    std::vector<bool> ineffective;
    OwnedPage* pending = nullptr;
    bool finishing = false;

    explicit DynFilterOp(tgpu_ctx* c) : tgpu_op(c) {}
    ~DynFilterOp() override { delete pending; }

    int set_domains(const tgpu_domain* in, int32_t n)
    {
        if (n < 0 || n > DF_MAX) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "dynamic filter over more than %d columns", DF_MAX);
        std::vector<HostDomain> nd((size_t)n);
        for (int i = 0; i < n; i++) {
            nd[i].d = in[i];
            if (in[i].kind < TGPU_DOMAIN_ALL || in[i].kind > TGPU_DOMAIN_DISCRETE) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "bad domain kind %d", in[i].kind);
            if (in[i].kind == TGPU_DOMAIN_DISCRETE) {
                if (in[i].num_values <= 0 || !in[i].values) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "discrete domain without values");
                nd[i].values.assign(in[i].values, in[i].values + in[i].num_values);
                std::sort(nd[i].values.begin(), nd[i].values.end());
                nd[i].d.min = nd[i].values.front();
                nd[i].d.max = nd[i].values.back();
                TG_TRY(nd[i].d_values.alloc(ctx, nd[i].values.size() * 8));
                TG_CUDA(ctx, cudaMemcpyAsync(nd[i].d_values.p, nd[i].values.data(), nd[i].values.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
            }
        }
        TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        domains = std::move(nd);
        // a new predicate gets a new DynamicFilterEvaluator, i.e. a fresh profiler (DynamicPageFilter.java:100-108,141-146)
        input_positions.assign((size_t)n, 0);
        output_positions.assign((size_t)n, 0);
        ineffective.assign((size_t)n, false);
        return TGPU_OK;
    }

    bool needs_input() override { return !finishing && !pending; }

    int add_input(const tgpu_page* page) override
    {
        if (pending) return tg_fail(ctx, TGPU_ERR_ILLEGAL_STATE, "addInput while the previous page's output has not been taken");
        const int64_t n = page->num_rows;
        if (n == 0) return TGPU_OK;
        if (n > (int64_t)INT32_MAX) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "page has more than 2^31-1 positions");
        DevPage in;
        TG_TRY(tg_ingest_page(ctx, page, &in));
        DDomains dd;
        memset(&dd, 0, sizeof(dd));
        dd.count = (int32_t)domains.size();
        for (int i = 0; i < dd.count; i++) {
            const tgpu_domain& d = domains[i].d;
            if (d.channel < 0 || d.channel >= (int32_t)in.cols.size()) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "dynamic filter channel %d out of range", d.channel);
            const DevColumn& col = in.cols[d.channel];
            const bool dbl = col.type == TGPU_FLOAT64;
            if (col.type == TGPU_FLOAT32 && d.kind != TGPU_DOMAIN_ALL && d.kind != TGPU_DOMAIN_NONE)
                return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "dynamic filter domains over REAL columns stay on the Java filter");
            // bounds and values are 64-bit: a long DECIMAL value cannot be compared with them
            if (col.type == TGPU_INT128 && d.kind != TGPU_DOMAIN_ALL && d.kind != TGPU_DOMAIN_NONE)
                return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "dynamic filter value sets over long DECIMAL columns stay on the Java filter");
            if (col.elem_size() == 0 && d.kind != TGPU_DOMAIN_ALL && d.kind != TGPU_DOMAIN_NONE)
                return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "dynamic filter value sets over variable-width columns stay on the Java filter");
            if (dbl && d.kind == TGPU_DOMAIN_DISCRETE) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "discrete DOUBLE domains stay on the Java filter");
            dd.d[i].col = tg_colref(col);
            dd.d[i].null_allowed = d.null_allowed;
            dd.d[i].kind = d.kind;
            dd.d[i].is_double = dbl ? 1 : 0;
            dd.d[i].num_values = (int32_t)domains[i].values.size();
            dd.d[i].lo = d.min;
            dd.d[i].hi = d.max;
            dd.d[i].values = domains[i].d_values.as<long long>();
            if (!ineffective[i]) dd.active |= 1u << i;
        }
        DevBuf flags, counters, sel;
        TG_TRY(flags.alloc(ctx, (size_t)n));
        TG_TRY(counters.alloc(ctx, 2 * DF_MAX * 8 + 8));
        TG_CUDA(ctx, cudaMemsetAsync(counters.p, 0, 2 * DF_MAX * 8 + 8, ctx->stream));
        TG_LAUNCH(ctx, df_flags_kernel, tg_grid(ctx, n, 1024, 8), 256, 0, dd, n, flags.as<uint8_t>(), counters.as<unsigned long long>());
        long long* d_count = (long long*)(counters.as<unsigned long long>() + 2 * DF_MAX);
        TG_TRY(tg_flagged_positions(ctx, flags.as<uint8_t>(), n, &sel, d_count));
        std::vector<unsigned long long> h((size_t)2 * DF_MAX + 1);
        TG_CUDA(ctx, cudaMemcpyAsync(h.data(), counters.p, h.size() * 8, cudaMemcpyDeviceToHost, ctx->stream));
        TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        for (int i = 0; i < dd.count; i++) {
            if (ineffective[i]) continue;
            // EffectiveFilterProfiler.recordSelectivity :197-204
            input_positions[i] += (int64_t)h[2 * i];
            output_positions[i] += (int64_t)h[2 * i + 1];
            ineffective[i] = input_positions[i] >= 2047 && (double)output_positions[i] > threshold * (double)input_positions[i];
        }
        const int64_t m = (int64_t)h[2 * DF_MAX];
        if (m == 0) return TGPU_OK;
        DevPage outp;
        outp.rows = m;
        if (m == n) outp.cols = in.cols;          // every position selected: the blocks pass through
        else {
            outp.cols.resize(in.cols.size());
            for (size_t c = 0; c < in.cols.size(); c++) TG_TRY(tg_gather_column(ctx, in.cols[c], sel.as<int32_t>(), m, false, &outp.cols[c]));
            TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));     // `sel` is released on return
        }
        pending = tg_make_owned_page(std::move(outp));
        if (m == n)
            for (int32_t c = 0; c < (int32_t)in.cols.size(); c++) pending->passthrough.push_back(c);
        return TGPU_OK;
    }

    int get_output(OwnedPage** out) override
    {
        *out = pending;
        pending = nullptr;
        return TGPU_OK;
    }
    int finish() override { finishing = true; return TGPU_OK; }
    bool is_finished() override { return finishing && !pending; }
};

}  // namespace

extern "C" int tgpu_dynamic_filter_create(tgpu_ctx* ctx, const tgpu_domain* domains, int32_t num_domains, double selectivity_threshold, tgpu_op** out)
{
    if (!ctx || !out || (num_domains > 0 && !domains)) return TGPU_ERR_INVALID_ARGUMENT;
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    std::unique_ptr<DynFilterOp> op(new DynFilterOp(ctx));
    op->threshold = selectivity_threshold;
    TG_TRY(op->set_domains(domains, num_domains));
    *out = op.release();
    return TGPU_OK;
}

extern "C" int tgpu_dynamic_filter_update(tgpu_op* op, const tgpu_domain* domains, int32_t num_domains)
{
    DynFilterOp* f = dynamic_cast<DynFilterOp*>(op);
    if (!f || (num_domains > 0 && !domains)) return TGPU_ERR_INVALID_ARGUMENT;
    cudaSetDevice(f->ctx->device);
    return f->set_domains(domains, num_domains);
}

extern "C" int tgpu_dynamic_filter_is_effective(tgpu_op* op, int32_t filter, int32_t* out)
{
    DynFilterOp* f = dynamic_cast<DynFilterOp*>(op);
    if (!f || !out || filter < 0 || filter >= (int32_t)f->domains.size()) return TGPU_ERR_INVALID_ARGUMENT;
    *out = f->ineffective[filter] ? 0 : 1;
    return TGPU_OK;
}
