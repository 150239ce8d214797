// common.cuh — context, device buffers, device-side page model and launch helpers shared by all
// translation units of libtrino_gpu.so.
#pragma once
#include <cuda_runtime.h>
#include <cub/cub.cuh>
#include <stdint.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <memory>
#include <string>
#include <utility>
#include <vector>

#include "../../include/trino_gpu.h"
#include "hash.cuh"
#include "device_lib.cuh"

struct ncclComm;

// ------------------------------------------------------------------------------------------------
// device scratch: the small counters and flags operators read back after a kernel.  Every user owns its own words, so
// no operator can overwrite a value another one has yet to read.
// ------------------------------------------------------------------------------------------------
constexpr size_t TG_SCRATCH_BYTES = 1024;     // ctx->d_scratch and ctx->h_scratch

struct TgScratch {
    // join build
    int32_t join_build_flags[4];      // [0] special_head, [1] dup flag, [2] rows off their home line, [3] rows more than 8 lines off
    uint32_t join_gave_up[2];         // rows a trial geometry could not place within its bound
    long long join_key_range[2];      // min / max insertable key
    int32_t join_moved[2];            // fingerprint rows that move on to their next hash function
    // join probe / lookup outer
    long long join_probe_count;       // matched probe rows
    long long join_outer_count;       // unvisited build rows
    uint32_t join_filter_flags[2];    // join filter function: [0] error bits of the evaluated candidates
    // FilterAndProject
    uint32_t fp_flags[2];             // [0] error bits, [1] any-NULL bit per computed column
    long long fp_count;               // selected rows
    // aggregation
    int32_t agg_small_flags[2];       // path S: [0] table overflow, [1] error bits
    int32_t agg_tickets[2];           // path G insert: [0] claimed slots, [1] overflow
    int32_t agg_retry_count[2];       // path G verify: rows that move on to their next hash function
    uint32_t agg_output_flags[4];     // output: [0] error bits, [2..3] any-NULL bit per column
    long long agg_finalize_count;     // fused path: used slots
    uint32_t agg_slice_counts[64];    // fused path: rows per table slice
    // string dictionary insert: [0] claims / retry count / new strings, [1] overflow, [2..3] new bytes
    int32_t strdict_counts[4];
    // page serializer
    long long serde_count;            // non-NULL positions
};
static_assert(sizeof(TgScratch) <= TG_SCRATCH_BYTES, "the scratch words must fit the scratch allocation");

// ------------------------------------------------------------------------------------------------
// context
// ------------------------------------------------------------------------------------------------
struct tgpu_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    std::string err;
    int64_t launches = 0;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    cudaEvent_t kev0 = nullptr, kev1 = nullptr;   // bracket the dominant kernel of the last operator call (tgpu_ctx_last_kernel_ms)
    bool kev_valid = false;
    void* flush_buf = nullptr;
    size_t flush_bytes = 0;
    int sm_count = 132;
    size_t smem_optin = 0;
    // pinned staging ring for host pages
    void* staging = nullptr;
    size_t staging_bytes = 0;
    // pinned staging of small readbacks (tg_read) and the device words they come from
    int64_t* h_scratch = nullptr;
    TgScratch* d_scratch = nullptr;
    cudaEvent_t fence_ev = nullptr;     // recorded on this context's stream by an exchange that must not outrun this consumer
    // cache of large device buffers released by operators (all work of a ctx is ordered on its one stream, so a block
    // can be handed to the next request without waiting): multi-GB cudaMallocAsync calls cost milliseconds even from a
    // warm pool, and operators allocate the same sizes page after page
    struct BigBlock { void* p; size_t bytes; };
    std::vector<BigBlock> big_cache;
    size_t big_cache_bytes = 0;
    // NCCL
    ncclComm* comm = nullptr;
    int rank = 0, world = 1;
    // peer-memory exchange arenas (two per rank, alternating): arena[k][r] = rank r's k-th arena mapped into this process
    void* arena_local[TGPU_NUM_ARENAS] = {nullptr, nullptr, nullptr};
    std::vector<void*> arena_peer[TGPU_NUM_ARENAS];
    ncclComm* comm2 = nullptr;               // second communicator: barriers of the split-phase exchange (copy stream)
    cudaStream_t copy_stream = nullptr;      // peer copies of the split-phase exchange (copy engines)
    int exchanges_in_flight = 0;
    size_t arena_bytes = 0;
    int64_t arena_epoch = 0;
};

int tg_fail(tgpu_ctx* ctx, int status, const char* fmt, ...);

constexpr size_t TG_BIG_BLOCK = (size_t)32 << 20;            // blocks at least this large go through the ctx cache
// bytes the cache may hold before blocks go back to the pool: a fifth of an H100's 80 GB, so that cached blocks do not starve
// allocations of other sizes
constexpr size_t TG_BIG_CACHE_LIMIT = (size_t)16 << 30;

#define TG_CUDA(ctx, call)                                                                           \
    do {                                                                                             \
        cudaError_t _e = (call);                                                                     \
        if (_e != cudaSuccess)                                                                       \
            return tg_fail((ctx), TGPU_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__, __LINE__); \
    } while (0)

#define TG_TRY(expr)                 \
    do {                             \
        int _s = (expr);             \
        if (_s != TGPU_OK) return _s; \
    } while (0)

#define TG_CHECK_ARG(ctx, cond, msg)                                               \
    do {                                                                           \
        if (!(cond)) return tg_fail((ctx), TGPU_ERR_INVALID_ARGUMENT, "%s", (msg)); \
    } while (0)

// kernel launch on the ctx stream with launch accounting (tgpu_ctx_kernel_launches)
#define TG_LAUNCH(ctx, kernel, grid, block, smem, ...)                                               \
    do {                                                                                             \
        kernel<<<(grid), (block), (smem), (ctx)->stream>>>(__VA_ARGS__);                             \
        (ctx)->launches++;                                                                           \
        cudaError_t _e = cudaGetLastError();                                                         \
        if (_e != cudaSuccess)                                                                       \
            return tg_fail((ctx), TGPU_ERR_CUDA, "launch of %s failed: %s (%s:%d)", #kernel, cudaGetErrorString(_e), __FILE__, __LINE__); \
    } while (0)

// bracket one kernel launch with events on the ctx stream so benchmarks can read its device time
#define TG_TIMED_BEGIN(ctx) do { cudaEventRecord((ctx)->kev0, (ctx)->stream); } while (0)
#define TG_TIMED_END(ctx) do { cudaEventRecord((ctx)->kev1, (ctx)->stream); (ctx)->kev_valid = true; } while (0)

static inline int64_t tg_div_up(int64_t a, int64_t b) { return (a + b - 1) / b; }

// grid size for a grid-stride kernel: whole waves of the SMs x resident CTAs, capped by the work
static inline int tg_grid(const tgpu_ctx* ctx, int64_t work_items, int items_per_block, int ctas_per_sm)
{
    int64_t need = tg_div_up(work_items, items_per_block);
    int64_t wave = (int64_t)ctx->sm_count * ctas_per_sm;
    if (need < 1) need = 1;
    if (need <= wave) return (int)need;
    return (int)wave;
}

// ------------------------------------------------------------------------------------------------
// device buffers (stream-ordered pool allocations on the ctx stream)
// ------------------------------------------------------------------------------------------------
struct DevBuf {
    tgpu_ctx* ctx = nullptr;
    void* p = nullptr;
    size_t bytes = 0;

    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    DevBuf(DevBuf&& o) noexcept { *this = std::move(o); }
    DevBuf& operator=(DevBuf&& o) noexcept
    {
        if (this != &o) {
            release();
            ctx = o.ctx; p = o.p; bytes = o.bytes;
            o.p = nullptr; o.bytes = 0;
        }
        return *this;
    }
    ~DevBuf() { release(); }
    int alloc(tgpu_ctx* c, size_t n)
    {
        release();
        ctx = c;
        if (n == 0) n = 16;
        n = (n + 255) & ~(size_t)255;
        if (n >= TG_BIG_BLOCK) {
            size_t best = (size_t)-1;
            for (size_t i = 0; i < c->big_cache.size(); i++) {
                size_t b = c->big_cache[i].bytes;
                if (b >= n && b <= n + n / 4 && (best == (size_t)-1 || b < c->big_cache[best].bytes)) best = i;
            }
            if (best != (size_t)-1) {
                p = c->big_cache[best].p;
                bytes = c->big_cache[best].bytes;
                c->big_cache_bytes -= bytes;
                c->big_cache.erase(c->big_cache.begin() + best);
                return TGPU_OK;
            }
        }
        cudaError_t e = cudaMallocAsync(&p, n, c->stream);
        if (e != cudaSuccess) {
            p = nullptr;
            return tg_fail(c, TGPU_ERR_CUDA, "cudaMallocAsync(%zu) failed: %s", n, cudaGetErrorString(e));
        }
        bytes = n;
        return TGPU_OK;
    }
    void release()
    {
        if (p && ctx) {
            if (bytes >= TG_BIG_BLOCK && ctx->big_cache.size() < 32 && ctx->big_cache_bytes + bytes <= TG_BIG_CACHE_LIMIT) {
                ctx->big_cache.push_back(tgpu_ctx::BigBlock{p, bytes});
                ctx->big_cache_bytes += bytes;
            }
            else cudaFreeAsync(p, ctx->stream);
        }
        p = nullptr;
        bytes = 0;
    }
    template <typename T> T* as() const { return (T*)p; }
};

// ------------------------------------------------------------------------------------------------
// device page model: flat Arrow-layout columns in HBM.  DICT32 / RLE inputs are decoded on ingest
// (values, not encodings, are the operator contract: SURVEY.md Appendix B.5).
// ------------------------------------------------------------------------------------------------
struct DevColumn {
    int32_t type = 0;            // TGPU_INT64/INT32/INT16/INT8/FLOAT64/UTF8
    int64_t length = 0;
    const void* data = nullptr;
    const int32_t* offsets = nullptr;
    const uint8_t* validity = nullptr;   // Arrow bitmap or null
    // ownership (empty when the column borrows a TGPU_PAGE_DEVICE input)
    std::shared_ptr<DevBuf> own_data, own_offsets, own_validity;
    int64_t data_bytes = 0;      // UTF8: number of value bytes

    int elem_size() const
    {
        switch (type) {
            case TGPU_INT128: return 16;
            case TGPU_INT64: case TGPU_FLOAT64: return 8;
            case TGPU_INT32: case TGPU_FLOAT32: return 4;
            case TGPU_INT16: return 2;
            case TGPU_INT8: return 1;
            default: return 0;
        }
    }
    int64_t memory_bytes() const
    {
        int64_t b = 0;
        if (own_data) b += (int64_t)own_data->bytes;
        if (own_offsets) b += (int64_t)own_offsets->bytes;
        if (own_validity) b += (int64_t)own_validity->bytes;
        return b;
    }
};

struct DevPage {
    int64_t rows = 0;
    std::vector<DevColumn> cols;
    int64_t memory_bytes() const { int64_t b = 0; for (auto& c : cols) b += c.memory_bytes(); return b; }
};

// a page handed to the caller by get_output: the tgpu_page header is the first member so the
// pointer can be cast back in tgpu_page_release
struct OwnedPage;
void tg_owned_page_unregister(OwnedPage* page);
struct OwnedPage {
    tgpu_page hdr;
    std::vector<tgpu_column> cols;
    DevPage page;
    int32_t partition = -1;
    std::vector<int32_t> passthrough;   // per column: input channel whose block this column IS (unchanged, same rows), else -1
    // Output pages are registered by the address of their column descriptors: when one is handed to another operator as a
    // TGPU_PAGE_DEVICE input (GPU -> GPU chaining), ingestion finds it and SHARES the buffers' ownership, so the caller may
    // release the upstream page right after addInput, as the Operator contract allows (ingest_value_column in core.cu).
    ~OwnedPage() { tg_owned_page_unregister(this); }
};

static inline ColRef tg_colref(const DevColumn& c) { return ColRef{c.data, c.validity, c.type, c.elem_size()}; }

// page ingestion: host pages are staged through pinned memory and copied H2D on the ctx stream;
// device pages are borrowed.  Both get DICT/RLE decoded and byte-map nulls packed to bitmaps.
int tg_ingest_page(tgpu_ctx* ctx, const tgpu_page* page, DevPage* out);
int tg_ingest_column(tgpu_ctx* ctx, const tgpu_column* col, bool device, DevColumn* out);
OwnedPage* tg_make_owned_page(DevPage&& page);
// gather rows of a column by int32 indices (idx < 0 -> NULL output row)
int tg_gather_column(tgpu_ctx* ctx, const DevColumn& src, const int32_t* d_idx, int64_t n, bool idx_may_be_negative, DevColumn* out);
// concatenation of column chunks of one type (PagesIndex keeps block references; the device keeps one flat column)
int tg_concat_columns(tgpu_ctx* ctx, const std::vector<const DevColumn*>& parts, DevColumn* out);
// contiguous slice copy of a column
int tg_slice_column(tgpu_ctx* ctx, const DevColumn& src, int64_t first, int64_t count, DevColumn* out);
// append `src` to a growing owned column (used by the build-side store)
int tg_read_i64(tgpu_ctx* ctx, const void* d_ptr, int64_t* out);   // synchronous small readback
int tg_read(tgpu_ctx* ctx, const void* d_ptr, size_t bytes, void* host_out);   // the same for up to TG_SCRATCH_BYTES

// small utility kernels, enqueued on the ctx stream
// byte null map (1 = NULL) -> Arrow validity bitmap (1 = valid); *d_any (if given) is or-ed with 1 when a NULL was seen
int tg_pack_nullmap(tgpu_ctx* ctx, const uint8_t* is_null, int64_t n, uint8_t* bitmap, unsigned int* d_any = nullptr);
int tg_iota(tgpu_ctx* ctx, int32_t* out, int64_t n, int32_t first = 0);                         // out[i] = first + i
int tg_add_i32(tgpu_ctx* ctx, const int32_t* in, int64_t n, int32_t delta, int32_t* out);      // out[i] = in[i] + delta
int tg_fill16(tgpu_ctx* ctx, int4* out, int64_t n, int4 value);                                // out[i] = value

// CUB device-wide algorithms: size query, temporary storage from the pool, run.  Either call failing is TGPU_ERR_CUDA.
// Iterator and item-count types pass through unchanged: they select the CUB kernels that get instantiated.
template <typename Call>
int tg_cub(tgpu_ctx* ctx, Call call)
{
    size_t bytes = 0;
    TG_CUDA(ctx, call(nullptr, bytes));
    DevBuf tmp;
    TG_TRY(tmp.alloc(ctx, bytes));
    TG_CUDA(ctx, call(tmp.p, bytes));
    return TGPU_OK;
}

template <typename InIt, typename OutIt, typename NumT>
int tg_exclusive_sum(tgpu_ctx* ctx, InIt in, OutIt out, NumT n)
{
    return tg_cub(ctx, [&](void* tmp, size_t& bytes) { return cub::DeviceScan::ExclusiveSum(tmp, bytes, in, out, n, ctx->stream); });
}

template <typename InIt, typename FlagIt, typename OutIt, typename CountIt, typename NumT>
int tg_select_flagged(tgpu_ctx* ctx, InIt in, FlagIt flags, OutIt out, CountIt d_count, NumT n)
{
    return tg_cub(ctx, [&](void* tmp, size_t& bytes) { return cub::DeviceSelect::Flagged(tmp, bytes, in, flags, out, d_count, n, ctx->stream); });
}

template <typename K, typename V, typename NumT>
int tg_sort_pairs(tgpu_ctx* ctx, const K* keys_in, K* keys_out, const V* values_in, V* values_out, NumT n, int begin_bit, int end_bit)
{
    return tg_cub(ctx, [&](void* tmp, size_t& bytes) {
        return cub::DeviceRadixSort::SortPairs(tmp, bytes, keys_in, keys_out, values_in, values_out, n, begin_bit, end_bit, ctx->stream);
    });
}

template <typename K, typename NumT>
int tg_sort_keys(tgpu_ctx* ctx, const K* keys_in, K* keys_out, NumT n, int begin_bit, int end_bit)
{
    return tg_cub(ctx, [&](void* tmp, size_t& bytes) { return cub::DeviceRadixSort::SortKeys(tmp, bytes, keys_in, keys_out, n, begin_bit, end_bit, ctx->stream); });
}

// int32 positions of the rows whose flag is set, in row order, into `positions` (allocated here); their count into *d_count
int tg_flagged_positions(tgpu_ctx* ctx, uint8_t* flags, int64_t n, DevBuf* positions, long long* d_count);

// ------------------------------------------------------------------------------------------------
// operator base (M/operator/Operator.java:21-102)
// ------------------------------------------------------------------------------------------------
struct tgpu_op {
    tgpu_ctx* ctx;
    explicit tgpu_op(tgpu_ctx* c) : ctx(c) {}
    virtual ~tgpu_op() {}
    virtual bool needs_input() = 0;
    virtual int add_input(const tgpu_page* page) = 0;
    virtual int get_output(OwnedPage** out) = 0;
    virtual int finish() = 0;
    virtual bool is_finished() = 0;
    virtual int64_t memory_bytes() { return 0; }
};

// device-side helpers -------------------------------------------------------------------------
#if defined(__CUDACC__)
// streaming (read-once) 128-bit load that does not allocate in L1
__device__ __forceinline__ int4 tg_ldg_stream(const int4* p)
{
    int4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ void tg_stg_stream(int4* p, const int4& v)
{
    asm volatile("st.global.L1::no_allocate.v4.s32 [%0], {%1, %2, %3, %4};"
                 :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w));
}
#endif
