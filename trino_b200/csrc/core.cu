// core.cu — context lifecycle, device memory helpers, page ingestion / gather / readback, and the
// generic Operator-protocol entry points of the C ABI (include/trino_gpu.h).
#include <thrust/iterator/counting_iterator.h>

#include <map>
#include <mutex>

#include "common.cuh"

// ------------------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------------------
static thread_local std::string g_last_error_no_ctx;

int tg_fail(tgpu_ctx* ctx, int status, const char* fmt, ...)
{
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    if (ctx) ctx->err = buf;
    else g_last_error_no_ctx = buf;
    return status;
}

extern "C" const char* tgpu_last_error(const tgpu_ctx* ctx)
{
    return ctx ? ctx->err.c_str() : g_last_error_no_ctx.c_str();
}

extern "C" const char* tgpu_status_name(int status)
{
    switch (status) {
        case TGPU_OK: return "OK";
        case TGPU_ERR_INVALID_ARGUMENT: return "INVALID_ARGUMENT";
        case TGPU_ERR_CUDA: return "GENERIC_INTERNAL_ERROR";
        case TGPU_ERR_INSUFFICIENT_RESOURCES: return "GENERIC_INSUFFICIENT_RESOURCES";
        case TGPU_ERR_NUMERIC_VALUE_OUT_OF_RANGE: return "NUMERIC_VALUE_OUT_OF_RANGE";
        case TGPU_ERR_DIVISION_BY_ZERO: return "DIVISION_BY_ZERO";
        case TGPU_ERR_NOT_SUPPORTED: return "NOT_SUPPORTED";
        case TGPU_ERR_ILLEGAL_STATE: return "ILLEGAL_STATE";
        case TGPU_ERR_INVALID_CAST_ARGUMENT: return "INVALID_CAST_ARGUMENT";
        case TGPU_ERR_INVALID_FUNCTION_ARGUMENT: return "INVALID_FUNCTION_ARGUMENT";
        default: return "UNKNOWN";
    }
}

// ------------------------------------------------------------------------------------------------
// context
// ------------------------------------------------------------------------------------------------
extern "C" int tgpu_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

extern "C" int tgpu_ctx_create(int device, tgpu_ctx** out)
{
    if (!out) return TGPU_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        cudaGetLastError();
        // no CPU fallback by design: the product path fails loudly without a device
        return tg_fail(nullptr, TGPU_ERR_CUDA, "no CUDA device available (%s); libtrino_gpu has no CPU fallback",
                       e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
    }
    if (device < 0 || device >= n) return tg_fail(nullptr, TGPU_ERR_INVALID_ARGUMENT, "device %d out of range [0,%d)", device, n);
    tgpu_ctx* ctx = new tgpu_ctx();
    ctx->device = device;
    TG_CUDA(ctx, cudaSetDevice(device));
    TG_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
    TG_CUDA(ctx, cudaEventCreate(&ctx->ev0));
    TG_CUDA(ctx, cudaEventCreate(&ctx->ev1));
    TG_CUDA(ctx, cudaEventCreate(&ctx->kev0));
    TG_CUDA(ctx, cudaEventCreate(&ctx->kev1));
    cudaDeviceProp prop;
    TG_CUDA(ctx, cudaGetDeviceProperties(&prop, device));
    ctx->sm_count = prop.multiProcessorCount;
    ctx->smem_optin = prop.sharedMemPerBlockOptin;
    // keep freed blocks in the pool: operators allocate and free per page
    cudaMemPool_t pool;
    TG_CUDA(ctx, cudaDeviceGetDefaultMemPool(&pool, device));
    uint64_t threshold = UINT64_MAX;
    TG_CUDA(ctx, cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &threshold));
    TG_CUDA(ctx, cudaMallocHost((void**)&ctx->h_scratch, TG_SCRATCH_BYTES));
    TG_CUDA(ctx, cudaMalloc((void**)&ctx->d_scratch, TG_SCRATCH_BYTES));
    TG_CUDA(ctx, cudaMemsetAsync(ctx->d_scratch, 0, TG_SCRATCH_BYTES, ctx->stream));
    *out = ctx;
    return TGPU_OK;
}

int tg_comm_destroy_internal(tgpu_ctx* ctx);

extern "C" void tgpu_ctx_destroy(tgpu_ctx* ctx)
{
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    tg_comm_destroy_internal(ctx);
    for (auto& b : ctx->big_cache) cudaFreeAsync(b.p, ctx->stream);
    ctx->big_cache.clear();
    cudaStreamSynchronize(ctx->stream);
    if (ctx->flush_buf) cudaFree(ctx->flush_buf);
    if (ctx->staging) cudaFreeHost(ctx->staging);
    if (ctx->h_scratch) cudaFreeHost(ctx->h_scratch);
    if (ctx->d_scratch) cudaFree(ctx->d_scratch);
    if (ctx->fence_ev) cudaEventDestroy(ctx->fence_ev);
    cudaEventDestroy(ctx->ev0);
    cudaEventDestroy(ctx->ev1);
    cudaEventDestroy(ctx->kev0);
    cudaEventDestroy(ctx->kev1);
    cudaStreamDestroy(ctx->stream);
    delete ctx;
}

extern "C" int tgpu_ctx_synchronize(tgpu_ctx* ctx)
{
    if (ctx) cudaSetDevice(ctx->device);     // callable from any thread: the calling thread's current device may differ
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return TGPU_OK;
}

extern "C" void* tgpu_ctx_stream(tgpu_ctx* ctx) { return (void*)ctx->stream; }
extern "C" int64_t tgpu_ctx_kernel_launches(const tgpu_ctx* ctx) { return ctx->launches; }

extern "C" int tgpu_ctx_set_l2_fetch_granularity(tgpu_ctx* ctx, int bytes)
{
    // cudaLimitMaxL2FetchGranularity: how much the L2 pulls from HBM per missing sector (32/64/128 B).  Hash probes
    // touch one 32-byte sector per lookup; anything wider is wasted DRAM traffic for them.
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    TG_CUDA(ctx, cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, (size_t)bytes));
    return TGPU_OK;
}

extern "C" int tgpu_ctx_get_l2_fetch_granularity(tgpu_ctx* ctx, int* bytes)
{
    size_t v = 0;
    TG_CUDA(ctx, cudaDeviceGetLimit(&v, cudaLimitMaxL2FetchGranularity));
    *bytes = (int)v;
    return TGPU_OK;
}

extern "C" int tgpu_malloc(tgpu_ctx* ctx, size_t bytes, void** out)
{
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    TG_CUDA(ctx, cudaMallocAsync(out, bytes ? bytes : 16, ctx->stream));
    return TGPU_OK;
}

extern "C" int tgpu_free(tgpu_ctx* ctx, void* ptr)
{
    if (ctx) cudaSetDevice(ctx->device);     // callable from any thread: the calling thread's current device may differ
    if (ptr) TG_CUDA(ctx, cudaFreeAsync(ptr, ctx->stream));
    return TGPU_OK;
}

extern "C" int tgpu_memcpy_h2d(tgpu_ctx* ctx, void* dst, const void* src, size_t bytes)
{
    if (ctx) cudaSetDevice(ctx->device);     // callable from any thread: the calling thread's current device may differ
    TG_CUDA(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, ctx->stream));
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return TGPU_OK;
}

extern "C" int tgpu_memcpy_d2h(tgpu_ctx* ctx, void* dst, const void* src, size_t bytes)
{
    if (ctx) cudaSetDevice(ctx->device);     // callable from any thread: the calling thread's current device may differ
    TG_CUDA(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return TGPU_OK;
}

extern "C" int tgpu_host_alloc_pinned(size_t bytes, void** out)
{
    cudaError_t e = cudaMallocHost(out, bytes ? bytes : 16);
    if (e != cudaSuccess) return tg_fail(nullptr, TGPU_ERR_CUDA, "cudaMallocHost(%zu) failed: %s", bytes, cudaGetErrorString(e));
    return TGPU_OK;
}

extern "C" int tgpu_host_free_pinned(void* ptr)
{
    if (ptr) cudaFreeHost(ptr);
    return TGPU_OK;
}

__global__ void tg_flush_l2_kernel(int4* buf, int64_t n, int v)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) buf[i] = make_int4(v, v, v, v);
}

extern "C" int tgpu_flush_l2(tgpu_ctx* ctx)
{
    if (ctx) cudaSetDevice(ctx->device);     // callable from any thread: the calling thread's current device may differ
    // 256 MiB > the 50 MB L2 of an H100
    if (!ctx->flush_buf) {
        ctx->flush_bytes = (size_t)256 << 20;
        TG_CUDA(ctx, cudaMalloc(&ctx->flush_buf, ctx->flush_bytes));
    }
    static int counter = 0;
    int64_t n = (int64_t)(ctx->flush_bytes / sizeof(int4));
    tg_flush_l2_kernel<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>((int4*)ctx->flush_buf, n, ++counter);
    TG_CUDA(ctx, cudaGetLastError());
    return TGPU_OK;
}

extern "C" int tgpu_timer_start(tgpu_ctx* ctx)
{
    if (ctx) cudaSetDevice(ctx->device);     // callable from any thread: the calling thread's current device may differ
    TG_CUDA(ctx, cudaEventRecord(ctx->ev0, ctx->stream));
    return TGPU_OK;
}

extern "C" int tgpu_timer_stop_ms(tgpu_ctx* ctx, float* ms)
{
    if (ctx) cudaSetDevice(ctx->device);     // callable from any thread: the calling thread's current device may differ
    TG_CUDA(ctx, cudaEventRecord(ctx->ev1, ctx->stream));
    TG_CUDA(ctx, cudaEventSynchronize(ctx->ev1));
    TG_CUDA(ctx, cudaEventElapsedTime(ms, ctx->ev0, ctx->ev1));
    return TGPU_OK;
}

extern "C" int tgpu_ctx_last_kernel_ms(tgpu_ctx* ctx, float* ms)
{
    // device time of the dominant kernel of the last operator call that has one (fused probe, index probe,
    // small-group aggregation): CUDA events recorded right around that launch on the ctx stream
    if (!ctx || !ms) return TGPU_ERR_INVALID_ARGUMENT;
    if (!ctx->kev_valid) return tg_fail(ctx, TGPU_ERR_ILLEGAL_STATE, "no timed kernel has run on this context yet");
    TG_CUDA(ctx, cudaEventSynchronize(ctx->kev1));
    TG_CUDA(ctx, cudaEventElapsedTime(ms, ctx->kev0, ctx->kev1));
    return TGPU_OK;
}

int tg_read(tgpu_ctx* ctx, const void* d_ptr, size_t bytes, void* host_out)
{
    if (bytes > TG_SCRATCH_BYTES) return tg_fail(ctx, TGPU_ERR_ILLEGAL_STATE, "readback of %zu bytes exceeds the %zu-byte staging buffer", bytes, TG_SCRATCH_BYTES);
    TG_CUDA(ctx, cudaMemcpyAsync(ctx->h_scratch, d_ptr, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    memcpy(host_out, ctx->h_scratch, bytes);
    return TGPU_OK;
}

int tg_read_i64(tgpu_ctx* ctx, const void* d_ptr, int64_t* out) { return tg_read(ctx, d_ptr, 8, out); }

// ------------------------------------------------------------------------------------------------
// utility kernels
// ------------------------------------------------------------------------------------------------
// Java boolean[] valueIsNull (1 = NULL) -> Arrow validity bitmap (1 = valid); one thread packs 8 rows
__global__ void tg_pack_nullmap_kernel(const uint8_t* __restrict__ is_null, int64_t n, uint8_t* __restrict__ bitmap, unsigned int* __restrict__ any)
{
    int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t nbytes = (n + 7) >> 3;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    unsigned int seen = 0;
    for (; b < nbytes; b += stride) {
        unsigned int v = 0;
        int64_t base = b << 3;
#pragma unroll
        for (int k = 0; k < 8; k++) {
            int64_t i = base + k;
            if (i < n) { if (is_null[i] == 0) v |= 1u << k; else seen = 1; }
        }
        bitmap[b] = (uint8_t)v;
    }
    if (seen && any) atomicOr(any, 1u);
}

int tg_pack_nullmap(tgpu_ctx* ctx, const uint8_t* is_null, int64_t n, uint8_t* bitmap, unsigned int* d_any)
{
    TG_LAUNCH(ctx, tg_pack_nullmap_kernel, tg_grid(ctx, (n + 7) / 8, 256, 8), 256, 0, is_null, n, bitmap, d_any);
    return TGPU_OK;
}

__global__ void tg_iota_kernel(int32_t* out, int64_t n, int32_t first)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) out[i] = first + (int32_t)i;
}

int tg_iota(tgpu_ctx* ctx, int32_t* out, int64_t n, int32_t first)
{
    TG_LAUNCH(ctx, tg_iota_kernel, tg_grid(ctx, n, 1024, 8), 256, 0, out, n, first);
    return TGPU_OK;
}

__global__ void tg_add_i32_kernel(const int32_t* __restrict__ in, int64_t n, int32_t delta, int32_t* __restrict__ out)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) out[i] = in[i] + delta;
}

int tg_add_i32(tgpu_ctx* ctx, const int32_t* in, int64_t n, int32_t delta, int32_t* out)
{
    TG_LAUNCH(ctx, tg_add_i32_kernel, tg_grid(ctx, n, 1024, 8), 256, 0, in, n, delta, out);
    return TGPU_OK;
}

__global__ void tg_fill16_kernel(int4* out, int64_t n, int4 value)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) out[i] = value;
}

int tg_fill16(tgpu_ctx* ctx, int4* out, int64_t n, int4 value)
{
    TG_LAUNCH(ctx, tg_fill16_kernel, tg_grid(ctx, n, 1024, 8), 256, 0, out, n, value);
    return TGPU_OK;
}

int tg_flagged_positions(tgpu_ctx* ctx, uint8_t* flags, int64_t n, DevBuf* positions, long long* d_count)
{
    TG_TRY(positions->alloc(ctx, (size_t)n * 4));
    return tg_select_flagged(ctx, thrust::counting_iterator<int32_t>(0), flags, positions->as<int32_t>(), d_count, (int)n);
}

// ------------------------------------------------------------------------------------------------
// ingestion kernels
// ------------------------------------------------------------------------------------------------
// fixed-width gather: out[i] = src[idx[i]] (idx == nullptr -> broadcast of row 0); idx < 0 -> NULL row
template <typename T>
__global__ void tg_gather_fixed_kernel(const T* __restrict__ src, const int32_t* __restrict__ idx, int64_t n, T* __restrict__ out)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        int32_t j = idx ? idx[i] : 0;
        out[i] = j >= 0 ? src[j] : T{};
    }
}

// validity gather: one thread produces one output byte (8 rows) so no atomics are needed
__global__ void tg_gather_validity_kernel(const uint8_t* __restrict__ src_validity, const int32_t* __restrict__ idx, int64_t n,
                                          uint8_t* __restrict__ out)
{
    int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t nbytes = (n + 7) >> 3;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; b < nbytes; b += stride) {
        uint32_t v = 0;
        int64_t base = b << 3;
#pragma unroll
        for (int k = 0; k < 8; k++) {
            int64_t i = base + k;
            if (i < n) {
                int32_t j = idx ? idx[i] : 0;
                if (j >= 0 && tg_valid(src_validity, j)) v |= 1u << k;
            }
        }
        out[b] = (uint8_t)v;
    }
}

__global__ void tg_utf8_lengths_kernel(const int32_t* __restrict__ offsets, const int32_t* __restrict__ idx, int64_t n, int32_t* __restrict__ len)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        int32_t j = idx ? idx[i] : 0;
        len[i] = j >= 0 ? offsets[j + 1] - offsets[j] : 0;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) len[n] = 0;
}

__global__ void tg_utf8_copy_kernel(const uint8_t* __restrict__ src, const int32_t* __restrict__ src_off, const int32_t* __restrict__ idx,
                                    int64_t n, const int32_t* __restrict__ dst_off, uint8_t* __restrict__ dst)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        int32_t j = idx ? idx[i] : 0;
        if (j < 0) continue;
        int32_t a = src_off[j], len = src_off[j + 1] - a, d = dst_off[i];
        for (int32_t k = 0; k < len; k++) dst[d + k] = src[a + k];
    }
}

static int alloc_shared(tgpu_ctx* ctx, size_t bytes, std::shared_ptr<DevBuf>* out)
{
    auto b = std::make_shared<DevBuf>();
    TG_TRY(b->alloc(ctx, bytes));
    *out = std::move(b);
    return TGPU_OK;
}

int tg_gather_column(tgpu_ctx* ctx, const DevColumn& src, const int32_t* d_idx, int64_t n, bool idx_may_be_negative, DevColumn* out)
{
    DevColumn r;
    r.type = src.type;
    r.length = n;
    int threads = 256;
    int grid = tg_grid(ctx, n, threads * 4, 8);
    if (src.validity || idx_may_be_negative) {
        TG_TRY(alloc_shared(ctx, (size_t)((n + 7) / 8), &r.own_validity));
        int vgrid = tg_grid(ctx, (n + 7) / 8, threads, 8);
        TG_LAUNCH(ctx, tg_gather_validity_kernel, vgrid, threads, 0, src.validity, d_idx, n, r.own_validity->as<uint8_t>());
        r.validity = r.own_validity->as<uint8_t>();
    }
    if (src.type == TGPU_UTF8) {
        // lengths -> exclusive scan -> offsets; then byte copy
        TG_TRY(alloc_shared(ctx, (size_t)(n + 1) * 4, &r.own_offsets));
        DevBuf len;
        TG_TRY(len.alloc(ctx, (size_t)(n + 1) * 4));
        TG_LAUNCH(ctx, tg_utf8_lengths_kernel, grid, threads, 0, src.offsets, d_idx, n, len.as<int32_t>());
        TG_TRY(tg_exclusive_sum(ctx, len.as<int32_t>(), r.own_offsets->as<int32_t>(), n + 1));
        int32_t total = 0;
        TG_TRY(tg_read(ctx, r.own_offsets->as<int32_t>() + n, 4, &total));
        TG_TRY(alloc_shared(ctx, (size_t)total, &r.own_data));
        TG_LAUNCH(ctx, tg_utf8_copy_kernel, grid, threads, 0, (const uint8_t*)src.data, src.offsets, d_idx, n,
                  r.own_offsets->as<int32_t>(), r.own_data->as<uint8_t>());
        r.offsets = r.own_offsets->as<int32_t>();
        r.data = r.own_data->p;
        r.data_bytes = total;
    }
    else {
        int es = src.elem_size();
        if (es == 0) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "gather: unsupported column type %d", src.type);
        TG_TRY(alloc_shared(ctx, (size_t)n * es, &r.own_data));
        switch (es) {
            case 16: TG_LAUNCH(ctx, tg_gather_fixed_kernel<int4>, grid, threads, 0, (const int4*)src.data, d_idx, n, r.own_data->as<int4>()); break;
            case 8: TG_LAUNCH(ctx, tg_gather_fixed_kernel<int64_t>, grid, threads, 0, (const int64_t*)src.data, d_idx, n, r.own_data->as<int64_t>()); break;
            case 4: TG_LAUNCH(ctx, tg_gather_fixed_kernel<int32_t>, grid, threads, 0, (const int32_t*)src.data, d_idx, n, r.own_data->as<int32_t>()); break;
            case 2: TG_LAUNCH(ctx, tg_gather_fixed_kernel<int16_t>, grid, threads, 0, (const int16_t*)src.data, d_idx, n, r.own_data->as<int16_t>()); break;
            default: TG_LAUNCH(ctx, tg_gather_fixed_kernel<int8_t>, grid, threads, 0, (const int8_t*)src.data, d_idx, n, r.own_data->as<int8_t>()); break;
        }
        r.data = r.own_data->p;
    }
    *out = std::move(r);
    return TGPU_OK;
}

int tg_slice_column(tgpu_ctx* ctx, const DevColumn& src, int64_t first, int64_t count, DevColumn* out)
{
    // byte-aligned fixed-width slices without nulls are plain copies; everything else goes through gather
    if (src.type != TGPU_UTF8 && !src.validity) {
        DevColumn r;
        r.type = src.type;
        r.length = count;
        int es = src.elem_size();
        TG_TRY(alloc_shared(ctx, (size_t)count * es, &r.own_data));
        TG_CUDA(ctx, cudaMemcpyAsync(r.own_data->p, (const char*)src.data + first * es, (size_t)count * es, cudaMemcpyDeviceToDevice, ctx->stream));
        r.data = r.own_data->p;
        *out = std::move(r);
        return TGPU_OK;
    }
    DevBuf idx;
    TG_TRY(idx.alloc(ctx, (size_t)count * 4));
    TG_TRY(tg_iota(ctx, idx.as<int32_t>(), count, (int32_t)first));
    return tg_gather_column(ctx, src, idx.as<int32_t>(), count, false, out);
}

struct ConcatParts {
    const uint8_t* validity[64];
    long long start[65];
    int count;
};

// validity of a concatenation: one thread per output byte, chunk found by a linear scan over <= 64 chunk starts
__global__ void tg_concat_validity_kernel(ConcatParts parts, int64_t n, uint8_t* __restrict__ out)
{
    int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t nbytes = (n + 7) >> 3;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; b < nbytes; b += stride) {
        unsigned int v = 0;
        for (int k = 0; k < 8; k++) {
            int64_t i = (b << 3) + k;
            if (i >= n) break;
            int c = 0;
            while (c + 1 < parts.count && i >= parts.start[c + 1]) c++;
            if (tg_valid(parts.validity[c], i - parts.start[c])) v |= 1u << k;
        }
        out[b] = (uint8_t)v;
    }
}

int tg_concat_columns(tgpu_ctx* ctx, const std::vector<const DevColumn*>& parts, DevColumn* out)
{
    DevColumn r;
    if (parts.empty()) { *out = std::move(r); return TGPU_OK; }
    r.type = parts[0]->type;
    int64_t n = 0;
    bool any_validity = false;
    for (auto* p : parts) {
        if (p->type != r.type) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "column type changed between pages (%d vs %d)", p->type, r.type);
        n += p->length;
        any_validity |= p->validity != nullptr;
    }
    r.length = n;
    if (r.type == TGPU_UTF8) {
        // value bytes back to back, offsets rebased chunk by chunk
        std::vector<int32_t> first(parts.size()), last(parts.size());
        for (size_t c = 0; c < parts.size(); c++) {
            first[c] = last[c] = 0;
            if (parts[c]->length == 0) continue;
            TG_CUDA(ctx, cudaMemcpyAsync(ctx->h_scratch, parts[c]->offsets, 4, cudaMemcpyDeviceToHost, ctx->stream));
            TG_CUDA(ctx, cudaMemcpyAsync((char*)ctx->h_scratch + 8, parts[c]->offsets + parts[c]->length, 4, cudaMemcpyDeviceToHost, ctx->stream));
            TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
            first[c] = *(int32_t*)ctx->h_scratch;
            last[c] = *(int32_t*)((char*)ctx->h_scratch + 8);
        }
        int64_t total_bytes = 0;
        for (size_t c = 0; c < parts.size(); c++) total_bytes += last[c] - first[c];
        if (total_bytes > INT32_MAX) return tg_fail(ctx, TGPU_ERR_INSUFFICIENT_RESOURCES, "variable-width column exceeds 2 GB");
        TG_TRY(alloc_shared(ctx, (size_t)(n + 1) * 4, &r.own_offsets));
        TG_TRY(alloc_shared(ctx, (size_t)total_bytes, &r.own_data));
        int64_t row = 0, byte = 0;
        for (size_t c = 0; c < parts.size(); c++) {
            int64_t len = parts[c]->length;
            if (len == 0) continue;
            TG_TRY(tg_add_i32(ctx, parts[c]->offsets, len + 1, (int32_t)(byte - first[c]), r.own_offsets->as<int32_t>() + row));
            if (last[c] > first[c])
                TG_CUDA(ctx, cudaMemcpyAsync(r.own_data->as<char>() + byte, (const char*)parts[c]->data + first[c], (size_t)(last[c] - first[c]), cudaMemcpyDeviceToDevice, ctx->stream));
            row += len;
            byte += last[c] - first[c];
        }
        if (n == 0) TG_CUDA(ctx, cudaMemsetAsync(r.own_offsets->p, 0, 4, ctx->stream));
        r.offsets = r.own_offsets->as<int32_t>();
        r.data = r.own_data->p;
        r.data_bytes = total_bytes;
    }
    else {
        int es = r.elem_size();
        if (es == 0) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "concat: unsupported column type %d", r.type);
        TG_TRY(alloc_shared(ctx, (size_t)n * es, &r.own_data));
        int64_t row = 0;
        for (auto* p : parts) {
            if (p->length) TG_CUDA(ctx, cudaMemcpyAsync(r.own_data->as<char>() + row * es, p->data, (size_t)p->length * es, cudaMemcpyDeviceToDevice, ctx->stream));
            row += p->length;
        }
        r.data = r.own_data->p;
    }
    if (any_validity && n > 0) {
        TG_TRY(alloc_shared(ctx, (size_t)((n + 7) / 8), &r.own_validity));
        // merge chunk runs so the kernel's table holds at most 64 entries per launch
        size_t c = 0;
        int64_t row = 0;
        if (parts.size() <= 64) {
            ConcatParts cp;
            memset(&cp, 0, sizeof(cp));
            cp.count = (int)parts.size();
            for (c = 0; c < parts.size(); c++) { cp.validity[c] = parts[c]->validity; cp.start[c] = row; row += parts[c]->length; }
            cp.start[parts.size()] = row;
            TG_LAUNCH(ctx, tg_concat_validity_kernel, tg_grid(ctx, (n + 7) / 8, 256, 8), 256, 0, cp, n, r.own_validity->as<uint8_t>());
        }
        else {
            // many small pages: fold 64 chunks at a time into an intermediate column, then concatenate those
            std::vector<DevColumn> mids;
            for (size_t at = 0; at < parts.size(); at += 64) {
                std::vector<const DevColumn*> group(parts.begin() + at, parts.begin() + std::min(parts.size(), at + 64));
                DevColumn mid;
                TG_TRY(tg_concat_columns(ctx, group, &mid));
                mids.push_back(std::move(mid));
            }
            std::vector<const DevColumn*> refs;
            for (auto& m : mids) refs.push_back(&m);
            return tg_concat_columns(ctx, refs, out);
        }
        r.validity = r.own_validity->as<uint8_t>();
    }
    *out = std::move(r);
    return TGPU_OK;
}

// registry of live library-owned pages, keyed by the first element of their column descriptor array
static std::mutex g_owned_lock;
static std::map<const tgpu_column*, OwnedPage*> g_owned;

void tg_owned_page_unregister(OwnedPage* page)
{
    if (page->cols.empty()) return;
    std::lock_guard<std::mutex> guard(g_owned_lock);
    auto it = g_owned.find(page->cols.data());
    if (it != g_owned.end() && it->second == page) g_owned.erase(it);
}

// `col` is a column descriptor of a live library-owned page: copy its DevColumn (shares the buffers' ownership)
static bool share_owned_column(const tgpu_column* col, DevColumn* out)
{
    std::lock_guard<std::mutex> guard(g_owned_lock);
    auto it = g_owned.upper_bound(col);
    if (it == g_owned.begin()) return false;
    --it;
    OwnedPage* o = it->second;
    size_t idx = (size_t)(col - it->first);
    if (idx >= o->cols.size() || &o->cols[idx] != col) return false;
    const DevColumn& d = o->page.cols[idx];
    if (d.data != col->data || d.length != col->length || d.type != col->type) return false;   // descriptor was edited by the caller
    *out = d;
    return true;
}

// upload (host) or borrow (device) `bytes` of a buffer
static int put_buffer(tgpu_ctx* ctx, const void* src, size_t bytes, bool device, std::shared_ptr<DevBuf>* own, const void** out)
{
    if (device) { *out = src; return TGPU_OK; }
    TG_TRY(alloc_shared(ctx, bytes, own));
    if (bytes) TG_CUDA(ctx, cudaMemcpyAsync((*own)->p, src, bytes, cudaMemcpyHostToDevice, ctx->stream));
    *out = (*own)->p;
    return TGPU_OK;
}

static int ingest_value_column(tgpu_ctx* ctx, const tgpu_column* col, bool device, DevColumn* out)
{
    if (device && share_owned_column(col, out)) return TGPU_OK;
    DevColumn r;
    r.type = col->type;
    r.length = col->length;
    int64_t n = col->length;
    if (col->validity) {
        if (col->flags & TGPU_COL_NULLS_BYTEMAP) {
            std::shared_ptr<DevBuf> raw;
            const void* d_raw = nullptr;
            TG_TRY(put_buffer(ctx, col->validity, (size_t)n, device, &raw, &d_raw));
            TG_TRY(alloc_shared(ctx, (size_t)((n + 7) / 8), &r.own_validity));
            TG_TRY(tg_pack_nullmap(ctx, (const uint8_t*)d_raw, n, r.own_validity->as<uint8_t>()));
            r.validity = r.own_validity->as<uint8_t>();
        }
        else {
            const void* v = nullptr;
            TG_TRY(put_buffer(ctx, col->validity, (size_t)((n + 7) / 8), device, &r.own_validity, &v));
            r.validity = (const uint8_t*)v;
        }
    }
    if (col->type == TGPU_UTF8) {
        if (!col->offsets) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "UTF8 column without offsets");
        const void* o = nullptr;
        TG_TRY(put_buffer(ctx, col->offsets, (size_t)(n + 1) * 4, device, &r.own_offsets, &o));
        r.offsets = (const int32_t*)o;
        int32_t first = 0, last = 0;
        if (device) {
            if (n > 0) {
                TG_CUDA(ctx, cudaMemcpyAsync(ctx->h_scratch, col->offsets, 4, cudaMemcpyDeviceToHost, ctx->stream));
                TG_CUDA(ctx, cudaMemcpyAsync((char*)ctx->h_scratch + 8, col->offsets + n, 4, cudaMemcpyDeviceToHost, ctx->stream));
                TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
                first = *(int32_t*)ctx->h_scratch;
                last = *(int32_t*)((char*)ctx->h_scratch + 8);
            }
            r.data = col->data;
        }
        else {
            first = n > 0 ? col->offsets[0] : 0;
            last = n > 0 ? col->offsets[n] : 0;
            const void* d = nullptr;
            TG_TRY(put_buffer(ctx, (const char*)col->data + first, (size_t)(last - first), false, &r.own_data, &d));
            r.data = (const char*)d - first;   // offsets stay absolute
        }
        r.data_bytes = last - first;
    }
    else {
        int es = r.elem_size();
        if (es == 0) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "unsupported column type %d", col->type);
        TG_TRY(put_buffer(ctx, col->data, (size_t)n * es, device, &r.own_data, &r.data));
    }
    *out = std::move(r);
    return TGPU_OK;
}

int tg_ingest_column(tgpu_ctx* ctx, const tgpu_column* col, bool device, DevColumn* out)
{
    if (col->type == TGPU_DICT32) {
        if (!col->dictionary) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "DICT32 column without dictionary");
        DevColumn dict;
        TG_TRY(tg_ingest_column(ctx, col->dictionary, device, &dict));
        std::shared_ptr<DevBuf> own_ids;
        const void* ids = nullptr;
        TG_TRY(put_buffer(ctx, col->data, (size_t)col->length * 4, device, &own_ids, &ids));
        return tg_gather_column(ctx, dict, (const int32_t*)ids, col->length, false, out);
    }
    if (col->type == TGPU_RLE) {
        if (!col->dictionary) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "RLE column without value");
        DevColumn value;
        TG_TRY(tg_ingest_column(ctx, col->dictionary, device, &value));
        return tg_gather_column(ctx, value, nullptr, col->length, false, out);
    }
    return ingest_value_column(ctx, col, device, out);
}

int tg_ingest_page(tgpu_ctx* ctx, const tgpu_page* page, DevPage* out)
{
    if (!page) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "page is null");
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    bool device = (page->flags & TGPU_PAGE_DEVICE) != 0;
    DevPage p;
    p.rows = page->num_rows;
    p.cols.resize(page->num_columns);
    for (int32_t c = 0; c < page->num_columns; c++) {
        if (page->columns[c].length != page->num_rows)
            return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "column %d has %lld positions, page has %lld", c,
                           (long long)page->columns[c].length, (long long)page->num_rows);
        TG_TRY(tg_ingest_column(ctx, &page->columns[c], device, &p.cols[c]));
    }
    // the caller keeps ownership of host buffers: the copies must have left them before we return
    if (!device) TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    *out = std::move(p);
    return TGPU_OK;
}

OwnedPage* tg_make_owned_page(DevPage&& page)
{
    OwnedPage* o = new OwnedPage();
    o->page = std::move(page);
    o->cols.resize(o->page.cols.size());
    for (size_t c = 0; c < o->page.cols.size(); c++) {
        const DevColumn& d = o->page.cols[c];
        tgpu_column& t = o->cols[c];
        memset(&t, 0, sizeof(t));
        t.type = d.type;
        t.length = d.length;
        t.data = d.data;
        t.offsets = d.offsets;
        t.validity = d.validity;
    }
    o->hdr.num_columns = (int32_t)o->cols.size();
    o->hdr.flags = TGPU_PAGE_DEVICE;
    o->hdr.num_rows = o->page.rows;
    o->hdr.columns = o->cols.data();
    if (!o->cols.empty()) {
        std::lock_guard<std::mutex> guard(g_owned_lock);
        g_owned[o->cols.data()] = o;
    }
    return o;
}

// ------------------------------------------------------------------------------------------------
// Operator protocol entry points
// ------------------------------------------------------------------------------------------------
extern "C" int tgpu_op_needs_input(tgpu_op* op, int* out)
{
    if (!op || !out) return TGPU_ERR_INVALID_ARGUMENT;
    *out = op->needs_input() ? 1 : 0;
    return TGPU_OK;
}

extern "C" int tgpu_op_add_input(tgpu_op* op, const tgpu_page* page)
{
    if (!op) return TGPU_ERR_INVALID_ARGUMENT;
    if (!page) return tg_fail(op->ctx, TGPU_ERR_INVALID_ARGUMENT, "page is null");
    // Operator.addInput contract: only legal when needsInput() (M/operator/Operator.java:49-53)
    if (!op->needs_input()) return tg_fail(op->ctx, TGPU_ERR_ILLEGAL_STATE, "addInput called while the operator does not need input");
    cudaSetDevice(op->ctx->device);
    return op->add_input(page);
}

extern "C" int tgpu_op_get_output(tgpu_op* op, tgpu_page** out)
{
    if (!op || !out) return TGPU_ERR_INVALID_ARGUMENT;
    cudaSetDevice(op->ctx->device);
    OwnedPage* o = nullptr;
    int s = op->get_output(&o);
    *out = o ? &o->hdr : nullptr;
    return s;
}

extern "C" int tgpu_op_finish(tgpu_op* op)
{
    if (!op) return TGPU_ERR_INVALID_ARGUMENT;
    cudaSetDevice(op->ctx->device);
    return op->finish();
}

extern "C" int tgpu_op_is_finished(tgpu_op* op, int* out)
{
    if (!op || !out) return TGPU_ERR_INVALID_ARGUMENT;
    *out = op->is_finished() ? 1 : 0;
    return TGPU_OK;
}

extern "C" int64_t tgpu_op_memory_bytes(tgpu_op* op) { return op ? op->memory_bytes() : 0; }

extern "C" void tgpu_op_close(tgpu_op* op)
{
    if (!op) return;
    cudaSetDevice(op->ctx->device);
    delete op;
}

extern "C" void tgpu_page_release(tgpu_ctx* ctx, tgpu_page* page)
{
    if (!page) return;
    if (ctx) cudaSetDevice(ctx->device);
    delete reinterpret_cast<OwnedPage*>(page);
}

extern "C" int tgpu_page_passthrough_channel(const tgpu_page* device_page, int32_t channel, int32_t* input_channel)
{
    if (!device_page || !input_channel) return TGPU_ERR_INVALID_ARGUMENT;
    const OwnedPage* o = reinterpret_cast<const OwnedPage*>(device_page);
    if (channel < 0 || channel >= (int32_t)o->cols.size()) return TGPU_ERR_INVALID_ARGUMENT;
    *input_channel = channel < (int32_t)o->passthrough.size() ? o->passthrough[channel] : -1;
    return TGPU_OK;
}

extern "C" int64_t tgpu_page_utf8_bytes(tgpu_ctx* ctx, const tgpu_page* device_page, int32_t channel)
{
    (void)ctx;
    const OwnedPage* o = reinterpret_cast<const OwnedPage*>(device_page);
    if (channel < 0 || channel >= (int32_t)o->page.cols.size()) return -1;
    return o->page.cols[channel].data_bytes;
}

extern "C" int tgpu_page_copy_to_host(tgpu_ctx* ctx, const tgpu_page* dp, tgpu_page* host)
{
    if (ctx) cudaSetDevice(ctx->device);     // callable from any thread: the calling thread's current device may differ
    if (!dp || !host) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "null page");
    if (host->num_columns != dp->num_columns) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "column count mismatch");
    int64_t n = dp->num_rows;
    for (int32_t c = 0; c < dp->num_columns; c++) {
        const tgpu_column& d = dp->columns[c];
        tgpu_column& h = const_cast<tgpu_column&>(host->columns[c]);
        h.type = d.type;
        h.length = n;
        if (!h.data) continue;   // the caller does not want this column (e.g. a pass-through block it already holds)
        if (!d.data && n > 0 && d.type != TGPU_UTF8)
            return tg_fail(ctx, TGPU_ERR_ILLEGAL_STATE, "column %d is a by-reference view of an input block (tgpu_page_passthrough_channel): it has no device data", c);
        if (d.type == TGPU_UTF8) {
            TG_CUDA(ctx, cudaMemcpyAsync((void*)h.offsets, d.offsets, (size_t)(n + 1) * 4, cudaMemcpyDeviceToHost, ctx->stream));
            TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
            int32_t first = n > 0 ? h.offsets[0] : 0, last = n > 0 ? h.offsets[n] : 0;
            if (last > first)
                TG_CUDA(ctx, cudaMemcpyAsync((char*)h.data + first, (const char*)d.data + first, (size_t)(last - first), cudaMemcpyDeviceToHost, ctx->stream));
        }
        else {
            int es = d.type == TGPU_INT128 ? 16 : d.type == TGPU_INT64 || d.type == TGPU_FLOAT64 ? 8 : d.type == TGPU_INT32 || d.type == TGPU_FLOAT32 ? 4 : d.type == TGPU_INT16 ? 2 : 1;
            if (n) TG_CUDA(ctx, cudaMemcpyAsync((void*)h.data, d.data, (size_t)n * es, cudaMemcpyDeviceToHost, ctx->stream));
        }
        if (d.validity) {
            if (!h.validity) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "column %d has nulls but the host page has no validity buffer", c);
            TG_CUDA(ctx, cudaMemcpyAsync((void*)h.validity, d.validity, (size_t)((n + 7) / 8), cudaMemcpyDeviceToHost, ctx->stream));
            h.flags = 0;
        }
        else if (h.validity) {
            memset((void*)h.validity, 0xFF, (size_t)((n + 7) / 8));
        }
    }
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return TGPU_OK;
}
