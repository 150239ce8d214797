// serde.cu — the reference's page wire format to and from device columns (SURVEY.md §8(f) rank 1).
//
// (round 1 left this on a branch; merged and run on hardware in round 2: tests/test_gpu_serde.py)
//
// Format (uncompressed, unencrypted; all integers little-endian) — restated in oracle/serde.py with the reference lines:
//   serialized page = int32 positionCount | int32 uncompressedSize | int32 compressedSize | raw page
//                     (M/execution/buffer/PagesSerdeUtil.java:44-48, CompressingEncryptingPageSerializer.java:173-181,351-361)
//   raw page        = int32 channelCount | block*                      (PagesSerdeUtil.java:58-64)
//   block           = int32 nameLength | name | int32 positionCount | byte hasNulls [| MSB-first NULL bits] | values
//                     LONG_ARRAY / INT_ARRAY / SHORT_ARRAY / BYTE_ARRAY: n values, or int32 nonNullCount + the non-NULL values
//                     (S/block/LongArrayBlockEncoding.java:61-133, EncoderUtil.java:35-70)
//                     VARIABLE_WIDTH: int32 nonNullCount | ending offsets of the non-NULL positions (from 0) | bytes
//                     (S/block/VariableWidthBlockEncoding.java:57-146)
//
// Shape: the byte stream lives in HOST memory (it goes to / comes from the HTTP exchange), so the device only does the two
// data-parallel pieces per column — the NULL bit transform (Arrow LSB-first validity <-> MSB-first is-NULL bits: one byte in, one
// byte out) and the NULL compaction / expansion of the values (ordered stream compaction, CUB) — and every piece is copied
// straight between its place in the pinned stream and the device with cudaMemcpyAsync.  Small fields are written by the host.
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <thrust/iterator/transform_iterator.h>

#include "common.cuh"

namespace {

using namespace tg;

// Arrow validity byte (bit i = position 8k+i is valid) -> wire byte (bit 7-i = position 8k+i is NULL); tail bits of the last byte 0
__global__ void serde_nullbits_encode_kernel(const uint8_t* __restrict__ validity, int64_t n, uint8_t* __restrict__ out)
{
    int64_t nb = (n + 7) / 8;
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < nb; i += stride) {
        unsigned int v = (unsigned int)(uint8_t)~validity[i];
        int live = (int)min((int64_t)8, n - i * 8);
        v &= (1u << live) - 1;                       // positions past the end are not NULL
        out[i] = (uint8_t)(__brev(v) >> 24);
    }
}

// wire byte -> Arrow validity byte (tail bits of the last byte set: "valid", never read)
__global__ void serde_nullbits_decode_kernel(const uint8_t* __restrict__ in, int64_t n, uint8_t* __restrict__ validity)
{
    int64_t nb = (n + 7) / 8;
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < nb; i += stride) validity[i] = (uint8_t)~(__brev((unsigned int)in[i]) >> 24);
}

struct ValidAt {
    const uint8_t* validity;
    __host__ __device__ unsigned char operator()(int64_t i) const { return (validity[i >> 3] >> (i & 7)) & 1; }
};

// expansion: position i takes compacted[rank of i among the valid positions]; NULL positions read as 0
// (LongArrayBlockEncoding.expandLongsWithNulls*)
template <class T>
__global__ void serde_expand_kernel(const T* __restrict__ compacted, const uint8_t* __restrict__ validity, const int* __restrict__ rank, int64_t n, T* __restrict__ out)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) out[i] = ((validity[i >> 3] >> (i & 7)) & 1) ? compacted[rank[i]] : T();
}

// VARIABLE_WIDTH write: ending offset of every position relative to the first (NULL positions have zero length)
__global__ void serde_end_offsets_kernel(const int32_t* __restrict__ offsets, int64_t n, int32_t* __restrict__ ends)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    int32_t first = offsets[0];
    for (; i < n; i += stride) ends[i] = offsets[i + 1] - first;
}

// VARIABLE_WIDTH read: offsets[i + 1] = ending offset of the last non-NULL position <= i (readOffsetsWithNullsCompacted)
__global__ void serde_expand_offsets_kernel(const int32_t* __restrict__ ends, const uint8_t* __restrict__ validity, const int* __restrict__ rank, int64_t n,
                                            int32_t* __restrict__ offsets)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    if (i == 0) offsets[0] = 0;
    for (; i < n; i += stride) {
        int r = rank[i] + (((validity[i >> 3] >> (i & 7)) & 1) ? 1 : 0);     // non-NULL positions among [0, i]
        offsets[i + 1] = r > 0 ? ends[r - 1] : 0;
    }
}

const char* encoding_name(int32_t type)
{
    switch (type) {
        case TGPU_INT128: return "INT128_ARRAY";     // S/block/Int128ArrayBlockEncoding.java:52-84: LONG_ARRAY's body with two longs per position
        case TGPU_INT64: case TGPU_FLOAT64: return "LONG_ARRAY";
        case TGPU_INT32: case TGPU_FLOAT32: return "INT_ARRAY";
        case TGPU_INT16: return "SHORT_ARRAY";
        case TGPU_INT8: return "BYTE_ARRAY";
        case TGPU_UTF8: return "VARIABLE_WIDTH";
        default: return nullptr;
    }
}

void put_i32(uint8_t* p, int32_t v) { memcpy(p, &v, 4); }
int32_t get_i32(const uint8_t* p) { int32_t v; memcpy(&v, p, 4); return v; }

// exclusive rank of every position among the valid ones (int32[n]) and the number of valid positions
int valid_ranks(tgpu_ctx* ctx, const uint8_t* validity, int64_t n, DevBuf* rank, int64_t* valid_count)
{
    TG_TRY(rank->alloc(ctx, (size_t)(n + 1) * 4));
    thrust::counting_iterator<int64_t> idx(0);
    auto flags = thrust::make_transform_iterator(idx, ValidAt{validity});
    size_t tmp_bytes = 0;
    DevBuf tmp;
    cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, flags, rank->as<int>(), (int)(n + 1), ctx->stream);
    TG_TRY(tmp.alloc(ctx, tmp_bytes));
    // n + 1 outputs: rank[n] = number of valid positions (the iterator is read one past the end: validity buffers are padded to
    // whole bytes and position n of the last byte is a defined bit; when n is a multiple of 8 the scan is split instead)
    if (n % 8 != 0) {
        TG_CUDA(ctx, cub::DeviceScan::ExclusiveSum(tmp.p, tmp_bytes, flags, rank->as<int>(), (int)(n + 1), ctx->stream));
        int32_t total = 0;
        TG_CUDA(ctx, cudaMemcpyAsync(&total, rank->as<int>() + n, 4, cudaMemcpyDeviceToHost, ctx->stream));
        TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        *valid_count = total;
        return TGPU_OK;
    }
    TG_CUDA(ctx, cub::DeviceScan::ExclusiveSum(tmp.p, tmp_bytes, flags, rank->as<int>(), (int)n, ctx->stream));
    int32_t last_rank = 0;
    uint8_t last_byte = 0;
    if (n > 0) {
        TG_CUDA(ctx, cudaMemcpyAsync(&last_rank, rank->as<int>() + (n - 1), 4, cudaMemcpyDeviceToHost, ctx->stream));
        TG_CUDA(ctx, cudaMemcpyAsync(&last_byte, validity + ((n - 1) >> 3), 1, cudaMemcpyDeviceToHost, ctx->stream));
        TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    *valid_count = n > 0 ? last_rank + ((last_byte >> ((n - 1) & 7)) & 1) : 0;
    return TGPU_OK;
}

}  // namespace

// Upper bound of the serialized size of `page` (host or device): what the caller must provide to tgpu_page_serialize.
extern "C" int64_t tgpu_page_serialized_size_bound(const tgpu_page* page)
{
    if (!page) return -1;
    int64_t total = 12 + 4;
    for (int32_t c = 0; c < page->num_columns; c++) {
        const tgpu_column& col = page->columns[c];
        const char* name = encoding_name(col.type);
        if (!name) return -1;
        int64_t n = page->num_rows;
        total += 4 + (int64_t)strlen(name) + 4 + 1 + (n + 7) / 8 + 4;
        if (col.type == TGPU_UTF8) total += 4 * n + (1LL << 31);      // the byte payload is only known on the device: see below
        else total += n * (col.type == TGPU_INT128 ? 16 : col.type == TGPU_INT64 || col.type == TGPU_FLOAT64 ? 8 : col.type == TGPU_INT32 || col.type == TGPU_FLOAT32 ? 4 : col.type == TGPU_INT16 ? 2 : 1);
    }
    return total;
}

// PageSerializer.serialize (uncompressed): device or host page -> wire bytes in `out` (host memory, pinned for speed).
extern "C" int tgpu_page_serialize(tgpu_ctx* ctx, const tgpu_page* page, uint8_t* out, int64_t capacity, int64_t* bytes_out)
{
    if (!ctx || !page || !out || !bytes_out) return TGPU_ERR_INVALID_ARGUMENT;
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    DevPage in;
    TG_TRY(tg_ingest_page(ctx, page, &in));
    const int64_t n = in.rows;
    if (n > (int64_t)INT32_MAX) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "page has more than 2^31-1 positions");
    int64_t pos = 12;
    auto need = [&](int64_t more) -> int {
        if (pos + more > capacity) return tg_fail(ctx, TGPU_ERR_INSUFFICIENT_RESOURCES, "serialized page does not fit the %lld-byte buffer", (long long)capacity);
        return TGPU_OK;
    };
    TG_TRY(need(4));
    put_i32(out + pos, (int32_t)in.cols.size());
    pos += 4;
    std::vector<DevBuf> keep;      // device pieces whose D2H copies are in flight
    for (const DevColumn& col : in.cols) {
        const char* name = encoding_name(col.type);
        if (!name) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "no block encoding for column type %d", col.type);
        const int32_t name_len = (int32_t)strlen(name);
        TG_TRY(need(4 + name_len + 4 + 1));
        put_i32(out + pos, name_len);
        memcpy(out + pos + 4, name, (size_t)name_len);
        pos += 4 + name_len;
        put_i32(out + pos, (int32_t)n);
        pos += 4;
        // a column carries NULL bits iff it has a validity bitmap with at least one NULL (the restatement's convention, oracle/serde.py)
        DevBuf rank;
        int64_t valid = n;
        bool has_nulls = false;
        if (col.validity && n > 0) {
            TG_TRY(valid_ranks(ctx, col.validity, n, &rank, &valid));
            has_nulls = valid < n;
        }
        out[pos++] = has_nulls ? 1 : 0;
        if (has_nulls) {
            const int64_t nb = (n + 7) / 8;
            TG_TRY(need(nb));
            DevBuf bits;
            TG_TRY(bits.alloc(ctx, (size_t)nb));
            TG_LAUNCH(ctx, serde_nullbits_encode_kernel, tg_grid(ctx, nb, 256, 8), 256, 0, col.validity, n, bits.as<uint8_t>());
            TG_CUDA(ctx, cudaMemcpyAsync(out + pos, bits.p, (size_t)nb, cudaMemcpyDeviceToHost, ctx->stream));
            pos += nb;
            keep.push_back(std::move(bits));
        }
        const int es = col.elem_size();
        if (es > 0) {
            if (!has_nulls) {
                TG_TRY(need(n * es));
                if (n) TG_CUDA(ctx, cudaMemcpyAsync(out + pos, col.data, (size_t)n * es, cudaMemcpyDeviceToHost, ctx->stream));
                pos += n * es;
            }
            else {
                TG_TRY(need(4 + valid * es));
                put_i32(out + pos, (int32_t)valid);
                pos += 4;
                DevBuf compact, tmp;
                TG_TRY(compact.alloc(ctx, (size_t)std::max<int64_t>(valid, 1) * es));
                long long* d_count = (long long*)(ctx->d_scratch + 40);
                thrust::counting_iterator<int64_t> idx(0);
                auto flags = thrust::make_transform_iterator(idx, ValidAt{col.validity});
                size_t tmp_bytes = 0;
#define SERDE_SELECT(T)                                                                                                                       \
    cub::DeviceSelect::Flagged(nullptr, tmp_bytes, (const T*)col.data, flags, compact.as<T>(), d_count, (int)n, ctx->stream);                \
    TG_TRY(tmp.alloc(ctx, tmp_bytes));                                                                                                        \
    TG_CUDA(ctx, cub::DeviceSelect::Flagged(tmp.p, tmp_bytes, (const T*)col.data, flags, compact.as<T>(), d_count, (int)n, ctx->stream));
                if (es == 16) { SERDE_SELECT(longlong2) }
                else if (es == 8) { SERDE_SELECT(long long) }
                else if (es == 4) { SERDE_SELECT(int) }
                else if (es == 2) { SERDE_SELECT(short) }
                else { SERDE_SELECT(signed char) }
#undef SERDE_SELECT
                if (valid) TG_CUDA(ctx, cudaMemcpyAsync(out + pos, compact.p, (size_t)valid * es, cudaMemcpyDeviceToHost, ctx->stream));
                pos += valid * es;
                keep.push_back(std::move(compact));
                keep.push_back(std::move(tmp));
            }
        }
        else {
            // VARIABLE_WIDTH: ending offsets from 0 of the non-NULL positions, then the bytes [offsets[0], offsets[n])
            TG_TRY(need(4 + valid * 4));
            put_i32(out + pos, (int32_t)valid);
            pos += 4;
            int32_t first = 0, last = 0;
            if (n > 0) {
                DevBuf ends, compact, tmp;
                TG_TRY(ends.alloc(ctx, (size_t)n * 4));
                TG_LAUNCH(ctx, serde_end_offsets_kernel, tg_grid(ctx, n, 1024, 8), 256, 0, col.offsets, n, ends.as<int32_t>());
                const int32_t* src = ends.as<int32_t>();
                if (has_nulls) {
                    TG_TRY(compact.alloc(ctx, (size_t)std::max<int64_t>(valid, 1) * 4));
                    long long* d_count = (long long*)(ctx->d_scratch + 40);
                    thrust::counting_iterator<int64_t> idx(0);
                    auto flags = thrust::make_transform_iterator(idx, ValidAt{col.validity});
                    size_t tmp_bytes = 0;
                    cub::DeviceSelect::Flagged(nullptr, tmp_bytes, ends.as<int32_t>(), flags, compact.as<int32_t>(), d_count, (int)n, ctx->stream);
                    TG_TRY(tmp.alloc(ctx, tmp_bytes));
                    TG_CUDA(ctx, cub::DeviceSelect::Flagged(tmp.p, tmp_bytes, ends.as<int32_t>(), flags, compact.as<int32_t>(), d_count, (int)n, ctx->stream));
                    src = compact.as<int32_t>();
                }
                if (valid) TG_CUDA(ctx, cudaMemcpyAsync(out + pos, src, (size_t)valid * 4, cudaMemcpyDeviceToHost, ctx->stream));
                TG_CUDA(ctx, cudaMemcpyAsync(&first, col.offsets, 4, cudaMemcpyDeviceToHost, ctx->stream));
                TG_CUDA(ctx, cudaMemcpyAsync(&last, col.offsets + n, 4, cudaMemcpyDeviceToHost, ctx->stream));
                TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
                keep.push_back(std::move(ends));
                keep.push_back(std::move(compact));
                keep.push_back(std::move(tmp));
            }
            pos += valid * 4;
            const int64_t payload = (int64_t)last - first;
            TG_TRY(need(payload));
            if (payload) TG_CUDA(ctx, cudaMemcpyAsync(out + pos, (const char*)col.data + first, (size_t)payload, cudaMemcpyDeviceToHost, ctx->stream));
            pos += payload;
        }
    }
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    put_i32(out, (int32_t)n);
    put_i32(out + 4, (int32_t)(pos - 12));
    put_i32(out + 8, (int32_t)(pos - 12));
    *bytes_out = pos;
    return TGPU_OK;
}

// PageDeserializer (uncompressed): wire bytes in host memory -> device page.  `types`: tgpu_type of every channel (the wire carries
// the block encoding, not the SQL type: LONG_ARRAY is TGPU_INT64 or TGPU_FLOAT64).
extern "C" int tgpu_page_deserialize(tgpu_ctx* ctx, const uint8_t* data, int64_t length, const int32_t* types, int32_t num_types, tgpu_page** out)
{
    if (!ctx || !data || !out || length < 16) return TGPU_ERR_INVALID_ARGUMENT;
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    *out = nullptr;
    const int64_t n = get_i32(data);
    if (get_i32(data + 8) != length - 12 || get_i32(data + 4) != get_i32(data + 8))
        return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "compressed, encrypted or truncated serialized page");
    int64_t pos = 12;
    const int32_t channels = get_i32(data + pos);
    pos += 4;
    if (channels != num_types) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "page has %d channels, %d types given", channels, num_types);
    auto need = [&](int64_t more) -> int {
        if (pos + more > length) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "serialized page is truncated");
        return TGPU_OK;
    };
    DevPage page;
    page.rows = n;
    page.cols.resize(channels);
    std::vector<DevBuf> keep;
    for (int32_t c = 0; c < channels; c++) {
        DevColumn& col = page.cols[c];
        col.type = types[c];
        col.length = n;
        const char* want = encoding_name(types[c]);
        if (!want) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "no block encoding for column type %d", types[c]);
        TG_TRY(need(4));
        const int32_t name_len = get_i32(data + pos);
        pos += 4;
        TG_TRY(need(name_len + 5));
        if (name_len != (int32_t)strlen(want) || memcmp(data + pos, want, (size_t)name_len) != 0)
            return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "channel %d: block encoding %.*s, expected %s (dictionary / RLE / nested blocks: keep the Java reader)", c,
                           name_len, (const char*)(data + pos), want);
        pos += name_len;
        if (get_i32(data + pos) != n) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "channel %d has %d positions, page has %lld", c, get_i32(data + pos), (long long)n);
        pos += 4;
        const bool has_nulls = data[pos++] != 0;
        DevBuf rank;
        int64_t valid = n;
        if (has_nulls) {
            const int64_t nb = (n + 7) / 8;
            TG_TRY(need(nb));
            DevBuf wire;
            TG_TRY(wire.alloc(ctx, (size_t)std::max<int64_t>(nb, 1)));
            col.own_validity = std::make_shared<DevBuf>();
            TG_TRY(col.own_validity->alloc(ctx, (size_t)std::max<int64_t>(nb, 1)));
            TG_CUDA(ctx, cudaMemcpyAsync(wire.p, data + pos, (size_t)nb, cudaMemcpyHostToDevice, ctx->stream));
            TG_LAUNCH(ctx, serde_nullbits_decode_kernel, tg_grid(ctx, nb, 256, 8), 256, 0, wire.as<uint8_t>(), n, col.own_validity->as<uint8_t>());
            col.validity = col.own_validity->as<uint8_t>();
            pos += nb;
            TG_TRY(valid_ranks(ctx, col.validity, n, &rank, &valid));
            keep.push_back(std::move(wire));
        }
        const int es = col.elem_size();
        if (es > 0) {
            col.own_data = std::make_shared<DevBuf>();
            TG_TRY(col.own_data->alloc(ctx, (size_t)std::max<int64_t>(n, 1) * es));
            col.data = col.own_data->p;
            if (!has_nulls) {
                TG_TRY(need(n * es));
                if (n) TG_CUDA(ctx, cudaMemcpyAsync(col.own_data->p, data + pos, (size_t)n * es, cudaMemcpyHostToDevice, ctx->stream));
                pos += n * es;
            }
            else {
                TG_TRY(need(4));
                const int64_t k = get_i32(data + pos);
                pos += 4;
                if (k != valid) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "channel %d: %lld values for %lld non-NULL positions", c, (long long)k, (long long)valid);
                TG_TRY(need(k * es));
                DevBuf compact;
                TG_TRY(compact.alloc(ctx, (size_t)std::max<int64_t>(k, 1) * es));
                if (k) TG_CUDA(ctx, cudaMemcpyAsync(compact.p, data + pos, (size_t)k * es, cudaMemcpyHostToDevice, ctx->stream));
                pos += k * es;
                int grid = tg_grid(ctx, n, 1024, 8);
                if (es == 16) TG_LAUNCH(ctx, serde_expand_kernel<longlong2>, grid, 256, 0, compact.as<longlong2>(), col.validity, rank.as<int>(), n, col.own_data->as<longlong2>());
                else if (es == 8) TG_LAUNCH(ctx, serde_expand_kernel<long long>, grid, 256, 0, compact.as<long long>(), col.validity, rank.as<int>(), n, col.own_data->as<long long>());
                else if (es == 4) TG_LAUNCH(ctx, serde_expand_kernel<int>, grid, 256, 0, compact.as<int>(), col.validity, rank.as<int>(), n, col.own_data->as<int>());
                else if (es == 2) TG_LAUNCH(ctx, serde_expand_kernel<short>, grid, 256, 0, compact.as<short>(), col.validity, rank.as<int>(), n, col.own_data->as<short>());
                else TG_LAUNCH(ctx, serde_expand_kernel<signed char>, grid, 256, 0, compact.as<signed char>(), col.validity, rank.as<int>(), n, col.own_data->as<signed char>());
                keep.push_back(std::move(compact));
            }
        }
        else {
            TG_TRY(need(4));
            const int64_t k = get_i32(data + pos);
            pos += 4;
            if (k != valid) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "channel %d: %lld offsets for %lld non-NULL positions", c, (long long)k, (long long)valid);
            TG_TRY(need(k * 4));
            const int64_t payload = k > 0 ? get_i32(data + pos + (k - 1) * 4) : 0;
            col.own_offsets = std::make_shared<DevBuf>();
            TG_TRY(col.own_offsets->alloc(ctx, (size_t)(n + 1) * 4));
            col.offsets = col.own_offsets->as<int32_t>();
            if (!has_nulls) {
                TG_CUDA(ctx, cudaMemsetAsync(col.own_offsets->p, 0, 4, ctx->stream));
                if (n) TG_CUDA(ctx, cudaMemcpyAsync(col.own_offsets->as<int32_t>() + 1, data + pos, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
            }
            else {
                DevBuf ends;
                TG_TRY(ends.alloc(ctx, (size_t)std::max<int64_t>(k, 1) * 4));
                if (k) TG_CUDA(ctx, cudaMemcpyAsync(ends.p, data + pos, (size_t)k * 4, cudaMemcpyHostToDevice, ctx->stream));
                if (n) TG_LAUNCH(ctx, serde_expand_offsets_kernel, tg_grid(ctx, n, 1024, 8), 256, 0, ends.as<int32_t>(), col.validity, rank.as<int>(), n, col.own_offsets->as<int32_t>());
                else TG_CUDA(ctx, cudaMemsetAsync(col.own_offsets->p, 0, 4, ctx->stream));
                keep.push_back(std::move(ends));
            }
            pos += k * 4;
            TG_TRY(need(payload));
            col.own_data = std::make_shared<DevBuf>();
            TG_TRY(col.own_data->alloc(ctx, (size_t)std::max<int64_t>(payload, 1)));
            col.data = col.own_data->p;
            if (payload) TG_CUDA(ctx, cudaMemcpyAsync(col.own_data->p, data + pos, (size_t)payload, cudaMemcpyHostToDevice, ctx->stream));
            pos += payload;
        }
        keep.push_back(std::move(rank));
    }
    if (pos != length) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "%lld trailing bytes after the last block", (long long)(length - pos));
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));     // the caller's buffer is free again; staging pieces are released
    OwnedPage* o = tg_make_owned_page(std::move(page));
    *out = &o->hdr;
    return TGPU_OK;
}
