// strdict.cuh — device string dictionary: variable-width GROUP BY keys become dense fixed-width ids.
//
// Reference: FlatHash keeps variable-width key bytes in AppendOnlyVariableWidthData next to fixed-size records
// (M/operator/FlatHash.java:309-348, M/operator/AppendOnlyVariableWidthData.java:46, record layout by
// M/operator/FlatHashStrategyCompiler.java:125-146) and compares full values on a hash hit (FlatHash.valueIdentical :445-469).
// Here every UTF8 key column of a group-by owns one StringDict: an append-only byte store (the AppendOnlyVariableWidthData
// analogue) plus an open-addressing table from string to a dense int32 id.  A page's key column is translated to ids in a
// pre-pass and the group-by itself - shared-memory path, general path, first-seen ids, output - runs on fixed-width keys
// (30 bits per string key inside the packed composite key); the output step turns ids back into strings.
//
// Identity is exact, not probabilistic:
//   - strings of up to 7 bytes are keyed by (length << 56 | bytes): the key IS the string (bit 63 clear);
//   - longer strings are keyed by XXH64(bytes, seed = attempt) with bit 63 set and every hit is compared byte by byte with the
//     slot's string (the stored bytes, or the bytes of the slot's first row in this page while the slot is still new); a row
//     whose bytes differ - two strings sharing a 64-bit hash - moves on to attempt + 1, a different hash function of the same
//     bytes: chaining by rehash, never a query failure.
#pragma once
#include "common.cuh"

namespace tg {

struct __align__(16) StrSlot {
    unsigned long long key;
    int id;            // -1 while the string is new in the current page
    int first_row;     // lowest row of the current page that mapped here (owner of a new slot)
};

constexpr unsigned long long SD_EMPTY = ~0ULL;
constexpr int SD_MAX_ATTEMPTS = 8;
constexpr int64_t SD_MAX_IDS = 1LL << 30;     // ids travel as 30-bit fields of the packed group-by key

__device__ __forceinline__ unsigned long long sd_key(const uint8_t* p, int len, int attempt)
{
    if (len <= 7 && attempt == 0) {
        unsigned long long k = (unsigned long long)len << 56;
        for (int i = 0; i < len; i++) k |= (unsigned long long)p[i] << (8 * i);
        return k;
    }
    unsigned long long h = xxh64_bytes(p, len, (uint64_t)attempt) | (1ULL << 63);
    return h == SD_EMPTY ? h - 1 : h;
}

__device__ __forceinline__ bool sd_bytes_equal(const uint8_t* a, const uint8_t* b, int len)
{
    for (int i = 0; i < len; i++)
        if (a[i] != b[i]) return false;
    return true;
}

__global__ void sd_init_kernel(StrSlot* table, int64_t cap)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < cap; i += stride) { table[i].key = SD_EMPTY; table[i].id = -1; table[i].first_row = 0x7FFFFFFF; }
}

// find-or-claim the slot of every listed row's string (`rows` == nullptr: rows [0, n)).  counters: [0] slots claimed by this
// launch, [1] overflow flag (claims beyond `budget`: the host grows the table and re-runs the page)
__global__ void __launch_bounds__(256) sd_insert_kernel(const int32_t* __restrict__ offsets, const uint8_t* __restrict__ bytes, const uint8_t* __restrict__ validity,
                                                       const int* __restrict__ rows, int64_t n, const uint8_t* __restrict__ attempt, StrSlot* __restrict__ table,
                                                       unsigned long long mask, int* __restrict__ slot_of_row, int* __restrict__ counters, int budget)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        const int row = rows ? rows[i] : (int)i;
        if (!tg_valid(validity, row)) { slot_of_row[row] = -1; continue; }
        const int off = offsets[row], len = offsets[row + 1] - off;
        const unsigned long long key = sd_key(bytes + off, len, attempt[row]);
        unsigned long long pos = murmur3_mix(key) & mask;
        int found = -2;
        while (true) {
            unsigned long long cur = *((volatile unsigned long long*)&table[pos].key);
            if (cur == SD_EMPTY) {
                if (atomicAdd(counters, 1) >= budget) { atomicSub(counters, 1); counters[1] = 1; break; }
                cur = atomicCAS(&table[pos].key, SD_EMPTY, key);
                if (cur == SD_EMPTY) { found = (int)pos; break; }
                atomicSub(counters, 1);            // lost the race for this slot: the claim was not consumed
            }
            if (cur == key) { found = (int)pos; break; }
            pos = (pos + 1) & mask;
        }
        slot_of_row[row] = found;
        if (found >= 0 && *((volatile int*)&table[found].id) < 0) {
            // rows of one warp that share a new slot elect their lowest row; it touches the slot only if it would lower the owner
            // (a page of 10^9 rows over three new strings would otherwise serialise 10^9 atomics on three addresses)
            const unsigned int peers = __match_any_sync(__activemask(), found);
            const int lowest = __reduce_min_sync(peers, row);
            if (row == lowest && *((volatile int*)&table[found].first_row) > row) atomicMin(&table[found].first_row, row);
        }
    }
}

// fast path for pages whose strings are (almost) all known: look up, write the id, flag the chunk on a miss.  One pass: offsets + bytes
// in, ids out.  chunk_miss[row / chunk_rows] != 0 -> that chunk has to go through the insert path.
__device__ __forceinline__ int sd_find(const uint8_t* __restrict__ p, int len, const StrSlot* __restrict__ table, unsigned long long mask,
                                       const uint8_t* __restrict__ dict_bytes, const long long* __restrict__ dict_start, const int* __restrict__ dict_len,
                                       unsigned long long key0)
{
    for (int attempt = 0; attempt < SD_MAX_ATTEMPTS; attempt++) {
        const unsigned long long key = attempt == 0 ? key0 : sd_key(p, len, attempt);
        unsigned long long pos = murmur3_mix(key) & mask;
        bool other = false;       // a slot with this key holds a different string: try the next hash function
        while (true) {
            const int4 raw = __ldg((const int4*)&table[pos]);
            const unsigned long long skey = (unsigned long long)(unsigned int)raw.x | ((unsigned long long)(unsigned int)raw.y << 32);
            if (skey == SD_EMPTY) break;
            if (skey == key && raw.z >= 0) {
                if ((len <= 7 && attempt == 0) || (dict_len[raw.z] == len && sd_bytes_equal(p, dict_bytes + dict_start[raw.z], len))) return raw.z;
                other = true;
            }
            pos = (pos + 1) & mask;
        }
        if (!other) return -1;
    }
    return -1;
}

// R rows per thread: the offsets of the R rows first, then their (first) bytes, then the table probes - independent chains
__global__ void __launch_bounds__(256) sd_lookup_kernel(const int32_t* __restrict__ offsets, const uint8_t* __restrict__ bytes, const uint8_t* __restrict__ validity,
                                                       int64_t first, int64_t n, const StrSlot* __restrict__ table, unsigned long long mask,
                                                       const uint8_t* __restrict__ dict_bytes, const long long* __restrict__ dict_start, const int* __restrict__ dict_len,
                                                       int32_t* __restrict__ ids, int64_t chunk_rows, int* __restrict__ chunk_miss)
{
    constexpr int R = 4;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t base = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; base < n; base += stride * R) {
        int off[R], len[R];
        unsigned long long key[R];
        bool live[R];
#pragma unroll
        for (int j = 0; j < R; j++) {
            const int64_t i = base + (int64_t)j * stride;
            live[j] = i < n && tg_valid(validity, first + i);
            off[j] = 0; len[j] = 0;
            if (live[j]) { off[j] = __ldg(offsets + first + i); len[j] = __ldg(offsets + first + i + 1) - off[j]; }
        }
#pragma unroll
        for (int j = 0; j < R; j++) key[j] = live[j] ? sd_key(bytes + off[j], len[j], 0) : 0;
#pragma unroll
        for (int j = 0; j < R; j++) {
            const int64_t i = base + (int64_t)j * stride;
            if (i >= n) continue;
            int id = 0;
            if (live[j]) {
                id = sd_find(bytes + off[j], len[j], table, mask, dict_bytes, dict_start, dict_len, key[j]);
                if (id < 0) { chunk_miss[i / chunk_rows] = 1; id = 0; }
            }
            ids[first + i] = id;
        }
    }
}

// first tier for columns of very short strings (VARCHAR(1) flags, status codes): strings of length <= 1 resolve through a 257-entry direct
// map (byte value, or 256 for the empty string) held in shared memory - offsets + byte in, id out, ~20 instructions per row.  A longer
// or yet unmapped string flags its chunk for the general lookup / insert path.
__global__ void __launch_bounds__(256) sd_lookup_direct_kernel(const int32_t* __restrict__ offsets, const uint8_t* __restrict__ bytes, const uint8_t* __restrict__ validity,
                                                              int64_t first, int64_t n, const int32_t* __restrict__ direct, int32_t* __restrict__ ids,
                                                              int64_t chunk_rows, int* __restrict__ chunk_miss)
{
    __shared__ int32_t map[257];
    for (int i = threadIdx.x; i < 257; i += blockDim.x) map[i] = direct[i];
    __syncthreads();
    constexpr int R = 4;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t base = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; base < n; base += stride * R) {
        int off[R], len[R];
#pragma unroll
        for (int j = 0; j < R; j++) {
            const int64_t i = base + (int64_t)j * stride;
            off[j] = 0; len[j] = -1;
            if (i < n) { off[j] = __ldg(offsets + first + i); len[j] = __ldg(offsets + first + i + 1) - off[j]; }
        }
        int code[R];
#pragma unroll
        for (int j = 0; j < R; j++) code[j] = len[j] == 1 ? (int)__ldg(bytes + off[j]) : 256;
#pragma unroll
        for (int j = 0; j < R; j++) {
            const int64_t i = base + (int64_t)j * stride;
            if (i >= n) continue;
            int id = 0;
            if (tg_valid(validity, first + i)) {
                id = len[j] <= 1 ? map[code[j]] : -1;
                if (id < 0) { chunk_miss[i / chunk_rows] = 1; id = 0; }
            }
            ids[first + i] = id;
        }
    }
}

// long strings only: compare the row's bytes with its slot's string; rows that differ go to `retry` with attempt + 1
__global__ void __launch_bounds__(256) sd_verify_kernel(const int32_t* __restrict__ offsets, const uint8_t* __restrict__ bytes, const int* __restrict__ rows, int64_t n,
                                                       uint8_t* __restrict__ attempt, const StrSlot* __restrict__ table, const int* __restrict__ slot_of_row,
                                                       const uint8_t* __restrict__ dict_bytes, const long long* __restrict__ dict_start, const int* __restrict__ dict_len,
                                                       int* __restrict__ retry, int* __restrict__ retry_count)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        const int row = rows ? rows[i] : (int)i;
        const int s = slot_of_row[row];
        if (s < 0) continue;
        const int off = offsets[row], len = offsets[row + 1] - off;
        if (len <= 7 && attempt[row] == 0) continue;                 // the key is the string
        const StrSlot slot = table[s];
        bool same;
        if (slot.id >= 0) same = dict_len[slot.id] == len && sd_bytes_equal(bytes + off, dict_bytes + dict_start[slot.id], len);
        else {
            const int o2 = offsets[slot.first_row], l2 = offsets[slot.first_row + 1] - o2;
            same = l2 == len && sd_bytes_equal(bytes + off, bytes + o2, len);
        }
        if (!same) {
            attempt[row] = (uint8_t)(attempt[row] + 1);
            retry[atomicAdd(retry_count, 1)] = row;
        }
    }
}

// counters: [0] new strings, [1..2] their total bytes (64-bit)
__global__ void __launch_bounds__(256) sd_count_new_kernel(const int32_t* __restrict__ offsets, int64_t n, const StrSlot* __restrict__ table,
                                                          const int* __restrict__ slot_of_row, int* __restrict__ new_count, unsigned long long* __restrict__ new_bytes)
{
    int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; row < n; row += stride) {
        const int s = slot_of_row[row];
        if (s < 0) continue;
        if (table[s].id < 0 && table[s].first_row == (int)row) {
            atomicAdd(new_count, 1);
            atomicAdd(new_bytes, (unsigned long long)(offsets[row + 1] - offsets[row]));
        }
    }
}

// the owner row of every new slot appends its string to the store and publishes the id
__global__ void __launch_bounds__(256) sd_assign_kernel(const int32_t* __restrict__ offsets, const uint8_t* __restrict__ bytes, int64_t n, StrSlot* __restrict__ table,
                                                       const int* __restrict__ slot_of_row, int first_id, long long first_byte, int* __restrict__ next_id,
                                                       unsigned long long* __restrict__ next_byte, uint8_t* __restrict__ dict_bytes, long long* __restrict__ dict_start,
                                                       int* __restrict__ dict_len, unsigned long long* __restrict__ dict_key, int32_t* __restrict__ direct)
{
    int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; row < n; row += stride) {
        const int s = slot_of_row[row];
        if (s < 0) continue;
        if (table[s].id >= 0 || table[s].first_row != (int)row) continue;
        const int off = offsets[row], len = offsets[row + 1] - off;
        const int id = first_id + atomicAdd(next_id, 1);
        const long long at = first_byte + (long long)atomicAdd(next_byte, (unsigned long long)len);
        for (int i = 0; i < len; i++) dict_bytes[at + i] = bytes[off + i];
        dict_start[id] = at;
        dict_len[id] = len;
        dict_key[id] = table[s].key;
        table[s].id = id;
        if (len <= 1) direct[len == 1 ? (int)bytes[off] : 256] = id;
    }
}

__global__ void sd_ids_kernel(int64_t n, const StrSlot* __restrict__ table, const int* __restrict__ slot_of_row, int32_t* __restrict__ ids)
{
    int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; row < n; row += stride) {
        const int s = slot_of_row[row];
        ids[row] = s >= 0 ? table[s].id : 0;
    }
}

// new slots of a page that has to be re-run (table growth) must not survive as provisional entries
__global__ void sd_rehash_kernel(const unsigned long long* __restrict__ dict_key, int count, StrSlot* __restrict__ table, unsigned long long mask)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    int stride = gridDim.x * blockDim.x;
    for (; i < count; i += stride) {
        unsigned long long key = dict_key[i];
        unsigned long long pos = murmur3_mix(key) & mask;
        while (atomicCAS(&table[pos].key, SD_EMPTY, key) != SD_EMPTY) pos = (pos + 1) & mask;   // (equal keys of two colliding strings take two slots)
        table[pos].id = i;
    }
}

__global__ void sd_lens_kernel(const int32_t* __restrict__ ids, const uint8_t* __restrict__ is_null, int64_t n, const int* __restrict__ dict_len, int32_t* __restrict__ out)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) out[i] = (is_null && is_null[i]) ? 0 : dict_len[ids[i]];
    if (blockIdx.x == 0 && threadIdx.x == 0) out[n] = 0;
}

__global__ void sd_copy_out_kernel(const int32_t* __restrict__ ids, const uint8_t* __restrict__ is_null, int64_t n, const uint8_t* __restrict__ dict_bytes,
                                   const long long* __restrict__ dict_start, const int32_t* __restrict__ out_offsets, uint8_t* __restrict__ out_bytes)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        if (is_null && is_null[i]) continue;
        const int len = out_offsets[i + 1] - out_offsets[i];
        const uint8_t* src = dict_bytes + dict_start[ids[i]];
        uint8_t* dst = out_bytes + out_offsets[i];
        for (int k = 0; k < len; k++) dst[k] = src[k];
    }
}

struct StringDict {
    tgpu_ctx* ctx = nullptr;
    DevBuf table;
    int64_t cap = 0;
    DevBuf bytes, start, len, key;           // the store: bytes, and per id: first byte, length, table key (for rehashing)
    DevBuf direct;                           // int32[257]: id of every string of length <= 1 (byte value / 256 = empty), -1 = not in the dictionary
    int64_t bytes_cap = 0, bytes_used = 0, ids_cap = 0, count = 0;
    bool has_direct = false;                 // some string of length <= 1 was ever inserted (the direct map can answer something)

    explicit StringDict(tgpu_ctx* c) : ctx(c) {}
    int64_t memory_bytes() const { return (int64_t)(table.bytes + bytes.bytes + start.bytes + len.bytes + key.bytes); }

    int alloc_table(int64_t slots)
    {
        if (!direct.p) {
            TG_TRY(direct.alloc(ctx, 257 * 4));
            TG_CUDA(ctx, cudaMemsetAsync(direct.p, 0xFF, 257 * 4, ctx->stream));
        }
        DevBuf t;
        TG_TRY(t.alloc(ctx, (size_t)slots * sizeof(StrSlot)));
        TG_LAUNCH(ctx, sd_init_kernel, tg_grid(ctx, slots, 1024, 8), 256, 0, t.as<StrSlot>(), slots);
        if (count > 0) TG_LAUNCH(ctx, sd_rehash_kernel, tg_grid(ctx, count, 256, 8), 256, 0, key.as<unsigned long long>(), (int)count, t.as<StrSlot>(), (unsigned long long)slots - 1);
        table = std::move(t);
        cap = slots;
        return TGPU_OK;
    }

    template <typename T>
    int grow(DevBuf* buf, int64_t old_elems, int64_t new_elems)
    {
        DevBuf nb;
        TG_TRY(nb.alloc(ctx, (size_t)new_elems * sizeof(T)));
        if (old_elems > 0) TG_CUDA(ctx, cudaMemcpyAsync(nb.p, buf->p, (size_t)old_elems * sizeof(T), cudaMemcpyDeviceToDevice, ctx->stream));
        *buf = std::move(nb);
        return TGPU_OK;
    }

    // UTF8 column -> INT32 id column (NULL rows keep their validity; their id is 0).  Pages are taken in chunks: the first chunk goes
    // through the insert path (it meets the new strings), the rest through the one-pass lookup kernel; only chunks that met an
    // unknown string are re-run through the insert path.
    int encode(const DevColumn& col, DevColumn* out)
    {
        const int64_t n = col.length;
        if (n > (int64_t)INT32_MAX) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "page has more than 2^31-1 positions");
        DevColumn ids;
        ids.type = TGPU_INT32;
        ids.length = n;
        ids.own_data = std::make_shared<DevBuf>();
        TG_TRY(ids.own_data->alloc(ctx, (size_t)std::max<int64_t>(n, 1) * 4));
        ids.data = ids.own_data->p;
        ids.own_validity = col.own_validity;
        ids.validity = col.validity;
        if (n == 0) { *out = std::move(ids); return TGPU_OK; }
        constexpr int64_t CHUNK = 4 << 20;
        int32_t* d_ids = (int32_t*)ids.own_data->p;
        const int64_t head = count == 0 ? std::min<int64_t>(n, CHUNK) : 0;      // an empty dictionary learns from the first chunk
        if (head > 0) TG_TRY(encode_rows(col, 0, head, d_ids));
        if (head < n) {
            const int64_t rest = n - head, chunks = tg_div_up(rest, CHUNK);
            DevBuf miss;
            TG_TRY(miss.alloc(ctx, (size_t)chunks * 4));
            TG_CUDA(ctx, cudaMemsetAsync(miss.p, 0, (size_t)chunks * 4, ctx->stream));
            if (cap == 0) TG_TRY(alloc_table(1 << 12));
            std::vector<int> h_miss((size_t)chunks);
            // tier 1: the direct map of strings of length <= 1 (tried when the dictionary holds such strings at all)
            bool tier1 = has_direct;
            if (tier1) {
                TG_LAUNCH(ctx, sd_lookup_direct_kernel, tg_grid(ctx, rest, 1024, 8), 256, 0, col.offsets, (const uint8_t*)col.data, col.validity, head, rest,
                          direct.as<int32_t>(), d_ids, CHUNK, miss.as<int>());
                TG_CUDA(ctx, cudaMemcpyAsync(h_miss.data(), miss.p, (size_t)chunks * 4, cudaMemcpyDeviceToHost, ctx->stream));
                TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
            }
            // tier 2: the table lookup, for the chunks tier 1 could not finish (all of them without tier 1); tier 3: the insert path
            for (int64_t c = 0; c < chunks; c++) {
                if (tier1 && !h_miss[c]) continue;
                const int64_t lo = head + c * CHUNK, cnt = std::min<int64_t>(CHUNK, n - lo);
                TG_CUDA(ctx, cudaMemsetAsync(miss.as<int>() + c, 0, 4, ctx->stream));
                TG_LAUNCH(ctx, sd_lookup_kernel, tg_grid(ctx, cnt, 1024, 6), 256, 0, col.offsets, (const uint8_t*)col.data, col.validity, lo, cnt, table.as<StrSlot>(),
                          (unsigned long long)cap - 1, bytes.as<uint8_t>(), start.as<long long>(), len.as<int>(), d_ids, CHUNK, miss.as<int>() + c);
            }
            TG_CUDA(ctx, cudaMemcpyAsync(h_miss.data(), miss.p, (size_t)chunks * 4, cudaMemcpyDeviceToHost, ctx->stream));
            TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
            for (int64_t c = 0; c < chunks; c++)
                if (h_miss[c]) TG_TRY(encode_rows(col, head + c * CHUNK, std::min<int64_t>(CHUNK, n - (head + c * CHUNK)), d_ids));
        }
        *out = std::move(ids);
        return TGPU_OK;
    }

    // insert path over rows [first, first + n) of the column: find-or-claim, verify, append the new strings, write the ids
    int encode_rows(const DevColumn& whole, int64_t first, int64_t n, int32_t* d_ids_whole)
    {
        DevColumn col = whole;
        col.offsets = whole.offsets + first;                     // row r of the slice is row first + r: offsets keep pointing into `data`
        col.length = n;
        const uint8_t* slice_validity = nullptr;
        DevBuf shifted_validity;
        if (whole.validity) {
            if ((first & 7) == 0) slice_validity = whole.validity + (first >> 3);
            else return tg_fail(ctx, TGPU_ERR_ILLEGAL_STATE, "string dictionary chunk is not byte aligned");
        }
        col.validity = slice_validity;
        int32_t* d_ids = d_ids_whole + first;
        if (cap == 0) TG_TRY(alloc_table(1 << 12));
        DevBuf slot_of_row, attempt, retry_a, retry_b;
        TG_TRY(slot_of_row.alloc(ctx, (size_t)n * 4));
        TG_TRY(attempt.alloc(ctx, (size_t)n));
        int* d_cnt = ctx->d_scratch->strdict_counts;
        const int32_t* offs = col.offsets;
        const uint8_t* data = (const uint8_t*)col.data;
        const int grid = tg_grid(ctx, n, 256, 8);
        int32_t h[4];
        while (true) {          // (re-run after a table growth)
            TG_CUDA(ctx, cudaMemsetAsync(attempt.p, 0, (size_t)n, ctx->stream));
            const int* rows = nullptr;
            int64_t todo = n;
            bool overflow = false;
            for (int round = 0; ; round++) {
                if (round >= SD_MAX_ATTEMPTS) return tg_fail(ctx, TGPU_ERR_INSUFFICIENT_RESOURCES, "string keys collide under %d independent 64-bit hashes", SD_MAX_ATTEMPTS);
                TG_CUDA(ctx, cudaMemsetAsync(d_cnt, 0, 16, ctx->stream));
                const int64_t budget = cap / 2 - count;
                TG_LAUNCH(ctx, sd_insert_kernel, tg_grid(ctx, todo, 256, 8), 256, 0, offs, data, col.validity, rows, todo, attempt.as<uint8_t>(), table.as<StrSlot>(),
                          (unsigned long long)cap - 1, slot_of_row.as<int>(), d_cnt, (int)std::min<int64_t>(std::max<int64_t>(budget, 0), INT32_MAX));
                TG_TRY(tg_read(ctx, d_cnt, 8, h));
                if (h[1]) { overflow = true; break; }
                DevBuf& retry = (round & 1) ? retry_b : retry_a;
                TG_TRY(retry.alloc(ctx, (size_t)todo * 4));
                TG_CUDA(ctx, cudaMemsetAsync(d_cnt, 0, 4, ctx->stream));
                TG_LAUNCH(ctx, sd_verify_kernel, tg_grid(ctx, todo, 256, 8), 256, 0, offs, data, rows, todo, attempt.as<uint8_t>(), table.as<StrSlot>(), slot_of_row.as<int>(),
                          bytes.as<uint8_t>(), start.as<long long>(), len.as<int>(), retry.as<int>(), d_cnt);
                TG_TRY(tg_read(ctx, d_cnt, 4, h));
                if (h[0] == 0) break;
                rows = retry.as<int>();
                todo = h[0];
            }
            if (!overflow) break;
            int64_t slots = cap * 4;
            if (slots > (1LL << 31)) return tg_fail(ctx, TGPU_ERR_INSUFFICIENT_RESOURCES, "string dictionary exceeds %lld entries", (long long)SD_MAX_IDS);
            TG_TRY(alloc_table(slots));     // rebuilt from the assigned ids: the provisional slots of the aborted pass are gone
        }
        // new strings: count, make room, append
        TG_CUDA(ctx, cudaMemsetAsync(d_cnt, 0, 16, ctx->stream));
        TG_LAUNCH(ctx, sd_count_new_kernel, grid, 256, 0, offs, n, table.as<StrSlot>(), slot_of_row.as<int>(), d_cnt, (unsigned long long*)(d_cnt + 2));
        TG_TRY(tg_read(ctx, d_cnt, 16, h));
        const int64_t fresh = h[0];
        long long fresh_bytes = 0;
        memcpy(&fresh_bytes, h + 2, 8);
        if (fresh > 0) {
            if (count + fresh > SD_MAX_IDS) return tg_fail(ctx, TGPU_ERR_INSUFFICIENT_RESOURCES, "more than %lld distinct strings in one group-by key", (long long)SD_MAX_IDS);
            if (count + fresh > ids_cap) {
                int64_t ncap = std::max<int64_t>(1024, ids_cap);
                while (ncap < count + fresh) ncap *= 2;
                TG_TRY(grow<long long>(&start, count, ncap));
                TG_TRY(grow<int>(&len, count, ncap));
                TG_TRY(grow<unsigned long long>(&key, count, ncap));
                ids_cap = ncap;
            }
            if (bytes_used + fresh_bytes > bytes_cap) {
                int64_t ncap = std::max<int64_t>(1 << 16, bytes_cap);
                while (ncap < bytes_used + fresh_bytes) ncap *= 2;
                TG_TRY(grow<uint8_t>(&bytes, bytes_used, ncap));
                bytes_cap = ncap;
            }
            TG_CUDA(ctx, cudaMemsetAsync(d_cnt, 0, 16, ctx->stream));
            TG_LAUNCH(ctx, sd_assign_kernel, grid, 256, 0, offs, data, n, table.as<StrSlot>(), slot_of_row.as<int>(), (int)count, (long long)bytes_used, d_cnt,
                      (unsigned long long*)(d_cnt + 2), bytes.as<uint8_t>(), start.as<long long>(), len.as<int>(), key.as<unsigned long long>(), direct.as<int32_t>());
            count += fresh;
            if (!has_direct) {      // did a string of length <= 1 arrive?  (tier 1 of encode() is only worth a pass then)
                std::vector<int32_t> h_direct(257);
                TG_CUDA(ctx, cudaMemcpyAsync(h_direct.data(), direct.p, 257 * 4, cudaMemcpyDeviceToHost, ctx->stream));
                TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
                for (int32_t v : h_direct) has_direct = has_direct || v >= 0;
            }
            bytes_used += fresh_bytes;
        }
        TG_LAUNCH(ctx, sd_ids_kernel, grid, 256, 0, n, table.as<StrSlot>(), slot_of_row.as<int>(), d_ids);
        return TGPU_OK;
    }

    // ids (+ one NULL byte per row, may be nullptr) -> UTF8 column
    int decode(const int32_t* d_ids, const uint8_t* d_is_null, int64_t n, DevColumn* out)
    {
        DevColumn c;
        c.type = TGPU_UTF8;
        c.length = n;
        c.own_offsets = std::make_shared<DevBuf>();
        TG_TRY(c.own_offsets->alloc(ctx, (size_t)(n + 1) * 4));
        DevBuf lens;
        TG_TRY(lens.alloc(ctx, (size_t)(n + 1) * 4));
        TG_LAUNCH(ctx, sd_lens_kernel, tg_grid(ctx, n, 1024, 8), 256, 0, d_ids, d_is_null, n, len.as<int>(), lens.as<int32_t>());
        TG_TRY(tg_exclusive_sum(ctx, lens.as<int32_t>(), c.own_offsets->as<int32_t>(), (int)(n + 1)));
        int32_t total = 0;
        TG_TRY(tg_read(ctx, c.own_offsets->as<int32_t>() + n, 4, &total));
        if (total < 0) return tg_fail(ctx, TGPU_ERR_INSUFFICIENT_RESOURCES, "variable-width key column of one output page exceeds 2 GB");
        c.own_data = std::make_shared<DevBuf>();
        TG_TRY(c.own_data->alloc(ctx, (size_t)std::max<int32_t>(total, 1)));
        c.data = c.own_data->p;
        c.offsets = c.own_offsets->as<int32_t>();
        c.data_bytes = total;
        if (total > 0)
            TG_LAUNCH(ctx, sd_copy_out_kernel, tg_grid(ctx, n, 256, 8), 256, 0, d_ids, d_is_null, n, bytes.as<uint8_t>(), start.as<long long>(), c.offsets, (uint8_t*)c.own_data->p);
        *out = std::move(c);
        return TGPU_OK;
    }
};

}  // namespace tg
