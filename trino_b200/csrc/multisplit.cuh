// multisplit.cuh — stable multi-split (histogram -> offsets -> scatter) of fixed-width columns into <= 64 partitions.
// Shared by the PagePartitioner / exchange (partition.cu) and the sliced general group-by (groupby.cu).  Everything here has
// internal linkage (anonymous namespace): each translation unit gets its own copy.
#pragma once
#include "rowkeys.cuh"

namespace {

using namespace tg;

// ------------------------------------------------------------------------------------------------
// exchange: stable multi-split (histogram -> offsets -> scatter), all columns in one pass
// ------------------------------------------------------------------------------------------------
constexpr int XT = 256;          // threads per CTA
constexpr int XMAXP = 64;        // partitions the fused exchange path handles (one per GPU)
constexpr int XMAXC = 48;        // value columns + null-byte columns (lanes) of one multi-split
constexpr int XCHG_ROW_NUMBER = 16;   // XchgCols.elem code of a lane without source: the scatter writes each row's input position (int32; CTA kernel only)

// pass A: partition id per row (uint8) and a histogram per CTA chunk
__global__ void __launch_bounds__(XT) xchg_hist_kernel(KeyCols keys, int64_t n, int64_t chunk, int32_t bucket_count, const int32_t* __restrict__ bucket_to_partition,
                                                       int32_t P, uint8_t* __restrict__ pid_out, unsigned int* __restrict__ hist /* [grid][P] */)
{
    __shared__ unsigned int sh[XMAXP];
    for (int i = threadIdx.x; i < P; i += XT) sh[i] = 0;
    __syncthreads();
    int64_t begin = (int64_t)blockIdx.x * chunk, end = min(n, begin + chunk);
    if (P <= 8) {
        // few partitions (one per GPU of a box): private register counters, no per-row atomics or warp votes;
        // U independent rows in flight per thread, loads issued together on the single-BIGINT-key fast path
        constexpr int U = 8;
        const bool fast = keys.count == 1 && !keys.is_utf8[0] && !keys.is_double[0] && keys.cols[0].elem == 8 && !keys.cols[0].validity;
        const long long* __restrict__ key0 = (const long long*)keys.cols[0].data;
        unsigned int cnt[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        for (int64_t base = begin; base < end; base += U * XT) {
            int pidv[U];
            if (fast && base + U * XT <= end) {
                long long v[U];
#pragma unroll
                for (int u = 0; u < U; u++) v[u] = key0[base + u * XT + threadIdx.x];
#pragma unroll
                for (int u = 0; u < U; u++) {
                    int32_t bucket = process_raw_hash(hash_long(v[u]), bucket_count);
                    pidv[u] = bucket_to_partition ? bucket_to_partition[bucket] : bucket;
                }
            }
            else {
#pragma unroll
                for (int u = 0; u < U; u++) {
                    int64_t row = base + u * XT + threadIdx.x;
                    pidv[u] = -1;
                    if (row < end) {
                        uint64_t h = 0;
                        for (int c = 0; c < keys.count; c++) h = combine_hash(h, type_hash(keys, c, row));
                        int32_t bucket = process_raw_hash(h, bucket_count);
                        pidv[u] = bucket_to_partition ? bucket_to_partition[bucket] : bucket;
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < U; u++) {
                int64_t row = base + u * XT + threadIdx.x;
                if (row < end) pid_out[row] = (uint8_t)pidv[u];
#pragma unroll
                for (int q = 0; q < 8; q++) cnt[q] += (pidv[u] == q);
            }
        }
#pragma unroll
        for (int q = 0; q < 8; q++) {
            unsigned int v = cnt[q];
            for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
            if ((threadIdx.x & 31) == 0 && v && q < P) atomicAdd(&sh[q], v);
        }
    }
    else {
        for (int64_t row = begin + threadIdx.x; row < end; row += XT) {
            uint64_t h = 0;
            for (int c = 0; c < keys.count; c++) h = combine_hash(h, type_hash(keys, c, row));
            int32_t bucket = process_raw_hash(h, bucket_count);
            int32_t pid = bucket_to_partition ? bucket_to_partition[bucket] : bucket;
            pid_out[row] = (uint8_t)pid;
            // warp-aggregated histogram update
            unsigned int peers = __match_any_sync(__activemask(), pid);
            if ((int)(__ffs(peers) - 1) == (int)(threadIdx.x & 31)) atomicAdd(&sh[pid], __popc(peers));
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < P; i += XT) hist[(size_t)blockIdx.x * P + i] = sh[i];
}

// pass B: where every CTA chunk starts inside every partition, and the partition totals.  One CTA per partition.
__global__ void __launch_bounds__(256) xchg_offsets_kernel(const unsigned int* __restrict__ hist, int grid, int32_t P, long long* __restrict__ block_off /* [grid][P] */,
                                                           long long* __restrict__ totals /* [P] */)
{
    __shared__ long long part[256];
    const int p = blockIdx.x, t = threadIdx.x;
    const int per = (grid + 255) / 256;
    const int b0 = min(grid, t * per), b1 = min(grid, b0 + per);
    long long sum = 0;
    for (int b = b0; b < b1; b++) sum += hist[(size_t)b * P + p];
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
        block_off[(size_t)b * P + p] = run;
        run += hist[(size_t)b * P + p];
    }
    if (t == 255) totals[p] = part[255];
}

struct XchgCols {
    int32_t count;
    int32_t elem[XMAXC];          // element bytes; 0 = "null byte" pseudo column (reads the validity bitmap, writes 1 = NULL)
    const void* src[XMAXC];       // column data, or the validity bitmap for pseudo columns
    char* const* dst;             // device array [count][P] of destination base pointers (local send buffer or peer memory)
};

// pass C: stable scatter, staged through shared memory.  A CTA walks its chunk in tiles of XTILE rows.  Per tile it ranks
// every row inside its partition (warp __match_any_sync rank + scan over the tile's (iteration, warp) cells), lays the tile
// out partition-contiguously in shared memory one column at a time, and copies each partition's run to its destination with
// consecutive threads writing consecutive addresses: the stores that cross NVLink (peer arenas) are >= 128-byte contiguous
// segments instead of one 8-byte store per row.  Rows keep their order inside a partition.
constexpr int XR = 8;                 // rows per thread per tile
constexpr int XTILE = XT * XR;        // 2048 rows
constexpr int XCELLS = XR * (XT / 32);
static_assert(XCELLS == 64, "the cell scan assumes two cells per lane");

template <int OCC>
__global__ void __launch_bounds__(XT, OCC) xchg_scatter_kernel(const uint8_t* __restrict__ pids, int64_t n, int64_t chunk, int32_t P,
                                                               const long long* __restrict__ block_off, XchgCols cols)
{
    __shared__ long long stage[XTILE];
    __shared__ uint8_t spid[XTILE];
    __shared__ __align__(16) unsigned short wcount[XCELLS][XMAXP];
    __shared__ long long running[XMAXP];
    __shared__ int tile_cnt[XMAXP];
    __shared__ int tile_off[XMAXP];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    constexpr int NW = XT / 32;
    for (int i = threadIdx.x; i < P; i += XT) running[i] = block_off[(size_t)blockIdx.x * P + i];
    const int64_t begin = (int64_t)blockIdx.x * chunk, end = min(n, begin + chunk);
    for (int64_t tile = begin; tile < end; tile += XTILE) {
        const int tile_rows = (int)min((int64_t)XTILE, end - tile);
        for (int i = threadIdx.x; i < XCELLS * XMAXP * 2 / 16; i += XT) ((uint4*)&wcount[0][0])[i] = make_uint4(0, 0, 0, 0);
        __syncthreads();
        int pid[XR];
        int pos[XR];
#pragma unroll
        for (int i = 0; i < XR; i++) {
            int64_t row = tile + (int64_t)i * XT + threadIdx.x;
            bool live = row < end;
            pid[i] = live ? (int)pids[row] : -1;
            unsigned int peers = __match_any_sync(0xffffffffu, live ? pid[i] : -1 - lane);
            pos[i] = __popc(peers & ((1u << lane) - 1));
            if (live && pos[i] == 0) wcount[i * NW + warp][pid[i]] = (unsigned short)__popc(peers);
        }
        __syncthreads();
        // exclusive scan over the 64 cells of every partition (cells are in row order: iteration-major, then warp)
        for (int p = warp; p < P; p += NW) {
            unsigned int a = wcount[2 * lane][p], b = wcount[2 * lane + 1][p];
            unsigned int incl = a + b;
            for (int off = 1; off < 32; off <<= 1) {
                unsigned int v = __shfl_up_sync(0xffffffffu, incl, off);
                if (lane >= off) incl += v;
            }
            unsigned int excl = incl - (a + b);
            wcount[2 * lane][p] = (unsigned short)excl;
            wcount[2 * lane + 1][p] = (unsigned short)(excl + a);
            if (lane == 31) tile_cnt[p] = (int)incl;
        }
        __syncthreads();
        if (warp == 0) {
            int c0 = 2 * lane < P ? tile_cnt[2 * lane] : 0, c1 = 2 * lane + 1 < P ? tile_cnt[2 * lane + 1] : 0;
            int incl = c0 + c1;
            for (int off = 1; off < 32; off <<= 1) {
                int v = __shfl_up_sync(0xffffffffu, incl, off);
                if (lane >= off) incl += v;
            }
            int excl = incl - (c0 + c1);
            if (2 * lane < P) tile_off[2 * lane] = excl;
            if (2 * lane + 1 < P) tile_off[2 * lane + 1] = excl + c0;
        }
        __syncthreads();
#pragma unroll
        for (int i = 0; i < XR; i++) {
            if (pid[i] < 0) continue;
            pos[i] += tile_off[pid[i]] + wcount[i * NW + warp][pid[i]];
            spid[pos[i]] = (uint8_t)pid[i];
        }
        for (int c = 0; c < cols.count; c++) {
            const int elem = cols.elem[c];
            const void* src = cols.src[c];
#pragma unroll
            for (int i = 0; i < XR; i++) {
                if (pid[i] < 0) continue;
                int64_t row = tile + (int64_t)i * XT + threadIdx.x;
                switch (elem) {
                    case 16: ((int*)stage)[pos[i]] = (int)row; break;          // XCHG_ROW_NUMBER lane: the row's position in the input
                    case 8: stage[pos[i]] = ((const long long*)src)[row]; break;
                    case 4: ((int*)stage)[pos[i]] = ((const int*)src)[row]; break;
                    case 2: ((short*)stage)[pos[i]] = ((const short*)src)[row]; break;
                    case 1: ((char*)stage)[pos[i]] = ((const char*)src)[row]; break;
                    default: ((char*)stage)[pos[i]] = tg_valid((const uint8_t*)src, row) ? 0 : 1; break;
                }
            }
            __syncthreads();
            for (int j = threadIdx.x; j < tile_rows; j += XT) {
                int q = spid[j];
                long long d = running[q] + (j - tile_off[q]);
                char* base = cols.dst[(size_t)c * P + q];
                switch (elem) {
                    case 8: ((long long*)base)[d] = stage[j]; break;
                    case 16:
                    case 4: ((int*)base)[d] = ((const int*)stage)[j]; break;
                    case 2: ((short*)base)[d] = ((const short*)stage)[j]; break;
                    default: base[d] = ((const char*)stage)[j]; break;
                }
            }
            __syncthreads();
        }
        if (threadIdx.x < P) running[threadIdx.x] += tile_cnt[threadIdx.x];
    }
}

// ---- CTA tiles, ANY ORDER inside a partition --------------------------------------------------------------------------------
// For callers that do not need the rows of a partition in input order (the sliced group-by: first-seen order travels in the
// row-number lane).  Ranks come from one shared-memory counter per partition (warp-aggregated atomicAdd: one atomic per distinct
// partition per warp), so there is no cell matrix to clear and scan; up to XU_G lanes are staged and copied out together, which
// leaves 3 + 2 * ceil(lanes / XU_G) barriers per 2048-row tile and puts XU_G * 8 independent loads in flight per thread.
constexpr int XU_G = 3;
constexpr int XU_DST = 8;              // lanes whose destination pointers are cached in shared memory
constexpr size_t XU_SMEM = (size_t)XU_G * XTILE * 8;

__device__ __forceinline__ long long xchg_load_lane(int elem, const void* src, int64_t row)
{
    switch (elem) {
        case 16: return (long long)row;                                           // XCHG_ROW_NUMBER
        case 8: return ((const long long*)src)[row];
        case 4: return ((const int*)src)[row];
        case 2: return ((const short*)src)[row];
        case 1: return ((const signed char*)src)[row];
        default: return tg_valid((const uint8_t*)src, row) ? 0 : 1;              // NULL-byte pseudo lane
    }
}

__global__ void __launch_bounds__(XT, 4) xchg_scatter_unordered_kernel(const uint8_t* __restrict__ pids, int64_t n, int64_t chunk, int32_t P,
                                                                      const long long* __restrict__ block_off, XchgCols cols)
{
    extern __shared__ long long xu_stage[];          // [XU_G][XTILE]
    __shared__ uint8_t spid[XTILE];
    __shared__ int cnt[XMAXP];
    __shared__ int tile_off[XMAXP];
    __shared__ long long running[XMAXP];
    __shared__ char* sdst[XU_DST * XMAXP];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int i = threadIdx.x; i < P; i += XT) running[i] = block_off[(size_t)blockIdx.x * P + i];
    for (int i = threadIdx.x; i < min(cols.count, XU_DST) * P; i += XT) sdst[(i / P) * XMAXP + (i % P)] = cols.dst[i];
    const int64_t begin = (int64_t)blockIdx.x * chunk, end = min(n, begin + chunk);
    for (int64_t tile = begin; tile < end; tile += XTILE) {
        const int tile_rows = (int)min((int64_t)XTILE, end - tile);
        if (threadIdx.x < XMAXP) cnt[threadIdx.x] = 0;
        __syncthreads();
        int pid[XR], pos[XR];
#pragma unroll
        for (int i = 0; i < XR; i++) {
            int64_t row = tile + (int64_t)i * XT + threadIdx.x;
            pid[i] = row < end ? (int)pids[row] : -1;
        }
#pragma unroll
        for (int i = 0; i < XR; i++) {
            const bool live = pid[i] >= 0;
            unsigned int peers = __match_any_sync(0xffffffffu, live ? pid[i] : -1 - lane);
            const int leader = __ffs(peers) - 1;
            int base = 0;
            if (live && lane == leader) base = atomicAdd(&cnt[pid[i]], __popc(peers));
            base = __shfl_sync(0xffffffffu, base, leader);
            pos[i] = base + __popc(peers & ((1u << lane) - 1));
        }
        __syncthreads();
        if (warp == 0) {
            int c0 = cnt[2 * lane], c1 = cnt[2 * lane + 1];
            int incl = c0 + c1;
            for (int off = 1; off < 32; off <<= 1) {
                int v = __shfl_up_sync(0xffffffffu, incl, off);
                if (lane >= off) incl += v;
            }
            int excl = incl - (c0 + c1);
            tile_off[2 * lane] = excl;
            tile_off[2 * lane + 1] = excl + c0;
        }
        __syncthreads();
#pragma unroll
        for (int i = 0; i < XR; i++) {
            if (pid[i] < 0) continue;
            pos[i] += tile_off[pid[i]];
            spid[pos[i]] = (uint8_t)pid[i];
        }
        for (int c0 = 0; c0 < cols.count; c0 += XU_G) {
            const int g_count = min(XU_G, cols.count - c0);
            for (int g = 0; g < g_count; g++) {
                const int elem = cols.elem[c0 + g];
                const void* src = cols.src[c0 + g];
                long long v[XR];
#pragma unroll
                for (int i = 0; i < XR; i++) v[i] = pid[i] >= 0 ? xchg_load_lane(elem, src, tile + (int64_t)i * XT + threadIdx.x) : 0;
#pragma unroll
                for (int i = 0; i < XR; i++)
                    if (pid[i] >= 0) xu_stage[g * XTILE + pos[i]] = v[i];
            }
            __syncthreads();
            for (int g = 0; g < g_count; g++) {
                const int c = c0 + g;
                const int elem = cols.elem[c];
                const long long* st = xu_stage + g * XTILE;
                for (int j = threadIdx.x; j < tile_rows; j += XT) {
                    const int q = spid[j];
                    const long long d = running[q] + (j - tile_off[q]);
                    char* base = c < XU_DST ? sdst[c * XMAXP + q] : cols.dst[(size_t)c * P + q];
                    switch (elem) {
                        case 8: ((long long*)base)[d] = st[j]; break;
                        case 16:
                        case 4: ((int*)base)[d] = (int)st[j]; break;
                        case 2: ((short*)base)[d] = (short)st[j]; break;
                        default: base[d] = (char)st[j]; break;
                    }
                }
            }
            __syncthreads();
        }
        if (threadIdx.x < P) running[threadIdx.x] += cnt[threadIdx.x];
        // (the barrier at the top of the next tile orders this update and the counter reset against their readers)
    }
}

// ---- warp-granular variant for <= 8 partitions (one per GPU of a box) ------------------------------------------------------
// Every warp owns a contiguous chunk of rows and walks it in tiles of 256 rows (8 consecutive rows per lane), with no CTA
// barrier anywhere: warps drift apart, so the load latency of one warp hides behind the staging / copy-out of the others.
// Ranks come from packed per-lane counters and one warp scan (no __match_any_sync, no shared-memory counters).
constexpr int WR = 8;                  // consecutive rows per lane
constexpr int WTILE = 32 * WR;         // rows per warp tile
constexpr int WWARPS = 8;              // warps per CTA

// FAST: one BIGINT key channel without NULLs (the join-key shape) - the loads of a group of rows are issued together
template <bool FAST>
__global__ void __launch_bounds__(32 * WWARPS) xchg_hist_warp_kernel(KeyCols keys, int64_t n, int64_t wchunk, int32_t bucket_count,
                                                                     const int32_t* __restrict__ bucket_to_partition, int32_t P, uint8_t* __restrict__ pid_out,
                                                                     unsigned int* __restrict__ hist /* [chunks][P] */)
{
    constexpr int U = 8;
    const int lane = threadIdx.x & 31;
    const int64_t vchunk = (int64_t)blockIdx.x * WWARPS + (threadIdx.x >> 5);
    const int64_t begin = vchunk * wchunk, end = min(n, begin + wchunk);
    if (begin >= n) return;
    unsigned int cnt[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    unsigned long long packed = 0;
    int since_flush = 0;
    const long long* __restrict__ key0 = (const long long*)keys.cols[0].data;
    for (int64_t base = begin; base < end; base += U * 32) {
        int pidv[U];
        const bool full = base + U * 32 <= end;
        if (FAST && full) {
            long long v[U];
#pragma unroll
            for (int u = 0; u < U; u++) v[u] = key0[base + u * 32 + lane];
#pragma unroll
            for (int u = 0; u < U; u++) {
                int32_t bucket = process_raw_hash(hash_long(v[u]), bucket_count);
                pidv[u] = bucket_to_partition ? bucket_to_partition[bucket] : bucket;
            }
        }
        else {
#pragma unroll
            for (int u = 0; u < U; u++) {
                int64_t row = base + u * 32 + lane;
                pidv[u] = -1;
                if (row < end) {
                    uint64_t h = 0;
                    for (int c = 0; c < keys.count; c++) h = combine_hash(h, type_hash(keys, c, row));
                    int32_t bucket = process_raw_hash(h, bucket_count);
                    pidv[u] = bucket_to_partition ? bucket_to_partition[bucket] : bucket;
                }
            }
        }
        // one-hot byte counters: one add per row instead of eight compares; spilled into the 32-bit counters before a byte can wrap
#pragma unroll
        for (int u = 0; u < U; u++) {
            int64_t row = base + u * 32 + lane;
            if (pid_out && row < end) pid_out[row] = (uint8_t)pidv[u];     // pid_out == nullptr: the scatter recomputes the ids from the key
            if (pidv[u] >= 0) packed += 1ull << (8 * pidv[u]);
        }
        if (++since_flush == 31) {                                          // 31 trips x 8 rows = 248 < 256
#pragma unroll
            for (int q = 0; q < 8; q++) cnt[q] += (unsigned int)(packed >> (8 * q)) & 0xffu;
            packed = 0;
            since_flush = 0;
        }
    }
#pragma unroll
    for (int q = 0; q < 8; q++) cnt[q] += (unsigned int)(packed >> (8 * q)) & 0xffu;
#pragma unroll
    for (int q = 0; q < 8; q++) {
        unsigned int v = cnt[q];
        for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
        if (lane == 0 && q < P) hist[(size_t)vchunk * P + q] = v;
    }
}

// four packed bytes -> four 16-bit fields
__device__ __forceinline__ unsigned long long spread4(unsigned int x)
{
    return (unsigned long long)(x & 0xffu) | ((unsigned long long)(x & 0xff00u) << 8) | ((unsigned long long)(x & 0xff0000u) << 16) |
           ((unsigned long long)(x & 0xff000000u) << 24);
}
__device__ __forceinline__ unsigned int field16(unsigned long long lo, unsigned long long hi, int q)
{
    return (unsigned int)(((q & 4) ? hi : lo) >> ((q & 3) * 16)) & 0xffffu;
}

// (An aligned-window copy-out - every warp store one aligned segment of one partition run - was worth +15 % when the stores
// crossed NVLink and cost 50 % for local destinations; peer destinations no longer use this kernel, so it is gone.)
// KEYS: the partition ids are recomputed from the single BIGINT key column (`key0`, no NULLs) instead of being read from the 1-byte id
// array the histogram pass would otherwise have to write: 2 bytes per row less HBM traffic for one hash (two multiplies) per row
template <bool VEC, bool KEYS>
__global__ void __launch_bounds__(32 * WWARPS, 4) xchg_scatter_warp_kernel(const uint8_t* __restrict__ pids, int64_t n, int64_t wchunk, int32_t P,
                                                                        const long long* __restrict__ block_off, XchgCols cols,
                                                                        const long long* __restrict__ key0, int32_t bucket_count, const int32_t* __restrict__ b2p)
{
    __shared__ long long stage_all[WWARPS][WTILE];
    __shared__ long long run_all[WWARPS][8];
    __shared__ uint8_t spid_all[WWARPS][WTILE];
    __shared__ int toff_all[WWARPS][8];
    __shared__ char* sdst[XMAXC * 8];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int i = threadIdx.x; i < cols.count * P; i += blockDim.x) sdst[(i / P) * 8 + (i % P)] = cols.dst[i];
    __syncthreads();
    const int64_t vchunk = (int64_t)blockIdx.x * WWARPS + warp;
    const int64_t begin = vchunk * wchunk, end = min(n, begin + wchunk);
    if (begin >= n) return;
    long long* stage = stage_all[warp];
    long long* run = run_all[warp];
    uint8_t* spid = spid_all[warp];
    int* toff = toff_all[warp];
    if (lane < 8) run[lane] = lane < P ? block_off[(size_t)vchunk * P + lane] : 0;
    __syncwarp();
    auto load_pids = [&](int64_t tile) -> unsigned long long {
        int64_t row0 = tile + lane * WR;
        if (KEYS) {
            unsigned long long v = ~0ull;     // 0xff = no row
            if (row0 + WR <= end) {
                long long k[WR];
                if (VEC) {
                    const longlong2* s2 = (const longlong2*)(key0 + row0);
#pragma unroll
                    for (int j = 0; j < WR / 2; j++) { longlong2 t = s2[j]; k[2 * j] = t.x; k[2 * j + 1] = t.y; }
                }
                else {
#pragma unroll
                    for (int i = 0; i < WR; i++) k[i] = key0[row0 + i];
                }
                v = 0;
#pragma unroll
                for (int i = 0; i < WR; i++) {
                    int32_t bucket = process_raw_hash(hash_long(k[i]), bucket_count);
                    v |= (unsigned long long)(unsigned int)(b2p ? b2p[bucket] : bucket) << (8 * i);
                }
            }
            else {
                for (int i = 0; i < WR; i++)
                    if (row0 + i < end) {
                        int32_t bucket = process_raw_hash(hash_long(key0[row0 + i]), bucket_count);
                        v = (v & ~(0xffull << (8 * i))) | ((unsigned long long)(unsigned int)(b2p ? b2p[bucket] : bucket) << (8 * i));
                    }
            }
            return v;
        }
        if (row0 + WR <= end) return *(const unsigned long long*)(pids + row0);
        unsigned long long v = ~0ull;     // 0xff = no row
        for (int i = 0; i < WR; i++)
            if (row0 + i < end) v = (v & ~(0xffull << (8 * i))) | ((unsigned long long)pids[row0 + i] << (8 * i));
        return v;
    };
    unsigned long long next_pid8 = KEYS ? 0ull : load_pids(begin);
    for (int64_t tile = begin; tile < end; tile += WTILE) {
        // (the id-array form prefetches the next tile's ids; the key form would hold 16 more registers across the tile)
        const unsigned long long pid8 = KEYS ? load_pids(tile) : next_pid8;
        if (!KEYS && tile + WTILE < end) next_pid8 = load_pids(tile + WTILE);
        const int64_t row0 = tile + lane * WR;
        const int tile_rows = (int)min((int64_t)WTILE, end - tile);
        // per-lane counters (8-bit fields) and the rank of each of my rows among my earlier rows of the same partition
        unsigned long long c8 = 0, before8 = 0;
#pragma unroll
        for (int i = 0; i < WR; i++) {
            unsigned int q = (unsigned int)(pid8 >> (8 * i)) & 0xffu;
            if (q < 8) {
                before8 |= ((c8 >> (8 * q)) & 0xffull) << (8 * i);
                c8 += 1ull << (8 * q);
            }
        }
        unsigned long long lo = spread4((unsigned int)c8), hi = spread4((unsigned int)(c8 >> 32));
        unsigned long long ilo = lo, ihi = hi;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            unsigned long long a = __shfl_up_sync(0xffffffffu, ilo, off), b = __shfl_up_sync(0xffffffffu, ihi, off);
            if (lane >= off) { ilo += a; ihi += b; }
        }
        const unsigned long long tlo = __shfl_sync(0xffffffffu, ilo, 31), thi = __shfl_sync(0xffffffffu, ihi, 31);
        const unsigned long long elo = ilo - lo, ehi = ihi - hi;    // rows of lower lanes, per partition
        // start of every partition inside the tile
        unsigned long long olo = 0, ohi = 0;
        {
            unsigned int acc = 0;
#pragma unroll
            for (int q = 0; q < 8; q++) {
                if (q < 4) olo |= (unsigned long long)acc << (16 * q);
                else ohi |= (unsigned long long)acc << (16 * (q - 4));
                acc += field16(tlo, thi, q);
            }
        }
        if (lane < 8) toff[lane] = (int)field16(olo, ohi, lane);
        unsigned long long pos8 = 0;
#pragma unroll
        for (int i = 0; i < WR; i++) {
            unsigned int q = (unsigned int)(pid8 >> (8 * i)) & 0xffu;
            if (q < 8) {
                unsigned int pos = field16(olo, ohi, q) + field16(elo, ehi, q) + ((unsigned int)(before8 >> (8 * i)) & 0xffu);
                pos8 |= (unsigned long long)pos << (8 * i);
                spid[pos] = (uint8_t)q;
            }
        }
        for (int c = 0; c < cols.count; c++) {
            const int elem = cols.elem[c];
            const char* src = (const char*)cols.src[c];
            const bool full = row0 + WR <= end;
            if (elem == 8) {
                long long v[WR];
                if (VEC && full) {
                    const longlong2* s2 = (const longlong2*)(src + row0 * 8);
#pragma unroll
                    for (int k = 0; k < WR / 2; k++) { longlong2 t = s2[k]; v[2 * k] = t.x; v[2 * k + 1] = t.y; }
                }
                else {
#pragma unroll
                    for (int i = 0; i < WR; i++) v[i] = row0 + i < end ? ((const long long*)src)[row0 + i] : 0;
                }
#pragma unroll
                for (int i = 0; i < WR; i++)
                    if (((pid8 >> (8 * i)) & 0xffu) < 8) stage[(pos8 >> (8 * i)) & 0xffu] = v[i];
            }
            else if (elem == 4) {
                int v[WR];
                if (VEC && full) {
                    const int4* s4 = (const int4*)(src + row0 * 4);
#pragma unroll
                    for (int k = 0; k < WR / 4; k++) { int4 t = s4[k]; v[4 * k] = t.x; v[4 * k + 1] = t.y; v[4 * k + 2] = t.z; v[4 * k + 3] = t.w; }
                }
                else {
#pragma unroll
                    for (int i = 0; i < WR; i++) v[i] = row0 + i < end ? ((const int*)src)[row0 + i] : 0;
                }
#pragma unroll
                for (int i = 0; i < WR; i++)
                    if (((pid8 >> (8 * i)) & 0xffu) < 8) ((int*)stage)[(pos8 >> (8 * i)) & 0xffu] = v[i];
            }
            else if (elem == 2) {
#pragma unroll
                for (int i = 0; i < WR; i++)
                    if (((pid8 >> (8 * i)) & 0xffu) < 8) ((short*)stage)[(pos8 >> (8 * i)) & 0xffu] = ((const short*)src)[row0 + i];
            }
            else if (elem == 1) {
#pragma unroll
                for (int i = 0; i < WR; i++)
                    if (((pid8 >> (8 * i)) & 0xffu) < 8) ((char*)stage)[(pos8 >> (8 * i)) & 0xffu] = src[row0 + i];
            }
            else {
                // NULL-byte pseudo column: rows row0..row0+7 are exactly one byte of the validity bitmap (row0 % 8 == 0)
                // (src == nullptr: this rank's page has no NULLs in the column, another rank's has - every row is valid)
                unsigned int bits = (src && row0 < end) ? ((const uint8_t*)src)[row0 >> 3] : 0xffu;
#pragma unroll
                for (int i = 0; i < WR; i++)
                    if (((pid8 >> (8 * i)) & 0xffu) < 8) ((char*)stage)[(pos8 >> (8 * i)) & 0xffu] = ((bits >> i) & 1) ? 0 : 1;
            }
            __syncwarp();
            // copy-out in staged order: consecutive lanes write consecutive addresses inside a partition's run
            char* const* dstc = sdst + c * 8;
            const int es = elem ? elem : 1;
            for (int j = lane; j < tile_rows; j += 32) {
                int q = spid[j];
                long long d = run[q] + (j - toff[q]);
                char* base = dstc[q];
                switch (es) {
                    case 8: ((long long*)base)[d] = stage[j]; break;
                    case 4: ((int*)base)[d] = ((const int*)stage)[j]; break;
                    case 2: ((short*)base)[d] = ((const short*)stage)[j]; break;
                    default: base[d] = ((const char*)stage)[j]; break;
                }
            }
            __syncwarp();
        }
        if (lane < 8) run[lane] += field16(tlo, thi, lane);
        __syncwarp();
    }
}

// ---- lean warp-tile scatter for the exchange shape of a join: every lane is an 8-byte column without NULLs, the partition ids come from
// a plain BIGINT key, <= 8 partitions, 16-byte aligned columns.  Same tiles, ranks and output order as xchg_scatter_warp_kernel<VEC, KEYS>,
// with the per-row bookkeeping stripped (ncu on the generic kernel: 178 thread instructions per row, issue-bound at 59 %): 4-bit per-lane
// counters, the destination (partition, element offset) of every staged row computed ONCE per tile and reused by all columns, no
// element-size dispatch, no validity lanes.  A chunk's ragged last tile takes bounds-checked loads (rows beyond the end carry partition 8).
template <int NC, int MINB>
__global__ void __launch_bounds__(32 * WWARPS, MINB) xchg_scatter_lean8_kernel(int64_t n, int64_t wchunk, int32_t P, const long long* __restrict__ block_off, XchgCols cols,
                                                                          const long long* __restrict__ key0, int32_t bucket_count, const int32_t* __restrict__ b2p)
{
    __shared__ long long stage_all[WWARPS][WTILE];
    __shared__ long long delta_all[WWARPS][8];        // run[q] - tile offset of q: staged index j of partition q goes to element delta[q] + j
    __shared__ uint8_t spid_all[WWARPS][WTILE];
    __shared__ char* sdst[NC * 8];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int i = threadIdx.x; i < NC * P; i += blockDim.x) sdst[(i / P) * 8 + (i % P)] = cols.dst[i];
    __syncthreads();
    const int64_t vchunk = (int64_t)blockIdx.x * WWARPS + warp;
    const int64_t begin = vchunk * wchunk, end = min(n, begin + wchunk);
    if (begin >= n) return;
    long long* stage = stage_all[warp];
    long long* delta = delta_all[warp];
    uint8_t* spid = spid_all[warp];
    long long run = lane < P ? block_off[(size_t)vchunk * P + lane] : 0;      // lane q < 8 keeps partition q's running element offset
    for (int64_t tile = begin; tile < end; tile += WTILE) {
        const int64_t row0 = tile + lane * WR;
        const bool full = tile + WTILE <= end;
        // every column of the tile is requested up front (two at most are held in registers; the key doubles as a column when it is one):
        // the hash, the ranks and the staging of the first column then run under the latency of the others
        constexpr int NPRE = NC < 2 ? NC : 2;
        long long pre[NPRE][WR];
        auto load8 = [&](const long long* src, long long (&v)[WR]) {
            if (full) {
                const longlong2* s2 = (const longlong2*)(src + row0);
#pragma unroll
                for (int j = 0; j < WR / 2; j++) { longlong2 t = s2[j]; v[2 * j] = t.x; v[2 * j + 1] = t.y; }
            }
            else {
#pragma unroll
                for (int i = 0; i < WR; i++) v[i] = row0 + i < end ? src[row0 + i] : 0;
            }
        };
#pragma unroll
        for (int c = 0; c < NPRE; c++) load8((const long long*)cols.src[c], pre[c]);
        // partition of my 8 rows (4 bits each; 8 = no row)
        unsigned int pid4 = 0;
        {
            long long k[WR];
            const int key_col = (const void*)key0 == cols.src[0] ? 0 : (NPRE > 1 && (const void*)key0 == cols.src[1]) ? 1 : -1;      // warp-uniform
            if (key_col == 0) {
#pragma unroll
                for (int i = 0; i < WR; i++) k[i] = pre[0][i];
            }
            else if (NPRE > 1 && key_col == 1) {
#pragma unroll
                for (int i = 0; i < WR; i++) k[i] = pre[NPRE - 1][i];
            }
            else load8(key0, k);
#pragma unroll
            for (int i = 0; i < WR; i++) {
                int32_t bucket = process_raw_hash(hash_long(k[i]), bucket_count);
                unsigned int q = (unsigned int)(b2p ? b2p[bucket] : bucket);
                if (!full && row0 + i >= end) q = 8u;
                pid4 |= q << (4 * i);
            }
        }
        // my rows per partition (4-bit fields, <= 8) and, per row, how many of my earlier rows share its partition
        unsigned int c4 = 0, before4 = 0;
        unsigned int extra = 0;        // rows without a partition (ragged tile)
#pragma unroll
        for (int i = 0; i < WR; i++) {
            const unsigned int q = (pid4 >> (4 * i)) & 0xfu;
            if (q < 8u) {
                before4 |= ((c4 >> (4 * q)) & 0xfu) << (4 * i);
                c4 += 1u << (4 * q);
            }
            else extra++;
        }
        (void)extra;
        // inclusive scan over the lanes of the 8 counters as 16-bit fields in four 32-bit words (a field never exceeds 256).
        // (c4's fields can hold 8 = 0b1000 without touching their neighbour)
        unsigned int w0 = (c4 & 0xfu) | ((c4 & 0xf0u) << 12), w1 = ((c4 >> 8) & 0xfu) | ((c4 & 0xf000u) << 4),
                     w2 = ((c4 >> 16) & 0xfu) | ((c4 & 0xf00000u) >> 4), w3 = ((c4 >> 24) & 0xfu) | ((c4 & 0xf0000000u) >> 12);
        const unsigned int m0 = w0, m1 = w1, m2 = w2, m3 = w3;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            unsigned int a0 = __shfl_up_sync(0xffffffffu, w0, off), a1 = __shfl_up_sync(0xffffffffu, w1, off);
            unsigned int a2 = __shfl_up_sync(0xffffffffu, w2, off), a3 = __shfl_up_sync(0xffffffffu, w3, off);
            if (lane >= off) { w0 += a0; w1 += a1; w2 += a2; w3 += a3; }
        }
        // tile totals per partition, and where every partition starts inside the staged tile
        const unsigned int t0 = __shfl_sync(0xffffffffu, w0, 31), t1 = __shfl_sync(0xffffffffu, w1, 31);
        const unsigned int t2 = __shfl_sync(0xffffffffu, w2, 31), t3 = __shfl_sync(0xffffffffu, w3, 31);
        const unsigned int tot[8] = {t0 & 0xffffu, t0 >> 16, t1 & 0xffffu, t1 >> 16, t2 & 0xffffu, t2 >> 16, t3 & 0xffffu, t3 >> 16};
        unsigned int start[8];
        {
            unsigned int acc = 0;
#pragma unroll
            for (int q = 0; q < 8; q++) { start[q] = acc; acc += tot[q]; }
        }
        // exclusive counts of the lower lanes, per partition
        const unsigned int e0 = w0 - m0, e1 = w1 - m1, e2 = w2 - m2, e3 = w3 - m3;
        const unsigned int excl[8] = {e0 & 0xffffu, e0 >> 16, e1 & 0xffffu, e1 >> 16, e2 & 0xffffu, e2 >> 16, e3 & 0xffffu, e3 >> 16};
        // staged position of my rows (8 bits each) - the selects over q fold into a handful of instructions per row
        unsigned long long pos8 = 0;
#pragma unroll
        for (int i = 0; i < WR; i++) {
            const unsigned int q = (pid4 >> (4 * i)) & 0xfu;
            unsigned int base = 0;
#pragma unroll
            for (int p = 0; p < 8; p++) base = q == (unsigned int)p ? start[p] + excl[p] : base;
            const unsigned int pos = base + ((before4 >> (4 * i)) & 0xfu);
            if (q < 8u) {
                pos8 |= (unsigned long long)pos << (8 * i);
                spid[pos] = (uint8_t)q;
            }
        }
        if (lane < 8) {
            unsigned int st = 0, tt = 0;
#pragma unroll
            for (int p = 0; p < 8; p++) { st = lane == p ? start[p] : st; tt = lane == p ? tot[p] : tt; }
            delta[lane] = run - (long long)st;
            run += (long long)tt;
        }
        __syncwarp();
        const int tile_rows = (int)min((int64_t)WTILE, end - tile);
        // destination of the 8 staged rows this lane copies out (j = it * 32 + lane): partition (3 bits each) and element offset
        unsigned int qq = 0;
        unsigned int dd[WR];                 // (a page has at most 2^31 - 1 rows: element offsets fit 32 bits)
#pragma unroll
        for (int it = 0; it < WR; it++) {
            const int j = it * 32 + lane;
            const unsigned int q = j < tile_rows ? (unsigned int)spid[j] : 0u;
            qq |= q << (3 * it);
            dd[it] = (unsigned int)(delta[q] + j);
        }
#pragma unroll
        for (int c = 0; c < NC; c++) {
            long long v[WR];
            if (c < NPRE) {
#pragma unroll
                for (int i = 0; i < WR; i++) v[i] = pre[c < NPRE ? c : 0][i];
            }
            else load8((const long long*)cols.src[c], v);
            if (c > 0) __syncwarp();          // the previous column's copy-out has read the stage
#pragma unroll
            for (int i = 0; i < WR; i++)
                if (full || ((pid4 >> (4 * i)) & 0xfu) < 8u) stage[(pos8 >> (8 * i)) & 0xffu] = v[i];
            __syncwarp();
            char* const* dstc = sdst + c * 8;
#pragma unroll
            for (int it = 0; it < WR; it++) {
                const int j = it * 32 + lane;
                if (full || j < tile_rows) ((long long*)dstc[(qq >> (3 * it)) & 7u])[dd[it]] = stage[j];
            }
        }
        __syncwarp();
    }
}

// launch geometry shared by the histogram and scatter passes
struct XchgGeom {
    bool warp_mode;     // chunks are per warp (<= 8 partitions) or per CTA
    int grid;
    int64_t chunk;      // rows per chunk
    int nchunks;
};

// Local destinations and <= 8 partitions: warp-granular kernels.  Peer destinations: CTA-granular kernels - a warp-granular
// scatter keeps 8 x more destination streams open per SM, which on 8 GPUs (7 peer apertures) overruns the reach of the
// peer-aperture TLBs.
static XchgGeom xchg_geom(tgpu_ctx* ctx, int64_t n, int P, bool remote)
{
    XchgGeom g;
    n = std::max<int64_t>(n, 1);
    g.warp_mode = P <= 8 && !remote && !getenv("TGPU_XCHG_CTA");
    if (g.warp_mode) {
        // 12 CTAs per SM: whole waves for the kernels that keep 4 CTAs resident (3 waves) and for the lean scatter that keeps 3 (4 waves)
        int64_t warps = (int64_t)ctx->sm_count * 12 * WWARPS;
        g.chunk = tg_div_up(tg_div_up(n, warps), WTILE) * WTILE;
        g.nchunks = (int)tg_div_up(n, g.chunk);
        g.grid = (int)tg_div_up(g.nchunks, WWARPS);
    }
    else {
        int grid = tg_grid(ctx, n, XT * 16, 8);
        g.chunk = tg_div_up(tg_div_up(n, grid), XT) * XT;
        g.grid = g.nchunks = (int)std::max<int64_t>(1, tg_div_up(n, g.chunk));
    }
    return g;
}

// single BIGINT key channel without NULLs: the shape whose partition ids the scatter can recompute
static bool xchg_key_is_plain_bigint(const KeyCols& k)
{
    return k.count == 1 && !k.is_utf8[0] && !k.is_double[0] && k.cols[0].elem == 8 && !k.cols[0].validity;
}

// `pids` == nullptr (warp mode, plain BIGINT key only): no id array is written; pass the key to xchg_launch_scatter instead
static int xchg_launch_hist(tgpu_ctx* ctx, const XchgGeom& g, const KeyCols& k, int64_t n, int32_t bucket_count, const int32_t* b2p, int32_t P, uint8_t* pids,
                            unsigned int* hist)
{
    if (g.warp_mode) {
        bool fast = xchg_key_is_plain_bigint(k);
        if (fast) TG_LAUNCH(ctx, xchg_hist_warp_kernel<true>, g.grid, 32 * WWARPS, 0, k, n, g.chunk, bucket_count, b2p, P, pids, hist);
        else TG_LAUNCH(ctx, xchg_hist_warp_kernel<false>, g.grid, 32 * WWARPS, 0, k, n, g.chunk, bucket_count, b2p, P, pids, hist);
    }
    else TG_LAUNCH(ctx, xchg_hist_kernel, g.grid, XT, 0, k, n, g.chunk, bucket_count, b2p, P, pids, hist);
    return TGPU_OK;
}

// true when hist + scatter can run without the 1-byte id array for this geometry and key
static bool xchg_ids_from_key(const XchgGeom& g, const KeyCols& k)
{
    return g.warp_mode && xchg_key_is_plain_bigint(k) && !getenv("TGPU_XCHG_PID_ARRAY");
}

static int xchg_launch_scatter(tgpu_ctx* ctx, const XchgGeom& g, const uint8_t* pids, int64_t n, int32_t P, const long long* block_off, const XchgCols& xc,
                               const KeyCols* key = nullptr, int32_t bucket_count = 0, const int32_t* b2p = nullptr, bool any_order = false)
{
    if (any_order && !g.warp_mode && pids) {
        static bool attr_set = false;      // (per translation unit and process: the attribute is a property of the function)
        if (!attr_set) {
            TG_CUDA(ctx, cudaFuncSetAttribute(xchg_scatter_unordered_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)XU_SMEM));
            attr_set = true;
        }
        TG_LAUNCH(ctx, xchg_scatter_unordered_kernel, g.grid, XT, XU_SMEM, pids, n, g.chunk, P, block_off, xc);
        return TGPU_OK;
    }
    if (g.warp_mode) {
        const long long* key0 = pids ? nullptr : (const long long*)key->cols[0].data;
        bool vec = pids ? ((uintptr_t)pids & 7) == 0 : ((uintptr_t)key0 & 15) == 0;
        for (int c = 0; c < xc.count; c++) vec = vec && ((uintptr_t)xc.src[c] & 15) == 0;
        bool lean = key0 && vec && xc.count >= 1 && xc.count <= 4 && P <= 8 && !getenv("TGPU_XCHG_NO_LEAN");
        for (int c = 0; c < xc.count; c++) lean = lean && xc.elem[c] == 8;
        if (lean) {
            // 3 CTAs/SM leave the kernel 80 registers (no spills); 4 CTAs/SM cap it at 64 with ~100 bytes of spills per thread
            const char* e_minb = getenv("TGPU_XCHG_LEAN_MINB");
            const int minb = e_minb ? atoi(e_minb) : 3;
#define TG_LEAN(NC_)                                                                                                                                         \
    if (minb >= 4) TG_LAUNCH(ctx, (xchg_scatter_lean8_kernel<NC_, 4>), g.grid, 32 * WWARPS, 0, n, g.chunk, P, block_off, xc, key0, bucket_count, b2p);       \
    else if (minb == 2) TG_LAUNCH(ctx, (xchg_scatter_lean8_kernel<NC_, 2>), g.grid, 32 * WWARPS, 0, n, g.chunk, P, block_off, xc, key0, bucket_count, b2p);  \
    else TG_LAUNCH(ctx, (xchg_scatter_lean8_kernel<NC_, 3>), g.grid, 32 * WWARPS, 0, n, g.chunk, P, block_off, xc, key0, bucket_count, b2p)
            switch (xc.count) {
                case 1: TG_LEAN(1); break;
                case 2: TG_LEAN(2); break;
                case 3: TG_LEAN(3); break;
                default: TG_LEAN(4); break;
            }
#undef TG_LEAN
            return TGPU_OK;
        }
        if (key0) {
            if (vec) TG_LAUNCH(ctx, (xchg_scatter_warp_kernel<true, true>), g.grid, 32 * WWARPS, 0, pids, n, g.chunk, P, block_off, xc, key0, bucket_count, b2p);
            else TG_LAUNCH(ctx, (xchg_scatter_warp_kernel<false, true>), g.grid, 32 * WWARPS, 0, pids, n, g.chunk, P, block_off, xc, key0, bucket_count, b2p);
        }
        else {
            if (vec) TG_LAUNCH(ctx, (xchg_scatter_warp_kernel<true, false>), g.grid, 32 * WWARPS, 0, pids, n, g.chunk, P, block_off, xc, key0, bucket_count, b2p);
            else TG_LAUNCH(ctx, (xchg_scatter_warp_kernel<false, false>), g.grid, 32 * WWARPS, 0, pids, n, g.chunk, P, block_off, xc, key0, bucket_count, b2p);
        }
        return TGPU_OK;
    }
    TG_LAUNCH(ctx, xchg_scatter_kernel<4>, g.grid, XT, 0, pids, n, g.chunk, P, block_off, xc);
    return TGPU_OK;
}

}  // namespace
