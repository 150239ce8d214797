// join.cu — hash join build + probe for sm_90a.
//
// Reference semantics reproduced (bit-exact on address indices and output row order):
//   build : PagesIndex.addPage (M/operator/PagesIndex.java:224-256) keeps every build row; the address
//           index of a row is its global row number.  BigintPagesHash.insertValue
//           (M/operator/join/BigintPagesHash.java:122-141) + ArrayPositionLinks.link
//           (M/operator/join/ArrayPositionLinks.java:45-50): rows with a NULL key are skipped; for
//           duplicate keys the LAST inserted row is the chain head and links to the previous head, so a
//           chain lists its rows in descending row order.
//   probe : JoinProbe.fillCache (M/operator/join/unspilled/JoinProbe.java:112-180) ->
//           BigintPagesHash.getAddressIndex (:184-220): chain head or -1, NULL probe keys -> -1.
//   expand: PageJoiner.joinCurrentPosition / outerJoinCurrentPosition (PageJoiner.java:203-242) and
//           LookupJoinPageBuilder.build (LookupJoinPageBuilder.java:119-160): output rows in probe order,
//           within one probe row in chain order; probe columns first, then build output columns.
//   filter: JoinHash.isJoinPositionEligible (M/operator/join/JoinHash.java:154-157): a JoinFilterFunction over the
//           join-sources layout (build channels, then probe channels) drops the positions it does not accept, before
//           outputSingleMatch picks the first one and before an outer join falls back to its NULL-build row.
//
// Design: the table is an open-addressing array of 16-byte slots {int64 key, int32 head} so that one
// probe touches exactly one 32-byte sector; the deterministic "head = highest row" of the sequential
// reference insert order is obtained with atomicMax, and duplicate chains are materialised by a radix sort
// of (slot,row) pairs only when duplicates exist.  Slot placement (mix(key) & mask, linear probing) is not
// observable, only key -> head is.
#include <algorithm>
#include <mutex>

#include "expr.cuh"
#include "jit.cuh"
#include "rowkeys.cuh"

namespace {

using tg::KeyCols;
using tg::DProgram;

constexpr unsigned long long EMPTY_KEY = 0x8000000000000000ULL;   // INT64_MIN is kept out of the table

struct __align__(16) JoinSlot {
    unsigned long long key;
    int head;
    int pad;
};

enum KeyKind { KEY_INT = 0, KEY_DOUBLE = 1 };

// Slot of a key and the probe sequence.  Slot placement is not observable (only key -> head is).
//   mode 0: mix(key) & mask with linear probing, like the reference (M/operator/join/PagesHash.java:35-51).
//   mode 1: line-local: the 8 keys that share key >> 3 prefer the 8 slots of one 128-byte line (slot = key & 7), the
//           LINES are scattered with the murmur3 finaliser; the probe sequence walks the 8 slots of the line (wrapping
//           inside it) and then does the same in the following line.  Dense / clustered key domains probed in key
//           order turn random sector reads into sequential line reads; random keys behave like mode 0.
//   mode 2: order-preserving lines: line = (key - kmin) >> shift, with shift chosen at build time so that a line expects
//           about four keys; same in-line walk as mode 1.  The table is then laid out in key order: a probe page that arrives in
//           key order (TPC-H clustering; every sender's run after a stable hash exchange) walks the table front to back, whatever
//           subset of the key domain this table holds - after a hash exchange over W ranks a table holds every W-th key or so
//           of its domain, which leaves mode 1 with one useful key per line.  Chosen when the build keys spread evenly enough
//           over [kmin, kmax] (rows that had to leave their home line are counted during the build; too many -> mode 1).
struct JoinGeom {
    unsigned long long mask;   // capacity - 1 (capacity is a power of two, at least one 8-slot line)
    unsigned long long kmin;   // mode 2
    int shift;                 // mode 2
    int mode;
};

__host__ __device__ __forceinline__ unsigned long long join_slot_of(unsigned long long k, const JoinGeom& g)
{
    if (g.mode == 2) return ((((k - g.kmin) >> g.shift) << 3) | (k & 7)) & g.mask;
    if (g.mode == 1) return ((tg::murmur3_mix(k >> 3) << 3) | (k & 7)) & g.mask;
    return tg::murmur3_mix(k) & g.mask;
}

__host__ __device__ __forceinline__ unsigned long long join_next_slot(unsigned long long pos, unsigned long long k, const JoinGeom& g)
{
    if (g.mode != 0) {
        unsigned long long in = (pos + 1) & 7;
        if (in != (k & 7)) return (pos & ~7ULL) | in;
        return ((((pos >> 3) + 1) << 3) | (k & 7)) & g.mask;
    }
    return (pos + 1) & g.mask;
}

// canonical 64-bit join key; returns false when the row can never match (NULL, or NaN under EQUAL)
__device__ __forceinline__ bool join_key(const ColRef& c, int kind, int64_t i, unsigned long long* out)
{
    if (!tg_valid(c.validity, i)) return false;
    int64_t v = tg_load_i64(c, i);
    if (kind == KEY_DOUBLE) {
        unsigned long long u = (unsigned long long)v;
        if ((u << 1) == 0) u = 0;                                            // -0.0 == +0.0
        if ((u & 0x7FFFFFFFFFFFFFFFULL) > 0x7FF0000000000000ULL) return false;  // NaN != NaN
        v = (int64_t)u;
    }
    *out = (unsigned long long)v;
    return true;
}

// one thread per build row: claim/find the key's slot, head = max(row).  *dup_flag is set when a key repeats.
// moved[0] += rows that left their home line, moved[1] += rows that went more than 8 lines away (layout quality of modes 1 / 2).
// give_up_lines > 0 (a TRIAL geometry): a row that would have to move further than that many lines is not inserted and counted in
// *gave_up, and once more than give_up_limit rows did so the whole pass stops - the host rejects the geometry, so the rest of the
// table is never needed.  (Without the bound a geometry that does not suit the keys - e.g. the dense lines over the random half of an
// order-key domain that a hash exchange leaves on a rank - clusters into chains thousands of lines long: 174 s for 75 M rows, measured.)
__global__ void __launch_bounds__(256) join_build_kernel(ColRef key, int kind, int64_t n, JoinSlot* __restrict__ table, JoinGeom geo,
                                                         int* __restrict__ special_head, int* __restrict__ dup_flag, unsigned int* __restrict__ moved,
                                                         int give_up_lines, unsigned int give_up_limit, unsigned int* __restrict__ gave_up)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    unsigned int left_home = 0, went_far = 0;
    for (; i < n; i += stride) {
        if (give_up_lines > 0 && *((volatile unsigned int*)gave_up) > give_up_limit) break;
        unsigned long long k;
        if (!join_key(key, kind, i, &k)) continue;
        if (k == EMPTY_KEY) {
            int old = atomicMax(special_head, (int)i);
            if (old >= 0) *dup_flag = 1;
            continue;
        }
        unsigned long long pos = join_slot_of(k, geo);
        const unsigned long long home = pos >> 3;
        bool placed = true;
        while (true) {
            unsigned long long cur = *((volatile unsigned long long*)&table[pos].key);
            if (cur == EMPTY_KEY) cur = atomicCAS(&table[pos].key, EMPTY_KEY, k);
            if (cur == EMPTY_KEY || cur == k) {
                int old = atomicMax(&table[pos].head, (int)i);
                if (old >= 0) *dup_flag = 1;
                break;
            }
            pos = join_next_slot(pos, k, geo);
            if (give_up_lines > 0 && (((pos >> 3) - home) & (geo.mask >> 3)) > (unsigned long long)give_up_lines) { placed = false; break; }
        }
        if (!placed) { atomicAdd(gave_up, 1u); continue; }
        if (geo.mode != 0 && (pos >> 3) != home) {
            left_home++;
            went_far += (((pos >> 3) - home) & (geo.mask >> 3)) > 8;
        }
    }
    if (geo.mode != 0) {
        for (int off = 16; off > 0; off >>= 1) {
            left_home += __shfl_xor_sync(0xffffffffu, left_home, off);
            went_far += __shfl_xor_sync(0xffffffffu, went_far, off);
        }
        if ((threadIdx.x & 31) == 0 && left_home) { atomicAdd(moved, left_home); atomicAdd(moved + 1, went_far); }
    }
}

// min / max of the non-NULL integer keys of the build side (mode 2 geometry)
__global__ void join_key_range_kernel(ColRef key, int64_t n, long long* __restrict__ minmax)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    long long lo = INT64_MAX, hi = INT64_MIN;
    for (; i < n; i += stride) {
        if (!tg_valid(key.validity, i)) continue;
        long long v = tg_load_i64(key, i);
        if ((unsigned long long)v == EMPTY_KEY) continue;
        lo = v < lo ? v : lo;
        hi = v > hi ? v : hi;
    }
    for (int off = 16; off > 0; off >>= 1) {
        long long a = __shfl_xor_sync(0xffffffffu, lo, off), b = __shfl_xor_sync(0xffffffffu, hi, off);
        lo = a < lo ? a : lo;
        hi = b > hi ? b : hi;
    }
    if ((threadIdx.x & 31) == 0 && lo <= hi) { atomicMin(minmax, lo); atomicMax(minmax + 1, hi); }
}

__device__ __forceinline__ int join_lookup(const JoinSlot* __restrict__ table, JoinGeom geo, unsigned long long k, int special_head)
{
    if (k == EMPTY_KEY) return special_head;
    unsigned long long pos = join_slot_of(k, geo);
    while (true) {
        int4 s = __ldg((const int4*)&table[pos]);
        unsigned long long sk = (unsigned long long)(unsigned int)s.x | ((unsigned long long)(unsigned int)s.y << 32);
        if (sk == k) return s.z;
        if (sk == EMPTY_KEY) return -1;
        pos = join_next_slot(pos, k, geo);
    }
}

// Index-only probe (the headline kernel).  ROWS independent lookups per thread are issued before any is
// consumed so that each thread keeps ROWS random 16-byte sector reads in flight; consecutive probe rows with
// the same key (TPC-H clustering) collapse in the coalescer / L1.
// Algorithmic bytes per probe row: 8 (key) + 12 (slot) + 4 (position) = 24 (SURVEY.md §8d).
template <int ROWS, bool INT64_NO_NULLS>
__global__ void __launch_bounds__(256) join_probe_kernel(ColRef key, int kind, int64_t n, const JoinSlot* __restrict__ table, JoinGeom geo,
                                                         int special_head, int* __restrict__ out)
{
    int64_t tile = (int64_t)blockDim.x * ROWS;
    int64_t tiles = (n + tile - 1) / tile;
    for (int64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
        int64_t base = t * tile + threadIdx.x;
        unsigned long long k[ROWS];
        bool ok[ROWS];
        int4 s[ROWS];
        unsigned long long pos[ROWS];
#pragma unroll
        for (int j = 0; j < ROWS; j++) {
            int64_t i = base + (int64_t)j * blockDim.x;
            ok[j] = false;
            k[j] = 0;
            if (i < n) {
                if (INT64_NO_NULLS) { k[j] = (unsigned long long)__ldg((const long long*)key.data + i); ok[j] = true; }
                else ok[j] = join_key(key, kind, i, &k[j]);
            }
            pos[j] = join_slot_of(k[j], geo);
        }
#pragma unroll
        for (int j = 0; j < ROWS; j++) {
            if (ok[j] && k[j] != EMPTY_KEY) s[j] = __ldg((const int4*)&table[pos[j]]);
            else s[j] = make_int4(0, (int)0x80000000, -1, 0);
        }
        // each row walks its probe sequence on its own rather than in lock-step rounds over the ROWS rows of a thread
#pragma unroll
        for (int j = 0; j < ROWS; j++) {
            int64_t i = base + (int64_t)j * blockDim.x;
            if (i >= n) continue;
            int res = -1;
            if (ok[j]) {
                if (k[j] == EMPTY_KEY) res = special_head;
                else {
                    unsigned long long p = pos[j];
                    int4 cur = s[j];
                    while (true) {
                        unsigned long long sk = (unsigned long long)(unsigned int)cur.x | ((unsigned long long)(unsigned int)cur.y << 32);
                        if (sk == k[j]) { res = cur.z; break; }
                        if (sk == EMPTY_KEY) break;
                        p = join_next_slot(p, k[j], geo);
                        cur = __ldg((const int4*)&table[p]);
                    }
                }
            }
            out[i] = res;
        }
    }
}



struct GatherCols {
    int count;
    int by_slot;
    int elem[4];
    const void* src[4];
    void* dst[4];
};

// Match bitmap of the fused probes: bit i of 32-bit word i / 32 is set when probe row i found its key (Arrow LSB order, so the words
// are the build columns' validity under PROBE_OUTER).  Every fused kernel gives lane L of a warp row warp_row + L, 32 consecutive,
// 32-aligned rows: one ballot makes the word, lane 0 stores it and counts its bits.  All 32 lanes must get here.
__device__ __forceinline__ void store_match_word(unsigned int* __restrict__ match_bits, int64_t warp_row, bool hit, unsigned int* matched)
{
    const unsigned int word = __ballot_sync(0xffffffffu, hit);
    if ((threadIdx.x & 31) == 0) {
        match_bits[warp_row >> 5] = word;
        *matched += __popc(word);
    }
}

// lane 0 of each warp holds the warp's count: one atomic per warp
__device__ __forceinline__ void add_match_count(unsigned long long* __restrict__ match_count, unsigned int matched)
{
    if ((threadIdx.x & 31) == 0 && matched) atomicAdd(match_count, (unsigned long long)matched);
}

// Fused probe + build-side gather for the common join shape (no duplicate chains, fixed-width non-null build
// columns): the chain head is looked up and the build payload of the matching row is fetched while the slot is
// still in flight in the same thread, so the positions never make a round trip through HBM before the gather and
// no count/scan pass is needed when every probe row matches (FK -> PK joins).  Misses are counted; the host
// compacts only when there are any.  Which rows matched goes to the match bitmap (see store_match_word); its words past n are not
// written, its bits at or past n are 0.  Launched with blockDim.x a multiple of 32, and match_bits 32-row aligned.
template <int ROWS, bool INT64_NO_NULLS>
__global__ void __launch_bounds__(256) join_probe_gather_kernel(ColRef key, int kind, int64_t n, const JoinSlot* __restrict__ table, JoinGeom geo,
                                                                int special_head, unsigned int* __restrict__ match_bits, GatherCols g, unsigned long long* __restrict__ match_count)
{
    // g.by_slot: payload arrays are indexed by table slot (special key at index mask + 1), else by build row id
    int64_t tile = (int64_t)blockDim.x * ROWS;
    int64_t tiles = (n + tile - 1) / tile;
    unsigned int matched = 0;
    for (int64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
        int64_t base = t * tile + threadIdx.x;
        unsigned long long k[ROWS];
        bool ok[ROWS];
        int4 s[ROWS];
        unsigned long long pos[ROWS];
        int res[ROWS];
        long long at[ROWS];      // index into the payload arrays
#pragma unroll
        for (int j = 0; j < ROWS; j++) {
            int64_t i = base + (int64_t)j * blockDim.x;
            ok[j] = false;
            k[j] = 0;
            if (i < n) {
                if (INT64_NO_NULLS) { k[j] = (unsigned long long)__ldg((const long long*)key.data + i); ok[j] = true; }
                else ok[j] = join_key(key, kind, i, &k[j]);
            }
            pos[j] = join_slot_of(k[j], geo);
        }
#pragma unroll
        for (int j = 0; j < ROWS; j++) {
            if (ok[j] && k[j] != EMPTY_KEY) s[j] = __ldg((const int4*)&table[pos[j]]);
            else s[j] = make_int4(0, (int)0x80000000, -1, 0);
        }
#pragma unroll
        for (int j = 0; j < ROWS; j++) {
            int r = -1;
            long long where = 0;
            if (ok[j]) {
                if (k[j] == EMPTY_KEY) { r = special_head; where = (long long)geo.mask + 1; }
                else {
                    unsigned long long p = pos[j];
                    int4 cur = s[j];
                    while (true) {
                        unsigned long long sk = (unsigned long long)(unsigned int)cur.x | ((unsigned long long)(unsigned int)cur.y << 32);
                        if (sk == k[j]) { r = cur.z; where = (long long)p; break; }
                        if (sk == EMPTY_KEY) break;
                        p = join_next_slot(p, k[j], geo);
                        cur = __ldg((const int4*)&table[p]);
                    }
                }
            }
            res[j] = r;
            at[j] = g.by_slot ? where : (long long)r;
        }
        // build payload: ROWS x columns independent random loads, then coalesced stores
        for (int c = 0; c < g.count; c++) {
            long long v[ROWS];
#pragma unroll
            for (int j = 0; j < ROWS; j++) {
                v[j] = 0;
                if (res[j] >= 0) {
                    switch (g.elem[c]) {
                        case 8: v[j] = __ldg((const long long*)g.src[c] + at[j]); break;
                        case 4: v[j] = __ldg((const int*)g.src[c] + at[j]); break;
                        case 2: v[j] = __ldg((const short*)g.src[c] + at[j]); break;
                        default: v[j] = __ldg((const signed char*)g.src[c] + at[j]); break;
                    }
                }
            }
#pragma unroll
            for (int j = 0; j < ROWS; j++) {
                int64_t i = base + (int64_t)j * blockDim.x;
                if (i >= n) continue;
                switch (g.elem[c]) {
                    case 8: ((long long*)g.dst[c])[i] = v[j]; break;
                    case 4: ((int*)g.dst[c])[i] = (int)v[j]; break;
                    case 2: ((short*)g.dst[c])[i] = (short)v[j]; break;
                    default: ((signed char*)g.dst[c])[i] = (signed char)v[j]; break;
                }
            }
        }
#pragma unroll
        for (int j = 0; j < ROWS; j++) {
            // every lane takes part in the ballot: rows at or past n have res = -1; the warp's first row decides whether its word exists
            const int64_t warp_row = base - (threadIdx.x & 31) + (int64_t)j * blockDim.x;
            const unsigned int word = __ballot_sync(0xffffffffu, res[j] >= 0);
            if ((threadIdx.x & 31) == 0 && warp_row < n) {
                match_bits[warp_row >> 5] = word;
                matched += __popc(word);
            }
        }
    }
    add_match_count(match_count, matched);
}

// compaction flags of an INNER join page from the match bitmap: flags[i] = bit i
__global__ void join_match_flags_kernel(const unsigned int* __restrict__ match_bits, int64_t n, uint8_t* __restrict__ flags)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) flags[i] = (uint8_t)((match_bits[i >> 5] >> (i & 31)) & 1u);
}



// ---- generic join keys (DefaultPagesHash shape: several channels and/or variable width) ---------------------------
// The table is keyed by the 64-bit ROW HASH of the key columns (the reference's DefaultPagesHash also addresses by
// mix(rowHash), M/operator/join/DefaultPagesHash.java:105-122).  Exactness comes from two checks against the real key
// columns: at build time every row must carry the same key as the head of its slot (a 64-bit collision between
// different keys makes the build answer NOT_SUPPORTED so the caller keeps the Java operator), and at probe time a hit
// is kept only when the probe row's key equals the build row's key.
__global__ void join_fingerprint_kernel(KeyCols k, int64_t n, const uint8_t* __restrict__ attempt, long long* __restrict__ fp, uint8_t* __restrict__ is_null)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        bool ok = tg::row_joinable(k, i);
        fp[i] = ok ? (long long)tg::row_hash_attempt(k, i, attempt ? attempt[i] : 0) : 0;
        is_null[i] = ok ? 0 : 1;
    }
}

// build: a row whose key differs from the key of its slot's head row shares the slot's 64-bit hash with another key: it moves on to
// its next hash function (attempt + 1); the table is then rebuilt.  Rows of one key always agree with their head, so chains stay pure.
__global__ void join_verify_build_kernel(KeyCols k, const long long* __restrict__ fp, const uint8_t* __restrict__ fp_validity, int64_t n,
                                         const JoinSlot* __restrict__ table, JoinGeom geo, int special_head, uint8_t* __restrict__ attempt, int* __restrict__ moved)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        if (!tg_valid(fp_validity, i)) continue;
        int head = join_lookup(table, geo, (unsigned long long)fp[i], special_head);
        if (head != (int)i && head >= 0 && !tg::rows_equal_for_join(k, i, k, head)) {
            attempt[i] = (uint8_t)(attempt[i] + 1);
            atomicAdd(moved, 1);
        }
    }
}

// probe, attempt 0: a hit whose key differs is a miss when the build needed one hash function only, else it stays open (-2) for the
// next attempt
__global__ void join_verify_probe_kernel(KeyCols probe, KeyCols build, int64_t n, int more_attempts, int* __restrict__ jp)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        int b = jp[i];
        if (b >= 0 && !tg::rows_equal_for_join(probe, i, build, b)) jp[i] = more_attempts ? -2 : -1;
    }
}

// probe, attempt a >= 1 of the rows still open: look the a-th hash up; an empty slot or the last attempt closes the row as a miss
__global__ void join_probe_retry_kernel(KeyCols probe, KeyCols build, int64_t n, const JoinSlot* __restrict__ table, JoinGeom geo, int special_head, int attempt, int last,
                                        int* __restrict__ jp)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        if (jp[i] != -2) continue;
        int head = join_lookup(table, geo, (unsigned long long)tg::row_hash_attempt(probe, i, attempt), special_head);
        if (head >= 0 && tg::rows_equal_for_join(probe, i, build, head)) jp[i] = head;
        else if (head < 0 || last) jp[i] = -1;
    }
}

// ---- lean probe kernels for the headline shape (BIGINT key without NULLs, whole 1024-row tiles) -------------------
// Same algorithm as join_probe_kernel / join_probe_gather_kernel with the per-row bookkeeping stripped: the layout
// mode is a template parameter, slot indices are 32-bit, there are no bounds or validity checks (the ragged tail and
// every other key shape go through the generic kernels).  ncu showed the generic kernels spending ~215 thread
// instructions per probe row at 44-48 % issue utilisation, i.e. instruction-bound as much as latency-bound.
template <int MODE>
__device__ __forceinline__ unsigned int lean_slot(unsigned long long k, unsigned int mask, unsigned long long kmin, int shift)
{
    if (MODE == 2) return (((unsigned int)((k - kmin) >> shift) << 3) | ((unsigned int)k & 7u)) & mask;
    if (MODE == 1) return (((unsigned int)tg::murmur3_mix(k >> 3) << 3) | ((unsigned int)k & 7u)) & mask;
    return (unsigned int)tg::murmur3_mix(k) & mask;
}

template <int MODE>
__device__ __forceinline__ unsigned int lean_next(unsigned int pos, unsigned int k_low3, unsigned int mask)
{
    if (MODE != 0) {
        unsigned int in = (pos + 1) & 7u;
        return in != k_low3 ? ((pos & ~7u) | in) : (((pos & ~7u) + 8u + k_low3) & mask);
    }
    return (pos + 1) & mask;
}

// persistent-tile kernels: exactly as many CTAs as are co-resident, so that no partial second wave runs at low occupancy
template <class K>
static int lean_grid(tgpu_ctx* ctx, K kernel, int64_t tiles, int threads = 256, size_t smem = 0)
{
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem) != cudaSuccess || per_sm < 1) per_sm = 4;
    return (int)std::min<int64_t>(tiles, (int64_t)ctx->sm_count * per_sm);
}

// GATHER = false: the join position of every row goes to out[].  GATHER = true: the build payload goes to g.dst and the match bits
// to match_bits (out is unused)
template <int MODE, bool GATHER, int MINB = 1>
__global__ void __launch_bounds__(256, MINB) join_probe_lean_kernel(const long long* __restrict__ keys, int64_t tiles, const int4* __restrict__ table, unsigned int mask,
                                                              unsigned long long kmin, int shift, int special_head, int* __restrict__ out, unsigned int* __restrict__ match_bits,
                                                              GatherCols g, unsigned long long* __restrict__ match_count)
{
    // the word behind the match counter holds the layout choice of the page (0 = these 16-byte slots; join_probe_locality_kernel decides)
    if (GATHER && *(const volatile int*)(match_count + 1) != 0) return;
    unsigned int matched = 0;
    for (int64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
        const int64_t base = t * 1024 + threadIdx.x;
        unsigned long long k[4];
        unsigned int pos[4];
        int4 s[4];
#pragma unroll
        for (int j = 0; j < 4; j++) k[j] = (unsigned long long)__ldg(keys + base + j * 256);
#pragma unroll
        for (int j = 0; j < 4; j++) pos[j] = lean_slot<MODE>(k[j], mask, kmin, shift);
#pragma unroll
        for (int j = 0; j < 4; j++) s[j] = __ldg(table + pos[j]);
        int res[4];
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const unsigned int klo = (unsigned int)k[j], khi = (unsigned int)(k[j] >> 32);
            int r = -1;
            int4 cur = s[j];
            unsigned int p = pos[j];
            while (true) {
                if ((unsigned int)cur.x == klo && (unsigned int)cur.y == khi) { r = cur.z; break; }
                if (cur.x == 0 && cur.y == (int)0x80000000) break;                 // EMPTY_KEY
                p = lean_next<MODE>(p, klo & 7u, mask);
                cur = __ldg(table + p);
            }
            if (k[j] == EMPTY_KEY) { r = special_head; p = mask + 1u; }
            res[j] = r;
            pos[j] = p;
        }
        if (GATHER) {
#pragma unroll
            for (int c = 0; c < 4; c++) {      // static indices: the parameter struct stays in the constant bank
                if (c >= g.count) break;
                if (g.elem[c] == 8) {
                    long long v[4];
#pragma unroll
                    for (int j = 0; j < 4; j++) v[j] = res[j] >= 0 ? __ldg((const long long*)g.src[c] + (g.by_slot ? (long long)pos[j] : (long long)res[j])) : 0;
#pragma unroll
                    for (int j = 0; j < 4; j++) ((long long*)g.dst[c])[base + j * 256] = v[j];
                }
                else if (g.elem[c] == 4) {
                    int v[4];
#pragma unroll
                    for (int j = 0; j < 4; j++) v[j] = res[j] >= 0 ? __ldg((const int*)g.src[c] + (g.by_slot ? (long long)pos[j] : (long long)res[j])) : 0;
#pragma unroll
                    for (int j = 0; j < 4; j++) ((int*)g.dst[c])[base + j * 256] = v[j];
                }
                else {
#pragma unroll
                    for (int j = 0; j < 4; j++) {
                        long long at = g.by_slot ? (long long)pos[j] : (long long)res[j];
                        if (g.elem[c] == 2) ((short*)g.dst[c])[base + j * 256] = res[j] >= 0 ? ((const short*)g.src[c])[at] : (short)0;
                        else ((signed char*)g.dst[c])[base + j * 256] = res[j] >= 0 ? ((const signed char*)g.src[c])[at] : (signed char)0;
                    }
                }
            }
        }
#pragma unroll
        for (int j = 0; j < 4; j++) {
            if (GATHER) store_match_word(match_bits, base + j * 256, res[j] >= 0, &matched);
            else out[base + j * 256] = res[j];
        }
    }
    if (GATHER) add_match_count(match_count, matched);
}

// ---- TMA-staged probe for order-preserving tables (mode 2) ----------------------------------------------------------------
// With order-preserving lines a tile of probe keys that arrives in key order (TPC-H clustering; each sender's run after a stable
// exchange) needs ONE contiguous span of table lines.  The CTA computes the span of its 1024 keys, one elected thread stages the span -
// the 16-byte slots and, for the common single-BIGINT-payload shape, the slot-ordered payload next to them - into shared memory with
// cp.async.bulk (TMA bulk copy, completion on an mbarrier), and every thread then resolves its four rows against shared memory:
// one bulk copy of full 128-byte lines replaces ~2 x 1024 scattered 16 / 8-byte loads.  A tile whose span does not fit (shuffled keys, keys
// outside the build range) takes the direct path of the lean kernel; a row whose line walk leaves the staged span falls back to global
// loads for its remaining steps.
constexpr int SPAN_LINES = 80;            // table lines staged per tile: 10 KB of slots + 5 KB of payload

__device__ __forceinline__ unsigned int smem_u32(const void* p) { return (unsigned int)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(unsigned long long* bar, int count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned int bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, unsigned int bytes, unsigned long long* bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes),
                 "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned int parity)
{
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "TG_WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra TG_DONE_%=;\n"
        "bra TG_WAIT_%=;\n"
        "TG_DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long* bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

template <bool GATHER>
__global__ void __launch_bounds__(256, 6) join_probe_span_kernel(const long long* __restrict__ keys, int64_t tiles, const int4* __restrict__ table, unsigned int mask,
                                                                unsigned long long kmin, int shift, int special_head, int* __restrict__ out,
                                                                unsigned int* __restrict__ match_bits, GatherCols g, unsigned long long* __restrict__ match_count)
{
    __shared__ __align__(128) int4 s_slots[SPAN_LINES * 8];
    __shared__ __align__(128) long long s_pay[SPAN_LINES * 8];
    __shared__ __align__(8) unsigned long long bar;
    __shared__ unsigned int s_min[8], s_max[8];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const unsigned int line_mask = mask >> 3;
    // the slot-ordered single 8-byte payload is staged next to the slots; other payload shapes are read from global memory
    const bool stage_pay = GATHER && g.by_slot && g.count == 1 && g.elem[0] == 8;
    if (threadIdx.x == 0) mbar_init(&bar, 1);
    __syncthreads();
    unsigned int phase = 0;
    unsigned int matched = 0;
    for (int64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
        const int64_t base = t * 1024 + threadIdx.x;
        unsigned long long k[4];
        unsigned int pos[4];
#pragma unroll
        for (int j = 0; j < 4; j++) k[j] = (unsigned long long)__ldg(keys + base + j * 256);
        unsigned int lo = 0xffffffffu, hi = 0;
#pragma unroll
        for (int j = 0; j < 4; j++) {
            pos[j] = lean_slot<2>(k[j], mask, kmin, shift);
            const unsigned int line = pos[j] >> 3;
            lo = min(lo, line);
            hi = max(hi, line);
        }
        lo = __reduce_min_sync(0xffffffffu, lo);
        hi = __reduce_max_sync(0xffffffffu, hi);
        if (lane == 0) { s_min[warp] = lo; s_max[warp] = hi; }
        __syncthreads();
#pragma unroll
        for (int w = 0; w < 8; w++) { lo = min(lo, s_min[w]); hi = max(hi, s_max[w]); }
        // one extra line behind the span for line walks that overflow their home line
        const unsigned int first_line = lo, lines = min(hi + 1u, line_mask) - lo + 1u;
        const bool staged = lines <= (unsigned int)SPAN_LINES;
        if (staged) {
            if (threadIdx.x == 0) {
                const unsigned int slot_bytes = lines * 128u, pay_bytes = stage_pay ? lines * 64u : 0u;
                mbar_expect_tx(&bar, slot_bytes + pay_bytes);
                bulk_g2s(s_slots, table + (size_t)first_line * 8, slot_bytes, &bar);
                if (stage_pay) bulk_g2s(s_pay, (const long long*)g.src[0] + (size_t)first_line * 8, pay_bytes, &bar);
            }
            mbar_wait(&bar, phase);
            phase ^= 1u;
        }
        const unsigned int first_slot = first_line << 3, staged_slots = staged ? lines << 3 : 0u;
        int res[4];
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const unsigned int klo = (unsigned int)k[j], khi = (unsigned int)(k[j] >> 32);
            int r = -1;
            unsigned int p = pos[j];
            while (true) {
                const unsigned int local = p - first_slot;
                const int4 cur = local < staged_slots ? s_slots[local] : __ldg(table + p);
                if ((unsigned int)cur.x == klo && (unsigned int)cur.y == khi) { r = cur.z; break; }
                if (cur.x == 0 && cur.y == (int)0x80000000) break;                 // EMPTY_KEY
                p = lean_next<2>(p, klo & 7u, mask);
            }
            if (k[j] == EMPTY_KEY) { r = special_head; p = mask + 1u; }
            res[j] = r;
            pos[j] = p;
        }
        if (GATHER) {
#pragma unroll
            for (int c = 0; c < 4; c++) {
                if (c >= g.count) break;
                if (g.elem[c] == 8) {
                    long long v[4];
#pragma unroll
                    for (int j = 0; j < 4; j++) {
                        const unsigned int local = pos[j] - first_slot;
                        if (res[j] < 0) v[j] = 0;
                        else if (stage_pay && local < staged_slots) v[j] = s_pay[local];
                        else v[j] = __ldg((const long long*)g.src[c] + (g.by_slot ? (long long)pos[j] : (long long)res[j]));
                    }
#pragma unroll
                    for (int j = 0; j < 4; j++) ((long long*)g.dst[c])[base + j * 256] = v[j];
                }
                else if (g.elem[c] == 4) {
#pragma unroll
                    for (int j = 0; j < 4; j++)
                        ((int*)g.dst[c])[base + j * 256] = res[j] >= 0 ? __ldg((const int*)g.src[c] + (g.by_slot ? (long long)pos[j] : (long long)res[j])) : 0;
                }
                else {
#pragma unroll
                    for (int j = 0; j < 4; j++) {
                        long long at = g.by_slot ? (long long)pos[j] : (long long)res[j];
                        if (g.elem[c] == 2) ((short*)g.dst[c])[base + j * 256] = res[j] >= 0 ? ((const short*)g.src[c])[at] : (short)0;
                        else ((signed char*)g.dst[c])[base + j * 256] = res[j] >= 0 ? ((const signed char*)g.src[c])[at] : (signed char)0;
                    }
                }
            }
        }
#pragma unroll
        for (int j = 0; j < 4; j++) {
            if (GATHER) store_match_word(match_bits, base + j * 256, res[j] >= 0, &matched);
            else out[base + j * 256] = res[j];
        }
        __syncthreads();          // everyone is done with the staged span (and s_min / s_max) before the next tile overwrites them
    }
    if (GATHER) add_match_count(match_count, matched);
}

// launch of the lean probe kernel for the table's layout mode (out: positions of the index-only probe; match_bits: of the fused one)
template <bool GATHER>
static int launch_lean(tgpu_ctx* ctx, const JoinGeom& geo, const long long* keys, int64_t tiles, const int4* table, int special_head, int* out,
                       unsigned int* match_bits, const GatherCols& g, unsigned long long* matches)
{
    const unsigned int mask32 = (unsigned int)geo.mask;
    // 8 CTAs per SM (32 registers): full occupancy is worth more than the registers
    if (geo.mode == 2 && getenv("TGPU_JOIN_SPAN")) {
        // TMA-staged table spans (falls back per tile when the keys are not clustered).  Opt-in: with the dense table the lean kernel
        // already streams the table once, and the span kernel pays a block-wide span reduction plus a second dependent DRAM round trip per tile
        auto k = join_probe_span_kernel<GATHER>;
        TG_LAUNCH(ctx, k, lean_grid(ctx, k, tiles), 256, 0, keys, tiles, table, mask32, geo.kmin, geo.shift, special_head, out, match_bits, g, matches);
    }
    else if (geo.mode == 2) {
        auto k = join_probe_lean_kernel<2, GATHER, 8>;
        TG_LAUNCH(ctx, k, lean_grid(ctx, k, tiles), 256, 0, keys, tiles, table, mask32, geo.kmin, geo.shift, special_head, out, match_bits, g, matches);
    }
    else if (geo.mode == 1) {
        auto k = join_probe_lean_kernel<1, GATHER, 8>;
        TG_LAUNCH(ctx, k, lean_grid(ctx, k, tiles), 256, 0, keys, tiles, table, mask32, 0ULL, 0, special_head, out, match_bits, g, matches);
    }
    else {
        auto k = join_probe_lean_kernel<0, GATHER, 8>;
        TG_LAUNCH(ctx, k, lean_grid(ctx, k, tiles), 256, 0, keys, tiles, table, mask32, 0ULL, 0, special_head, out, match_bits, g, matches);
    }
    return TGPU_OK;
}

// ---- wide slots: key, head and the build payload of the head row in ONE 32-byte sector ------------------------------------------
// A probe page without key locality (the survey's variant B, or any join whose probe side is not clustered on the join key) pays one
// random DRAM sector per array it touches for a row: the 16-byte slot, then one sector per slot-ordered payload column.  The wide table
// holds the same slots at a 32-byte stride with up to two payload cells (8 bytes each) behind key and head, so that a row costs ONE
// random sector whatever the number of payload columns - and two independent 128-bit loads instead of three dependent-address loads.
// On a key-ordered probe page the bytes are the same as slot table + slot-ordered payload arrays, read front to back.
// Built next to the 16-byte table (which the index-only probe, the duplicate chains and every generic kernel keep using).
struct __align__(32) WideSlot {
    static constexpr int CELLS = 2;
    static constexpr bool LINE_RELATIVE = false;
    unsigned long long key;
    int head;
    int pad;
    unsigned long long cell[2];
};

// ---- keyed slots: key and the payload of its head row in 16 bytes, for builds with ONE payload column ------------------------------
// With a single payload column of at most 8 bytes (no NULLs, no duplicate keys) the head row id is never needed: the slot is {key, cell},
// and one 128-bit load both resolves a probe row and fetches its payload.  On a key-ordered probe page this reads 16 bytes per slot
// instead of the 16-byte slot plus its slot-ordered payload cell, with no dependent payload load; on a page without key locality it is
// one random sector per row, like the wide slot.  It replaces the wide table for these builds.  An occupied slot always matches (its key
// was inserted, so its head is >= 0); the special key INT64_MIN keeps its cell in slot mask + 1, as in the wide table.
struct __align__(16) KeyedSlot {
    static constexpr int CELLS = 1;
    static constexpr bool LINE_RELATIVE = false;
    unsigned long long key;
    unsigned long long cell;
};

// ---- packed keyed slots: the keyed slot in 4 or 8 bytes, for order-preserving tables (mode 2) ---------------------------------------------
// Under mode 2 a key in line L is kmin + (L << shift) + r, with r in [0, 2^shift) in its home line and a small negative r after it was
// displaced to a later line: the slot stores krel = key - kmin - ((slot >> 3) << shift).  The payload cell is stored relative to the smallest
// cell of the table, cmin (the cells sign-extended from their width; a DOUBLE by its bits).  The build picks the narrowest of the two that
// holds every occupied slot's krel and cell, else it keeps the 16-byte keyed slot.  Empty is krel = INT16_MIN / INT32_MIN, which no stored
// key uses.  The probe compares the full 64-bit rel = k - kmin - ((pos >> 3) << shift) of an OCCUPIED slot with its sign-extended krel: for a
// fixed slot rel is a bijection of the key (mod 2^64), so only the stored key matches, also against a key that reaches the same slot through
// the wrap of the slot mask.  An empty slot is excluded explicitly (slot_matches): a probe key whose rel equals the empty marker exists
// whenever the lines cover few enough key values.  The payload is cmin + cell (mod 2^64), truncated to the column's width by the store.
struct __align__(4) PackedSlot4 {
    static constexpr int CELLS = 1;
    static constexpr bool LINE_RELATIVE = true;
    static constexpr long long KREL_MIN = INT16_MIN, KREL_MAX = INT16_MAX;
    static constexpr unsigned long long CELL_MAX = 0xFFFFULL;
    short krel;
    unsigned short cell;
};

struct __align__(8) PackedSlot8 {
    static constexpr int CELLS = 1;
    static constexpr bool LINE_RELATIVE = true;
    static constexpr long long KREL_MIN = INT32_MIN, KREL_MAX = INT32_MAX;
    static constexpr unsigned long long CELL_MAX = 0xFFFFFFFFULL;
    int krel;
    unsigned int cell;
};

// sm_90 has no 256-bit load: a wide slot is read as the two 128-bit halves of its 32-byte sector, which costs one DRAM sector all the same.
// LD: 0 = plain read-only loads; 3 = the same with an explicit 64-byte L2 fetch size
template <int LD>
__device__ __forceinline__ WideSlot slot_load(const WideSlot* p)
{
    WideSlot w;
    unsigned long long kh;
    if (LD == 3) {
        asm("ld.global.nc.L2::64B.v2.u64 {%0,%1}, [%2];" : "=l"(w.key), "=l"(kh) : "l"(p));
        asm("ld.global.nc.L2::64B.v2.u64 {%0,%1}, [%2+16];" : "=l"(w.cell[0]), "=l"(w.cell[1]) : "l"(p));
    }
    else {
        asm("ld.global.nc.v2.u64 {%0,%1}, [%2];" : "=l"(w.key), "=l"(kh) : "l"(p));
        asm("ld.global.nc.v2.u64 {%0,%1}, [%2+16];" : "=l"(w.cell[0]), "=l"(w.cell[1]) : "l"(p));
    }
    w.head = (int)(unsigned int)kh;
    w.pad = 0;
    return w;
}

template <int LD>
__device__ __forceinline__ KeyedSlot slot_load(const KeyedSlot* p)
{
    KeyedSlot w;
    if (LD == 3) asm("ld.global.nc.L2::64B.v2.u64 {%0,%1}, [%2];" : "=l"(w.key), "=l"(w.cell) : "l"(p));
    else asm("ld.global.nc.v2.u64 {%0,%1}, [%2];" : "=l"(w.key), "=l"(w.cell) : "l"(p));
    return w;
}

template <int LD>
__device__ __forceinline__ PackedSlot8 slot_load(const PackedSlot8* p)
{
    PackedSlot8 w;
    if (LD == 3) asm("ld.global.nc.L2::64B.v2.u32 {%0,%1}, [%2];" : "=r"(w.krel), "=r"(w.cell) : "l"(p));
    else asm("ld.global.nc.v2.u32 {%0,%1}, [%2];" : "=r"(w.krel), "=r"(w.cell) : "l"(p));
    return w;
}

template <int LD>
__device__ __forceinline__ PackedSlot4 slot_load(const PackedSlot4* p)
{
    unsigned int v;
    if (LD == 3) asm("ld.global.nc.L2::64B.u32 %0, [%1];" : "=r"(v) : "l"(p));
    else asm("ld.global.nc.u32 %0, [%1];" : "=r"(v) : "l"(p));
    PackedSlot4 w;
    w.krel = (short)(v & 0xFFFFu);
    w.cell = (unsigned short)(v >> 16);
    return w;
}

__device__ __forceinline__ bool slot_empty(const WideSlot& w) { return w.key == EMPTY_KEY; }
__device__ __forceinline__ bool slot_empty(const KeyedSlot& w) { return w.key == EMPTY_KEY; }
__device__ __forceinline__ bool slot_empty(const PackedSlot4& w) { return w.krel == INT16_MIN; }
__device__ __forceinline__ bool slot_empty(const PackedSlot8& w) { return w.krel == INT32_MIN; }

// does the slot at pos hold key k (kmin, shift: the mode 2 geometry; only line-relative slots need them)
__device__ __forceinline__ bool slot_matches(const WideSlot& w, unsigned long long k, unsigned int, unsigned long long, int) { return w.key == k; }
__device__ __forceinline__ bool slot_matches(const KeyedSlot& w, unsigned long long k, unsigned int, unsigned long long, int) { return w.key == k; }
// An empty packed slot never matches: its krel (INT16_MIN / INT32_MIN) is not a stored key's, but a probe key can have exactly that rel
// (e.g. k = kmin - 2^15 + (L << shift) in line L when the lines cover at most 2^15 key values)
template <class S>
__device__ __forceinline__ bool slot_matches(const S& w, unsigned long long k, unsigned int pos, unsigned long long kmin, int shift)
{
    const unsigned long long rel = k - kmin - ((unsigned long long)(pos >> 3) << shift);
    return (long long)rel == (long long)w.krel && !slot_empty(w);
}

// head row of a slot whose key matched (a keyed slot has none: any non-negative value stands for "matched")
__device__ __forceinline__ int slot_head(const WideSlot& w) { return w.head; }
template <class S>
__device__ __forceinline__ int slot_head(const S&) { return 0; }

// payload cell c of a matched slot (cmin: the packed slots' cell offset)
__device__ __forceinline__ unsigned long long slot_value(const WideSlot& w, int c, unsigned long long) { return w.cell[c]; }
__device__ __forceinline__ unsigned long long slot_value(const KeyedSlot& w, int, unsigned long long) { return w.cell; }
template <class S>
__device__ __forceinline__ unsigned long long slot_value(const S& w, int, unsigned long long cmin) { return cmin + (unsigned long long)w.cell; }

__device__ __forceinline__ void put_slot(WideSlot* s, unsigned long long key, int head, unsigned long long c0, unsigned long long c1)
{
    WideSlot w;
    w.key = key;
    w.head = head;
    w.pad = 0;
    w.cell[0] = c0;
    w.cell[1] = c1;
    *s = w;
}
__device__ __forceinline__ void put_slot(KeyedSlot* s, unsigned long long key, int, unsigned long long c0, unsigned long long)
{
    KeyedSlot w;
    w.key = key;
    w.cell = c0;
    *s = w;
}

__device__ __forceinline__ unsigned long long wide_cell_of(const void* src, int elem, int row)
{
    switch (elem) {
        case 8: return ((const unsigned long long*)src)[row];
        case 4: return ((const unsigned int*)src)[row];
        case 2: return ((const unsigned short*)src)[row];
        default: return ((const unsigned char*)src)[row];
    }
}

// S = WideSlot (cells of up to two columns) or KeyedSlot (one column); slot i < slots mirrors the 16-byte table, slot `slots` holds INT64_MIN's
template <class S>
__global__ void join_wide_table_kernel(const JoinSlot* __restrict__ table, int64_t slots, int special_head, const void* __restrict__ src0, int elem0,
                                       const void* __restrict__ src1, int elem1, S* __restrict__ wide)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i <= slots; i += stride) {
        const unsigned long long key = i < slots ? table[i].key : EMPTY_KEY;
        const int head = i < slots ? table[i].head : special_head;
        put_slot(wide + i, key, head, head >= 0 && src0 ? wide_cell_of(src0, elem0, head) : 0ULL, head >= 0 && src1 ? wide_cell_of(src1, elem1, head) : 0ULL);
    }
}

// a payload cell as a signed 64-bit value: sign-extended from its width, so that small negative integers stay a small range
__device__ __forceinline__ long long cell_sext(const void* src, int elem, int row)
{
    switch (elem) {
        case 8: return ((const long long*)src)[row];
        case 4: return ((const int*)src)[row];
        case 2: return ((const short*)src)[row];
        default: return ((const signed char*)src)[row];
    }
}

// which packed slot holds the keyed table of a mode 2 build: min / max of krel over the occupied slots, and of the cell over the occupied
// slots and INT64_MIN's (special_head >= 0).  range: {krel min, krel max, cell min, cell max}, initialised to empty ranges
__global__ void join_packed_range_kernel(const JoinSlot* __restrict__ table, int64_t slots, unsigned long long kmin, int shift, int special_head,
                                         const void* __restrict__ src, int elem, long long* __restrict__ range)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    long long klo = INT64_MAX, khi = INT64_MIN, clo = INT64_MAX, chi = INT64_MIN;
    for (; i <= slots; i += stride) {
        int head = special_head;
        if (i < slots) {
            const unsigned long long key = table[i].key;
            if (key == EMPTY_KEY) continue;
            const long long krel = (long long)(key - kmin - ((unsigned long long)(i >> 3) << shift));
            klo = min(klo, krel);
            khi = max(khi, krel);
            head = table[i].head;
        }
        if (head < 0) continue;
        const long long c = cell_sext(src, elem, head);
        clo = min(clo, c);
        chi = max(chi, c);
    }
    for (int off = 16; off > 0; off >>= 1) {
        klo = min(klo, (long long)__shfl_xor_sync(0xffffffffu, klo, off));
        khi = max(khi, (long long)__shfl_xor_sync(0xffffffffu, khi, off));
        clo = min(clo, (long long)__shfl_xor_sync(0xffffffffu, clo, off));
        chi = max(chi, (long long)__shfl_xor_sync(0xffffffffu, chi, off));
    }
    if ((threadIdx.x & 31) == 0) {
        if (klo <= khi) { atomicMin(range, klo); atomicMax(range + 1, khi); }
        if (clo <= chi) { atomicMin(range + 2, clo); atomicMax(range + 3, chi); }
    }
}

// the packed table: slot i < slots from the 16-byte table, slot `slots` holds INT64_MIN's cell (as join_wide_table_kernel)
template <class S>
__global__ void join_packed_table_kernel(const JoinSlot* __restrict__ table, int64_t slots, unsigned long long kmin, int shift, int special_head,
                                         const void* __restrict__ src, int elem, unsigned long long cmin, S* __restrict__ packed)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i <= slots; i += stride) {
        const unsigned long long key = i < slots ? table[i].key : EMPTY_KEY;
        const int head = i < slots ? table[i].head : special_head;
        S w;
        w.krel = key == EMPTY_KEY ? (decltype(w.krel))S::KREL_MIN : (decltype(w.krel))(long long)(key - kmin - ((unsigned long long)(i >> 3) << shift));
        w.cell = head >= 0 ? (decltype(w.cell))((unsigned long long)cell_sext(src, elem, head) - cmin) : 0;
        packed[i] = w;
    }
}

// same contract as join_probe_lean_kernel<MODE, true>: whole 1024-row tiles of a BIGINT key without NULLs; ROWS rows of a thread are in
// flight together (a tile is 4 rows per thread, taken ROWS at a time).  S is the slot type of the table (WideSlot, KeyedSlot, or under
// MODE 2 a packed slot, whose cells are relative to cmin).  With layout_choice set the kernel runs only when join_probe_locality_kernel
// chose run_on for the page.
template <int MODE, int ROWS, int MINB, int LD, class S>
__global__ void __launch_bounds__(256, MINB) join_probe_wide_kernel(const long long* __restrict__ keys, int64_t tiles, const S* __restrict__ wide, unsigned int mask,
                                                                  unsigned long long kmin, int shift, int special_head, unsigned long long cmin,
                                                                  unsigned int* __restrict__ match_bits, GatherCols g, unsigned long long* __restrict__ match_count,
                                                                  const int* __restrict__ layout_choice, int run_on)
{
    static_assert(MODE == 2 || !S::LINE_RELATIVE, "packed slots need order-preserving lines");
    if (layout_choice && *layout_choice != run_on) return;
    unsigned int matched = 0;
    for (int64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
#pragma unroll
        for (int h = 0; h < 4; h += ROWS) {
            const int64_t base = t * 1024 + h * 256 + threadIdx.x;
            unsigned long long k[ROWS];
            unsigned int pos[ROWS];
            S w[ROWS];
            bool hit[ROWS];
#pragma unroll
            for (int j = 0; j < ROWS; j++) k[j] = (unsigned long long)__ldg(keys + base + j * 256);
#pragma unroll
            for (int j = 0; j < ROWS; j++) pos[j] = lean_slot<MODE>(k[j], mask, kmin, shift);
#pragma unroll
            for (int j = 0; j < ROWS; j++) w[j] = slot_load<LD>(wide + pos[j]);
#pragma unroll
            for (int j = 0; j < ROWS; j++) {
                unsigned int p = pos[j];
                int r = -1;
                while (true) {
                    if (slot_matches(w[j], k[j], p, kmin, shift)) { r = slot_head(w[j]); break; }
                    if (slot_empty(w[j])) break;
                    p = lean_next<MODE>(p, (unsigned int)k[j] & 7u, mask);
                    w[j] = slot_load<LD>(wide + p);
                }
                if (k[j] == EMPTY_KEY) {                       // INT64_MIN lives outside the table, in the slot behind the last one
                    r = special_head;
                    if (r >= 0) w[j] = slot_load<LD>(wide + (mask + 1u));
                }
                hit[j] = r >= 0;
            }
#pragma unroll
            for (int c = 0; c < S::CELLS; c++) {
                if (c >= g.count) break;
#pragma unroll
                for (int j = 0; j < ROWS; j++) {
                    const unsigned long long v = hit[j] ? slot_value(w[j], c, cmin) : 0ULL;
                    switch (g.elem[c]) {
                        case 8: ((unsigned long long*)g.dst[c])[base + j * 256] = v; break;
                        case 4: ((unsigned int*)g.dst[c])[base + j * 256] = (unsigned int)v; break;
                        case 2: ((unsigned short*)g.dst[c])[base + j * 256] = (unsigned short)v; break;
                        default: ((unsigned char*)g.dst[c])[base + j * 256] = (unsigned char)v; break;
                    }
                }
            }
#pragma unroll
            for (int j = 0; j < ROWS; j++) store_match_word(match_bits, base + j * 256, hit[j], &matched);
        }
    }
    add_match_count(match_count, matched);
}

// Which layout a probe page should read.  A wide slot is 32 bytes, a 16-byte slot plus its slot-ordered payload cells 16 + (payload bytes):
// with one payload column a probe page that arrives in key order reads fewer bytes from the narrow layout (whole lines are used either
// way), while a page without key locality pays a 32-byte sector per ARRAY it touches and is better off with the wide slot.  256 pairs of
// neighbouring rows, spread over the page, vote: a pair is local when its two slots lie within 8 lines of each other.
// choice: 0 = key-ordered (the 16-byte slots, or the keyed table in the lean kernel's 4-row shape), 1 = random access (the wide table, or
// the keyed table in the random-access shape).  No host round trip: both probe kernels are launched and the one not chosen returns at once.
template <int MODE>
__global__ void __launch_bounds__(256) join_probe_locality_kernel(const long long* __restrict__ keys, int64_t tiles, unsigned int mask, unsigned long long kmin, int shift,
                                                                  int* __restrict__ layout_choice)
{
    const int64_t at = (tiles * (int64_t)threadIdx.x / 256) * 1024 + (threadIdx.x & 31) * 32;
    const unsigned int a = lean_slot<MODE>((unsigned long long)__ldg(keys + at), mask, kmin, shift);
    const unsigned int b = lean_slot<MODE>((unsigned long long)__ldg(keys + at + 1), mask, kmin, shift);
    const unsigned int d = a > b ? a - b : b - a;
    const int local = __syncthreads_count(d <= 64u);
    if (threadIdx.x == 0) *layout_choice = local * 2 >= 256 ? 0 : 1;
}

static int launch_locality(tgpu_ctx* ctx, const JoinGeom& geo, const long long* keys, int64_t tiles, int* layout_choice)
{
    const unsigned int mask32 = (unsigned int)geo.mask;
    if (geo.mode == 2) TG_LAUNCH(ctx, join_probe_locality_kernel<2>, 1, 256, 0, keys, tiles, mask32, geo.kmin, geo.shift, layout_choice);
    else if (geo.mode == 1) TG_LAUNCH(ctx, join_probe_locality_kernel<1>, 1, 256, 0, keys, tiles, mask32, 0ULL, 0, layout_choice);
    else TG_LAUNCH(ctx, join_probe_locality_kernel<0>, 1, 256, 0, keys, tiles, mask32, 0ULL, 0, layout_choice);
    return TGPU_OK;
}

template <int ROWS, int MINB, int LD = 0, class S>
static int launch_wide_shape(tgpu_ctx* ctx, const JoinGeom& geo, const long long* keys, int64_t tiles, const S* wide, int special_head, unsigned long long cmin,
                             unsigned int* match_bits, const GatherCols& g, unsigned long long* matches, const int* layout_choice, int run_on)
{
    const unsigned int mask32 = (unsigned int)geo.mask;
    if (geo.mode == 2) {
        auto k = join_probe_wide_kernel<2, ROWS, MINB, LD, S>;
        TG_LAUNCH(ctx, k, lean_grid(ctx, k, tiles), 256, 0, keys, tiles, wide, mask32, geo.kmin, geo.shift, special_head, cmin, match_bits, g, matches,
                  layout_choice, run_on);
        return TGPU_OK;
    }
    if constexpr (S::LINE_RELATIVE) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "packed join slots need order-preserving lines");
    else {
        if (geo.mode == 1) {
            auto k = join_probe_wide_kernel<1, ROWS, MINB, LD, S>;
            TG_LAUNCH(ctx, k, lean_grid(ctx, k, tiles), 256, 0, keys, tiles, wide, mask32, 0ULL, 0, special_head, cmin, match_bits, g, matches, layout_choice, run_on);
        }
        else {
            auto k = join_probe_wide_kernel<0, ROWS, MINB, LD, S>;
            TG_LAUNCH(ctx, k, lean_grid(ctx, k, tiles), 256, 0, keys, tiles, wide, mask32, 0ULL, 0, special_head, cmin, match_bits, g, matches, layout_choice, run_on);
        }
        return TGPU_OK;
    }
}

// Random-access shape of the probe over a wide, keyed or packed table (runs when layout_choice is null or 1).
// rows in flight per thread x CTAs per SM; TGPU_JOIN_WIDE_SHAPE=<rows><ctas> picks one of the built shapes (sweeps)
template <class S>
static int launch_wide(tgpu_ctx* ctx, const JoinGeom& geo, const long long* keys, int64_t tiles, const S* wide, int special_head, unsigned long long cmin,
                       unsigned int* match_bits, const GatherCols& g, unsigned long long* matches, const int* layout_choice)
{
    const char* e = getenv("TGPU_JOIN_WIDE_SHAPE");
    int shape = e ? atoi(e) : 28;
    const char* le = getenv("TGPU_JOIN_WIDE_LOAD");
    int ld = le ? atoi(le) : 3;
    if (shape == 28 && ld == 3) return launch_wide_shape<2, 8, 3>(ctx, geo, keys, tiles, wide, special_head, cmin, match_bits, g, matches, layout_choice, 1);
    switch (shape) {
        case 18: return launch_wide_shape<1, 8>(ctx, geo, keys, tiles, wide, special_head, cmin, match_bits, g, matches, layout_choice, 1);
        case 26: return launch_wide_shape<2, 6>(ctx, geo, keys, tiles, wide, special_head, cmin, match_bits, g, matches, layout_choice, 1);
        case 45: return launch_wide_shape<4, 5>(ctx, geo, keys, tiles, wide, special_head, cmin, match_bits, g, matches, layout_choice, 1);
        case 44: return launch_wide_shape<4, 4>(ctx, geo, keys, tiles, wide, special_head, cmin, match_bits, g, matches, layout_choice, 1);
        default: return launch_wide_shape<2, 8>(ctx, geo, keys, tiles, wide, special_head, cmin, match_bits, g, matches, layout_choice, 1);
    }
}

// ---- pipelined key-ordered probe over the keyed table (mode 2) -------------------------------------------------------------------------
// A key-ordered page moves only the bytes it must: its keys in, the payload out, every table line once.  The thread-per-row kernel
// (join_probe_wide_kernel<2,2,8,0,KeyedSlot>) reaches 0.88 of a device copy's bandwidth on these bytes, and more rows per thread do not
// change that (2048 to 5120 rows in flight per SM: the same time from 3072 on).  What does is taking the reads off the threads: bulk copies
// of whole tiles are long sequential DRAM requests, where each thread otherwise loads its keys, waits, loads the dependent slots and waits
// again before it stores.  One producer warp per CTA bulk-copies (cp.async.bulk, completion on an mbarrier) the keys of the CTA's tiles
// into a ring of KP_STAGES shared-memory buffers.  As soon as the keys of a tile have landed it computes the span of order-preserving
// table lines they fall in (a key-ordered tile touches one short run of lines: about 33 for lineitem against orders) and copies that
// span, plus the line behind it for walks that overflow their home line, into one of two line buffers.  Meanwhile 8 consumer warps
// resolve the tile before it from shared memory and store payload and match bits, so the line copy of tile i + 1 overlaps the work on
// tile i.  Staging the lines as well as the keys is worth it: the same ring with slots loaded per row was about 1 % slower.  A tile whose span
// exceeds SPAN_LINES lines (keys far outside the build range, a page that is not key-ordered after all) reads its slots from global
// memory, and so does a line walk that leaves the staged span.  Rows per thread and the order of tiles over the CTAs are those of the
// other probe kernels: payload stores and match words are coalesced the same way, and neighbouring tiles run at the same time, so a
// line two tiles share is usually an L2 hit.
constexpr int KP_THREADS = 288;          // 8 consumer warps (rows threadIdx.x + j * 256, as in the other kernels) + 1 producer warp
constexpr int KP_STAGES = 2;             // key tiles in the ring (2, 3 and 4 measured: 2 is as fast and needs the least shared memory)
constexpr int KP_CTAS = 4;               // CTAs per SM: 4 x 288 threads, <= 56 registers (5 CTAs at <= 40 registers is slower)

// S: KeyedSlot or a packed slot (a line of 128, 64 or 32 bytes: the bulk copies stay multiples of 16 bytes)
template <class S>
struct KeyedPipeSmem {
    long long keys[KP_STAGES][1024];
    S lines[2][SPAN_LINES * 8];
    unsigned long long key_full[KP_STAGES], key_empty[KP_STAGES], line_full[2], line_empty[2];
    unsigned int first_line[2], staged_lines[2];      // staged_lines 0: the tile's slots are read from global memory
};

template <class S>
__global__ void __launch_bounds__(KP_THREADS, KP_CTAS) join_probe_keyed_pipe_kernel(const long long* __restrict__ keys, int64_t tiles, const S* __restrict__ keyed,
                                                                              unsigned int mask, unsigned long long kmin, int shift, int special_head,
                                                                              unsigned long long cmin, unsigned int* __restrict__ match_bits, GatherCols g,
                                                                              unsigned long long* __restrict__ match_count, const int* __restrict__ layout_choice)
{
    constexpr unsigned int LINE_BYTES = 8 * sizeof(S);
    static_assert(LINE_BYTES % 16 == 0, "bulk copies move multiples of 16 bytes");
    if (layout_choice && *layout_choice != 0) return;
    extern __shared__ __align__(128) unsigned char kp_smem[];
    KeyedPipeSmem<S>& sm = *reinterpret_cast<KeyedPipeSmem<S>*>(kp_smem);
    const int lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int s = 0; s < KP_STAGES; s++) {
            mbar_init(&sm.key_full[s], 1);
            mbar_init(&sm.key_empty[s], 8);            // one arrival per consumer warp
        }
        for (int b = 0; b < 2; b++) {
            mbar_init(&sm.line_full[b], 1);
            mbar_init(&sm.line_empty[b], 8);
        }
    }
    __syncthreads();
    const int64_t my_tiles = (tiles - 1 - blockIdx.x) / gridDim.x + 1;      // the grid is at most `tiles` CTAs: each has one or more
    if (threadIdx.x >= 256) {
        // producer warp.  Tile i of the CTA is tile blockIdx.x + i * gridDim.x of the page; its keys go to stage i % KP_STAGES, its lines to
        // buffer i & 1.  Key copies run up to KP_STAGES tiles ahead of the span; a stage is refilled once the consumers released it.
        const unsigned int line_mask = mask >> 3;
        if (lane == 0)
            for (int64_t i = 0; i < KP_STAGES && i < my_tiles; i++) {
                mbar_expect_tx(&sm.key_full[i], 8192u);
                bulk_g2s(sm.keys[i], keys + (blockIdx.x + i * gridDim.x) * 1024, 8192u, &sm.key_full[i]);
            }
        for (int64_t i = 0; i < my_tiles; i++) {
            const int s = (int)(i % KP_STAGES), b = (int)(i & 1);
            mbar_wait(&sm.key_full[s], (unsigned int)(i / KP_STAGES) & 1u);
            unsigned int lo = 0xffffffffu, hi = 0;
#pragma unroll 8
            for (int m = 0; m < 32; m++) {
                const unsigned int line = lean_slot<2>((unsigned long long)sm.keys[s][m * 32 + lane], mask, kmin, shift) >> 3;
                lo = min(lo, line);
                hi = max(hi, line);
            }
            lo = __reduce_min_sync(0xffffffffu, lo);
            hi = __reduce_max_sync(0xffffffffu, hi);
            if (lane == 0) {
                if (i >= 2) mbar_wait(&sm.line_empty[b], (unsigned int)((i - 2) >> 1) & 1u);     // the consumers are done with tile i - 2
                const unsigned int lines = min(hi + 1u, line_mask) - lo + 1u;
                sm.first_line[b] = lo;
                sm.staged_lines[b] = lines <= (unsigned int)SPAN_LINES ? lines : 0u;
                if (lines <= (unsigned int)SPAN_LINES) {
                    mbar_expect_tx(&sm.line_full[b], lines * LINE_BYTES);
                    bulk_g2s(sm.lines[b], keyed + (size_t)lo * 8, lines * LINE_BYTES, &sm.line_full[b]);
                }
                else mbar_arrive(&sm.line_full[b]);
            }
            // refill the stage of tile i - 1 with tile i - 1 + KP_STAGES
            const int64_t next = i - 1 + KP_STAGES;
            if (lane == 0 && i >= 1 && next < my_tiles) {
                const int sn = (int)((i - 1) % KP_STAGES);
                mbar_wait(&sm.key_empty[sn], (unsigned int)((i - 1) / KP_STAGES) & 1u);
                mbar_expect_tx(&sm.key_full[sn], 8192u);
                bulk_g2s(sm.keys[sn], keys + (blockIdx.x + next * gridDim.x) * 1024, 8192u, &sm.key_full[sn]);
            }
            __syncwarp();
        }
        return;
    }
    unsigned int matched = 0;
    for (int64_t i = 0; i < my_tiles; i++) {
        const int s = (int)(i % KP_STAGES), b = (int)(i & 1);
        const int64_t base = (blockIdx.x + i * gridDim.x) * 1024 + threadIdx.x;
        mbar_wait(&sm.key_full[s], (unsigned int)(i / KP_STAGES) & 1u);
        mbar_wait(&sm.line_full[b], (unsigned int)(i >> 1) & 1u);
        const unsigned int first_slot = sm.first_line[b] << 3, staged_slots = sm.staged_lines[b] << 3;
        unsigned long long k[4];
        unsigned int pos[4];
        S w[4];
        bool hit[4];
#pragma unroll
        for (int j = 0; j < 4; j++) {
            k[j] = (unsigned long long)sm.keys[s][threadIdx.x + j * 256];
            pos[j] = lean_slot<2>(k[j], mask, kmin, shift);
        }
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const unsigned int local = pos[j] - first_slot;
            w[j] = local < staged_slots ? sm.lines[b][local] : slot_load<0>(keyed + pos[j]);
        }
#pragma unroll
        for (int j = 0; j < 4; j++) {
            unsigned int p = pos[j];
            hit[j] = false;
            while (true) {
                if (slot_matches(w[j], k[j], p, kmin, shift)) { hit[j] = true; break; }
                if (slot_empty(w[j])) break;
                p = lean_next<2>(p, (unsigned int)k[j] & 7u, mask);
                const unsigned int local = p - first_slot;
                w[j] = local < staged_slots ? sm.lines[b][local] : slot_load<0>(keyed + p);
            }
            if (k[j] == EMPTY_KEY) {                       // INT64_MIN lives outside the table, in the slot behind the last one
                hit[j] = special_head >= 0;
                if (hit[j]) w[j] = slot_load<0>(keyed + (mask + 1u));
            }
        }
        // the warp is done with the tile's keys and lines: hand them back to the producer before the stores
        __syncwarp();
        if (lane == 0) {
            mbar_arrive(&sm.key_empty[s]);
            mbar_arrive(&sm.line_empty[b]);
        }
        if (g.count > 0) {
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const unsigned long long v = hit[j] ? slot_value(w[j], 0, cmin) : 0ULL;
                switch (g.elem[0]) {
                    case 8: ((unsigned long long*)g.dst[0])[base + j * 256] = v; break;
                    case 4: ((unsigned int*)g.dst[0])[base + j * 256] = (unsigned int)v; break;
                    case 2: ((unsigned short*)g.dst[0])[base + j * 256] = (unsigned short)v; break;
                    default: ((unsigned char*)g.dst[0])[base + j * 256] = (unsigned char)v; break;
                }
            }
        }
#pragma unroll
        for (int j = 0; j < 4; j++) store_match_word(match_bits, base + j * 256, hit[j], &matched);
    }
    add_match_count(match_count, matched);
}

// Key-ordered shape of the probe over a keyed table (runs when layout_choice is 0): the pipelined kernel above for order-preserving tables
// and key columns whose tiles the bulk copy can read (16-byte aligned).  Otherwise 8 CTAs per SM and plain read-only loads like the lean
// kernel, but 2 rows in flight per thread rather than 4: four keyed rows do not fit the 32 registers that 8 CTAs per SM allow (ptxas spills
// 88-144 bytes per thread), two take 28-30 registers without spilling
template <class S>
static int launch_keyed_ordered(tgpu_ctx* ctx, const JoinGeom& geo, const long long* keys, int64_t tiles, const S* keyed, int special_head,
                                unsigned long long cmin, unsigned int* match_bits, const GatherCols& g, unsigned long long* matches, const int* layout_choice)
{
    if (geo.mode == 2 && ((uintptr_t)keys & 15) == 0) {
        auto k = join_probe_keyed_pipe_kernel<S>;
        const int smem = (int)sizeof(KeyedPipeSmem<S>);
        TG_CUDA(ctx, cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        TG_LAUNCH(ctx, k, lean_grid(ctx, k, tiles, KP_THREADS, smem), KP_THREADS, smem, keys, tiles, keyed, (unsigned int)geo.mask, geo.kmin, geo.shift,
                  special_head, cmin, match_bits, g, matches, layout_choice);
        return TGPU_OK;
    }
    return launch_wide_shape<2, 8, 0>(ctx, geo, keys, tiles, keyed, special_head, cmin, match_bits, g, matches, layout_choice, 0);
}

// build payload re-laid out in SLOT order (one pass at build time): the fused probe then reads the payload right next
// to where it found the key instead of chasing the row id into the (arbitrarily ordered) build pages
__global__ void join_payload_by_slot_kernel(const JoinSlot* __restrict__ table, int64_t slots, int special_head, const void* __restrict__ src, int elem,
                                            void* __restrict__ dst)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i <= slots; i += stride) {
        int head = i < slots ? table[i].head : special_head;
        if (head < 0) continue;
        switch (elem) {
            case 8: ((long long*)dst)[i] = ((const long long*)src)[head]; break;
            case 4: ((int*)dst)[i] = ((const int*)src)[head]; break;
            case 2: ((short*)dst)[i] = ((const short*)src)[head]; break;
            default: ((signed char*)dst)[i] = ((const signed char*)src)[head]; break;
        }
    }
}

// --- duplicate chains -------------------------------------------------------------------------------
// sort key = (slot << 32 | row) for rows that are in the table; rows with NULL keys sort last
__global__ void join_slot_of_row_kernel(ColRef key, int kind, int64_t n, const JoinSlot* __restrict__ table, JoinGeom geo,
                                        unsigned long long special_slot, unsigned long long* __restrict__ out)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        unsigned long long k;
        unsigned long long slot = 0xFFFFFFFFULL;
        if (join_key(key, kind, i, &k)) {
            if (k == EMPTY_KEY) slot = special_slot;
            else {
                unsigned long long pos = join_slot_of(k, geo);
                while (table[pos].key != k) pos = join_next_slot(pos, k, geo);
                slot = pos;
            }
        }
        out[i] = (slot << 32) | (unsigned long long)(unsigned int)i;
    }
}

// after the sort rows of one key are adjacent in ascending row order: next(row) = previous row of the key
__global__ void join_links_kernel(const unsigned long long* __restrict__ sorted, int64_t n, int* __restrict__ links)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        unsigned long long cur = sorted[i];
        unsigned int slot = (unsigned int)(cur >> 32);
        int row = (int)(unsigned int)cur;
        int next = -1;
        if (slot != 0xFFFFFFFFu && i > 0) {
            unsigned long long prev = sorted[i - 1];
            if ((unsigned int)(prev >> 32) == slot) next = (int)(unsigned int)prev;
        }
        links[row] = next;
    }
}

// --- expansion --------------------------------------------------------------------------------------
__global__ void join_count_kernel(const int* __restrict__ jp, int64_t n, const int* __restrict__ links, int single_match, int outer,
                                  int* __restrict__ counts)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        int p = jp[i];
        int c = 0;
        if (p >= 0) {
            c = 1;
            if (links && !single_match) {
                p = links[p];
                while (p >= 0) { c++; p = links[p]; }
            }
        }
        else if (outer) c = 1;
        counts[i] = c;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) counts[n] = 0;
}

__global__ void join_fill_kernel(const int* __restrict__ jp, int64_t n, const int* __restrict__ links, int single_match, int outer,
                                 const long long* __restrict__ offsets, int* __restrict__ out_probe, int* __restrict__ out_build)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        int p = jp[i];
        long long o = offsets[i];
        if (p >= 0) {
            out_probe[o] = (int)i;
            out_build[o] = p;
            if (links && !single_match) {
                p = links[p];
                while (p >= 0) { o++; out_probe[o] = (int)i; out_build[o] = p; p = links[p]; }
            }
        }
        else if (outer) {
            out_probe[o] = (int)i;
            out_build[o] = -1;
        }
    }
}

// --- join filter function -----------------------------------------------------------------------------
// JoinFilterFunction.filter(leftPosition, rightPosition) (M/sql/gen/JoinFilterFunctionCompiler.java:94-131): the filter's channels are
// the join-sources layout.  DColumns slot c < nb holds build channel c, read at the build position; slot c >= nb holds probe channel
// c - nb, read at the probe row.  NULL or FALSE: the position is not eligible.
constexpr int JF_THREADS = 256;

__device__ __forceinline__ bool jf_eval(const DProgram* __restrict__ prog, const DColumns& cols, int nb, int64_t probe_row, int64_t build_pos,
                                        int64_t* temps, uint32_t* err)
{
    uint32_t te = 0;
    const uint32_t nulls = tg::vm_run(prog, 0, prog->num_filter_insns, cols, probe_row, temps, JF_THREADS, 0, &te, nb, build_pos);
    const int ft = prog->filter_temp;
    *err = tg::vm_temp_error(te, ft);
    return !((nulls >> ft) & 1) && temps[ft * JF_THREADS] != 0;
}

// lookup without position links: each probe row has at most one candidate; jp[i] = -1 where it is not eligible
__global__ void __launch_bounds__(JF_THREADS) join_filter_positions_kernel(const DProgram* __restrict__ prog, DColumns cols, int nb, int64_t n,
                                                                          int* __restrict__ jp, unsigned int* __restrict__ err_out)
{
    __shared__ int64_t temps[TGPU_MAX_TEMPS * JF_THREADS];
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    uint32_t err = 0;
    for (; i < n; i += stride) {
        const int b = jp[i];
        if (b < 0) continue;
        uint32_t e = 0;
        if (!jf_eval(prog, cols, nb, i, b, temps + threadIdx.x, &e)) jp[i] = -1;
        err |= e;
    }
    if (err) atomicOr(err_out, err);
}

// candidate pairs (probe row pp[k], build position pb[k]): verdict[k] = eligible | error bits << 1
__global__ void __launch_bounds__(JF_THREADS) join_filter_pairs_kernel(const DProgram* __restrict__ prog, DColumns cols, int nb, int64_t m,
                                                                      const int* __restrict__ pp, const int* __restrict__ pb, uint8_t* __restrict__ verdict)
{
    __shared__ int64_t temps[TGPU_MAX_TEMPS * JF_THREADS];
    int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; k < m; k += stride) {
        uint32_t e = 0;
        const bool ok = jf_eval(prog, cols, nb, pp[k], pb[k], temps + threadIdx.x, &e);
        verdict[k] = (uint8_t)((ok ? 1u : 0u) | (e << 1));
    }
}

// PageJoiner.joinCurrentPosition over the candidate pairs of probe row i, [off[i], off[i + 1]) in chain order: eligible pairs are kept,
// outputSingleMatch keeps the first one and evaluates no further pair; an outer join with no kept pair emits one NULL-build row
// (outerJoinCurrentPosition).  verdict[k] becomes 1 for the kept pairs; counts[i] = output rows of row i; the error bits of the
// evaluated pairs are or-ed into *err_out
__global__ void join_filter_select_kernel(const long long* __restrict__ off, int64_t n, int single_match, int outer, uint8_t* __restrict__ verdict,
                                          int* __restrict__ counts, unsigned int* __restrict__ err_out)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    uint32_t err = 0;
    for (; i < n; i += stride) {
        int kept = 0;
        bool done = false;
        for (long long k = off[i]; k < off[i + 1]; k++) {
            const uint8_t v = verdict[k];
            bool keep = false;
            if (!done) {
                err |= v >> 1;
                keep = v & 1;
                if (keep) { kept++; done = single_match != 0; }
            }
            verdict[k] = keep ? 1 : 0;
        }
        counts[i] = kept ? kept : (outer ? 1 : 0);
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) counts[n] = 0;
    if (err) atomicOr(err_out, err);
}

__global__ void join_filter_fill_kernel(const long long* __restrict__ off, int64_t n, const uint8_t* __restrict__ keep, const int* __restrict__ pb, int outer,
                                        const long long* __restrict__ out_off, int* __restrict__ out_probe, int* __restrict__ out_build)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        long long o = out_off[i];
        const long long first = o;
        for (long long k = off[i]; k < off[i + 1]; k++) {
            if (!keep[k]) continue;
            out_probe[o] = (int)i;
            out_build[o] = pb[k];
            o++;
        }
        if (o == first && outer) {
            out_probe[o] = (int)i;
            out_build[o] = -1;
        }
    }
}

// NVRTC form of the two evaluation kernels, specialised for one program over the given channel element sizes / nullability
std::string gen_join_filter_source(const DProgram& prog, int nb, const int* elems, int num_channels, uint32_t nullable_mask)
{
    std::string s, loads, temps;
    bool used[TGPU_MAX_CHANNELS] = {false};
    tg::fp_mark_columns(prog, 0, prog.num_filter_insns, used);
    for (int c = 0; c < num_channels && c < TGPU_MAX_CHANNELS; c++) {
        if (!used[c]) continue;
        const char* row = c < nb ? "b" : "p";
        tg::fp_appendf(loads, "    const long long c%d = tg_load_elem<%d>(cols.cols[%d].data, %s);", c, elems[c], c, row);
        if ((nullable_mask >> c) & 1) tg::fp_appendf(loads, " const bool c%dn = !tg_valid(cols.cols[%d].validity, %s);\n", c, c, row);
        else tg::fp_appendf(loads, " const bool c%dn = false;\n", c);
    }
    tg::fp_emit_temps(temps, prog);
    const int ft = prog.filter_temp;
    s += "struct JFProg {\n";
    s += "  static __device__ __forceinline__ bool eval(const DColumns& cols, long long p, long long b, unsigned int* errp) {\n";
    s += loads + temps;
    tg::fp_emit_insns(s, prog, 0, prog.num_filter_insns);
    tg::fp_appendf(s, "    *errp = te%d;\n    return !tn%d && t%d != 0;\n  }\n};\n", ft, ft, ft);
    s += "extern \"C\" __global__ void __launch_bounds__(256) tg_jf_positions_jit(DColumns cols, long long n, int* jp, unsigned int* err_out) {\n";
    s += "  unsigned int err = 0;\n  long long stride = (long long)gridDim.x * blockDim.x;\n";
    s += "  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {\n";
    s += "    const int b = jp[i];\n    if (b < 0) continue;\n    unsigned int e = 0;\n";
    s += "    if (!JFProg::eval(cols, i, b, &e)) jp[i] = -1;\n    err |= e;\n  }\n  if (err) atomicOr(err_out, err);\n}\n";
    s += "extern \"C\" __global__ void __launch_bounds__(256) tg_jf_pairs_jit(DColumns cols, long long m, const int* pp, const int* pb, unsigned char* verdict) {\n";
    s += "  long long stride = (long long)gridDim.x * blockDim.x;\n";
    s += "  for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < m; k += stride) {\n";
    s += "    unsigned int e = 0;\n    const bool ok = JFProg::eval(cols, pp[k], pb[k], &e);\n";
    s += "    verdict[k] = (unsigned char)((ok ? 1u : 0u) | (e << 1));\n  }\n}\n";
    return s;
}

// validate a join filter program (HashBuilderOperatorFactory's filterFunctionFactory) and flatten it
int join_filter_compile(tgpu_ctx* ctx, const tgpu_expr_program* program, int32_t num_build_channels, DProgram* out)
{
    if (!program) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "join filter program is null");
    if (program->num_projections != 0) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "a join filter program has no projections (got %d)", program->num_projections);
    if (program->filter_temp < 0) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "a join filter program needs a filter_temp");
    if (num_build_channels < 0) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "num_build_channels %d is negative", num_build_channels);
    int32_t max_channel = -1;
    TG_TRY(tg::expr_compile(ctx, program, out, &max_channel));
    if (tg::expr_uses_strings(*out)) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "join filters do not evaluate VARCHAR operations");
    if (tg::expr_uses_decimals(*out)) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "join filters do not evaluate DECIMAL operations");
    for (int i = 0; i < out->num_insns; i++)
        if (out->insns[i].op == TGPU_EX_IF || out->insns[i].op == TGPU_EX_COALESCE)
            return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "join filters do not evaluate IF or COALESCE");
    return TGPU_OK;
}

// a filter reads this channel as a value: only fixed-width integer / DOUBLE / BOOLEAN channels (as FilterAndProject)
bool join_filter_type_ok(const DevColumn& c) { return c.elem_size() != 0 && c.elem_size() != 16 && c.type != TGPU_FLOAT32; }

int key_kind_of(int type) { return type == TGPU_FLOAT64 ? KEY_DOUBLE : KEY_INT; }

// a probe channel can be looked up in a table keyed by one fixed-width channel: VARCHAR, long DECIMAL and REAL builds are generic
// lookups, so a probe channel of those types (read as 1- or 4-byte integers otherwise) never belongs to such a table
bool probe_key_fits_keyed_table(int probe_type, int build_type)
{
    if (probe_type == TGPU_UTF8 || probe_type == TGPU_INT128 || probe_type == TGPU_FLOAT32) return false;
    return key_kind_of(probe_type) == key_kind_of(build_type);
}

}  // namespace

// ------------------------------------------------------------------------------------------------
// LookupSource
// ------------------------------------------------------------------------------------------------
struct tgpu_lookup {
    tgpu_ctx* ctx = nullptr;
    int refs = 1;
    int64_t positions = 0;              // build rows (incl. NULL-key rows: PagesIndex keeps them)
    int key_type = 0;
    DevBuf table;                       // JoinSlot[capacity]
    JoinGeom geo = {0, 0, 0, 0};        // capacity - 1, slot placement mode and its parameters
    int special_head = -1;
    bool has_dups = false;
    DevBuf links;                       // int32[positions], only when has_dups
    DevPage store;                      // key column first, then build output columns
    int32_t num_output = 0;
    std::vector<DevBuf> by_slot;        // build output columns in table-slot order (fused probe fast path)
    DevBuf wide;                        // WideSlot[capacity + 1]: slots with the payload of their head row (2 build output columns)
    DevBuf keyed;                       // [capacity + 1] slots of keyed_bytes: key + payload cell (1 build output column; instead of `wide`)
    int keyed_bytes = 0;                // 16: KeyedSlot; 8 / 4: PackedSlot8 / PackedSlot4 (mode 2), cells relative to keyed_cmin
    unsigned long long keyed_cmin = 0;
    bool generic = false;               // keyed by row hash + verification against build_keys
    int attempts = 1;                   // generic only: hash functions the build needed (> 1 iff two keys shared a 64-bit hash)
    std::vector<DevColumn> build_keys;  // generic only: the real key columns of the build side
    // OuterPositionTracker (M/operator/join/OuterLookupSource.java:168-196): one byte per build position, set by the
    // LOOKUP_OUTER / FULL_OUTER probes for every build row they emit, read by the LookupOuterOperator
    DevBuf visited;
    std::mutex visited_lock;
    int64_t null_key_rows = -1;         // build rows whose (first) key channel is NULL; -1 = not counted yet
    int64_t nan_key_rows = -1;          // DOUBLE / REAL key: build rows whose key is NaN (members of a semi-join's ChannelSet); -1 = not counted yet
    // JoinFilterFunction (JoinHash.isJoinPositionEligible): the compiled filter over the join-sources layout [build channels, probe channels]
    bool has_filter = false;
    DProgram filter;                    // host copy (the NVRTC source is generated from it)
    DevBuf d_filter;                    // device copy (interpreter kernels)
    int32_t num_build_channels = 0;     // buildLayout.size(): layout channels below it are build channels
    std::vector<int32_t> filter_channels;   // layout channels the filter reads, ascending
    std::vector<DevColumn> filter_cols; // [num_build_channels]: the build channels the filter reads (shared with store / build_keys), others empty
    int64_t filter_extra_bytes = 0;     // device bytes of the filter's build channels kept for it alone
};

namespace {


// row-hash column (+ validity: NULL / NaN keys can never match) of a set of key columns
int make_fingerprint(tgpu_ctx* ctx, const std::vector<const DevColumn*>& keys, int64_t n, DevColumn* out, const uint8_t* d_attempt = nullptr)
{
    KeyCols k;
    memset(&k, 0, sizeof(k));
    if (keys.size() > (size_t)tg::MAX_KEY_COLS) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "more than %d join channels", tg::MAX_KEY_COLS);
    k.count = (int32_t)keys.size();
    for (size_t c = 0; c < keys.size(); c++) tg::key_cols_set(&k, (int)c, *keys[c]);
    DevColumn fp;
    fp.type = TGPU_INT64;
    fp.length = n;
    fp.own_data = std::make_shared<DevBuf>();
    TG_TRY(fp.own_data->alloc(ctx, (size_t)std::max<int64_t>(n, 1) * 8));
    fp.data = fp.own_data->p;
    DevBuf is_null;
    TG_TRY(is_null.alloc(ctx, (size_t)std::max<int64_t>(n, 1)));
    if (n > 0) {
        TG_LAUNCH(ctx, join_fingerprint_kernel, tg_grid(ctx, n, 256, 8), 256, 0, k, n, d_attempt, fp.own_data->as<long long>(), is_null.as<uint8_t>());
        tgpu_column bm;
        memset(&bm, 0, sizeof(bm));
        bm.type = TGPU_INT8;
        bm.flags = TGPU_COL_NULLS_BYTEMAP;
        bm.length = n;
        bm.data = is_null.p;
        bm.validity = is_null.as<uint8_t>();
        DevColumn packed;
        TG_TRY(tg_ingest_column(ctx, &bm, true, &packed));
        fp.own_validity = packed.own_validity;
        fp.validity = packed.validity;
    }
    *out = std::move(fp);
    return TGPU_OK;
}

KeyCols key_cols_of(const std::vector<DevColumn>& cols)
{
    KeyCols k;
    memset(&k, 0, sizeof(k));
    k.count = (int32_t)cols.size();
    for (size_t c = 0; c < cols.size(); c++) tg::key_cols_set(&k, (int)c, cols[c]);
    return k;
}

int lookup_positions(tgpu_ctx* ctx, const tgpu_lookup* lk, const DevColumn& key, int* d_out)
{
    int64_t n = key.length;
    if (n == 0) return TGPU_OK;
    if (lk->positions == 0) {      // nothing to match, and a build that never saw a page has no key type to compare with: every row misses
        TG_CUDA(ctx, cudaMemsetAsync(d_out, 0xFF, (size_t)n * 4, ctx->stream));
        return TGPU_OK;
    }
    if (!probe_key_fits_keyed_table(key.type, lk->key_type) || key.elem_size() == 0)
        return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "probe key type %d does not match build key type %d", key.type, lk->key_type);
    const JoinSlot* table = lk->table.as<JoinSlot>();
    bool fast = key.type == TGPU_INT64 && !key.validity;
    int kind = fast ? KEY_INT : key_kind_of(key.type);
    auto k4f = join_probe_kernel<4, true>;
    auto k4a = join_probe_kernel<4, false>;
    int64_t done = 0;
    TG_TIMED_BEGIN(ctx);
    if (fast && !getenv("TGPU_JOIN_GENERIC_KERNELS")) {
        // whole 1024-row tiles through the lean kernel, the ragged tail through the generic one
        int64_t tiles = n / 1024;
        if (tiles > 0) {
            GatherCols none;
            memset(&none, 0, sizeof(none));
            TG_TRY(launch_lean<false>(ctx, lk->geo, (const long long*)key.data, tiles, (const int4*)table, lk->special_head, d_out, nullptr, none,
                                      (unsigned long long*)nullptr));
            done = tiles * 1024;
        }
    }
    if (done < n) {
        ColRef kr = tg_colref(key);
        if (done > 0) kr.data = (const char*)kr.data + done * 8;   // only the fast (INT64, no validity) shape gets here with done > 0
        int grid = tg_grid(ctx, n - done, 256 * 4, 8);
        if (fast) TG_LAUNCH(ctx, k4f, grid, 256, 0, kr, kind, n - done, table, lk->geo, lk->special_head, d_out + done);
        else TG_LAUNCH(ctx, k4a, grid, 256, 0, kr, kind, n - done, table, lk->geo, lk->special_head, d_out + done);
    }
    TG_TIMED_END(ctx);
    return TGPU_OK;
}

// join positions for a generic-key lookup: probe the row hashes, then keep only hits whose key columns really match
int lookup_positions_generic(tgpu_ctx* ctx, const tgpu_lookup* lk, const std::vector<const DevColumn*>& keys, int64_t n, int* d_out)
{
    if (keys.size() != lk->build_keys.size()) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "probe has %zu join channels, build has %zu", keys.size(), lk->build_keys.size());
    // col_value_equal decides from the probe channel how both sides are read: VARCHAR, DOUBLE, REAL and long DECIMAL must agree per channel
    // (a 16-byte probe channel would read past the end of an 8-byte build column).  Integer channels of different widths compare by value,
    // each side read at its own width, as in a lookup keyed by one channel.  A build that never saw a page has no channel types and no row
    // to compare with: every probe row misses
    for (size_t c = 0; c < keys.size() && lk->positions > 0; c++) {
        const DevColumn &p = *keys[c], &b = lk->build_keys[c];
        bool same = (p.type == TGPU_UTF8) == (b.type == TGPU_UTF8) && (p.type == TGPU_FLOAT64) == (b.type == TGPU_FLOAT64) &&
                    (p.type == TGPU_FLOAT32) == (b.type == TGPU_FLOAT32) && (p.type == TGPU_INT128) == (b.type == TGPU_INT128);
        if (!same) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "join channel %zu: probe type %d does not match build type %d", c, p.type, b.type);
    }
    if (n == 0) return TGPU_OK;
    DevColumn fp;
    TG_TRY(make_fingerprint(ctx, keys, n, &fp));
    TG_TRY(lookup_positions(ctx, lk, fp, d_out));
    KeyCols pk;
    memset(&pk, 0, sizeof(pk));
    pk.count = (int32_t)keys.size();
    for (size_t c = 0; c < keys.size(); c++) tg::key_cols_set(&pk, (int)c, *keys[c]);
    const KeyCols bk = key_cols_of(lk->build_keys);
    TG_LAUNCH(ctx, join_verify_probe_kernel, tg_grid(ctx, n, 256, 8), 256, 0, pk, bk, n, lk->attempts > 1 ? 1 : 0, d_out);
    for (int a = 1; a < lk->attempts; a++)
        TG_LAUNCH(ctx, join_probe_retry_kernel, tg_grid(ctx, n, 256, 8), 256, 0, pk, bk, n, lk->table.as<JoinSlot>(), lk->geo, lk->special_head, a,
                  a == lk->attempts - 1 ? 1 : 0, d_out);
    return TGPU_OK;
}

// LookupSource.appendTo -> positionVisited for every build row an outer-tracking probe emitted
__global__ void join_mark_visited_kernel(const int* __restrict__ build_idx, int64_t n, uint8_t* __restrict__ visited)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        int b = build_idx[i];
        if (b >= 0) visited[b] = 1;
    }
}

__global__ void join_unvisited_flags_kernel(const uint8_t* __restrict__ visited, int64_t n, uint8_t* __restrict__ flags)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) flags[i] = visited[i] ? 0 : 1;
}

// HashSemiJoinOperator.process :181-199: value and NULL byte of the appended BOOLEAN column
// float_kind: 0 = not a floating-point key, 1 = DOUBLE, 2 = REAL.  The ChannelSet compares with IDENTICAL (M/operator/FlatSet.java:54,374): a NaN
// probe key is in the set iff the set holds a NaN - which the EQUAL-semantics lookup cannot answer (NaN matches nothing there) - while -0.0 / +0.0
// are one member under both
__device__ __forceinline__ bool key_is_nan(const ColRef& key, int float_kind, int64_t i)
{
    if (float_kind == 1) return ((unsigned long long)tg_load_i64(key, i) & 0x7FFFFFFFFFFFFFFFULL) > 0x7FF0000000000000ULL;
    if (float_kind == 2) return ((unsigned int)tg_load_i64(key, i) & 0x7FFFFFFFu) > 0x7F800000u;
    return false;
}

__global__ void count_nan_keys_kernel(ColRef key, int float_kind, int64_t n, unsigned long long* __restrict__ out)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    unsigned int mine = 0;
    for (; i < n; i += stride) mine += tg_valid(key.validity, i) && key_is_nan(key, float_kind, i);
    for (int off = 16; off > 0; off >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, off);
    if ((threadIdx.x & 31) == 0 && mine) atomicAdd(out, (unsigned long long)mine);
}

__global__ void semi_join_kernel(const int* __restrict__ positions, const uint8_t* __restrict__ key_validity, int64_t n, int set_empty, int set_has_null,
                                 signed char* __restrict__ value, uint8_t* __restrict__ is_null, ColRef key, int float_kind, int set_has_nan)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        bool probe_null = !tg_valid(key_validity, i);
        bool contains = positions[i] >= 0;
        if (float_kind && !probe_null && key_is_nan(key, float_kind, i)) contains = set_has_nan != 0;
        bool out_null, v;
        if (probe_null) { out_null = !set_empty; v = false; }
        else if (!contains && set_has_null) { out_null = true; v = false; }
        else { out_null = false; v = contains; }
        value[i] = v ? 1 : 0;
        is_null[i] = out_null ? 1 : 0;
    }
}

__global__ void count_nulls_kernel(const uint8_t* __restrict__ validity, int64_t n, unsigned long long* __restrict__ out)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    unsigned int c = 0;
    for (; i < n; i += stride) c += tg_valid(validity, i) ? 0 : 1;
    for (int off = 16; off > 0; off >>= 1) c += __shfl_xor_sync(0xffffffffu, c, off);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, (unsigned long long)c);
}

// DynamicFilterSourceOperator / JoinDomainBuilder: min, max, number of distinct keys and (while they fit) the keys themselves,
// read off the table (one occupied slot per distinct non-NULL key)
__global__ void join_key_domain_kernel(const JoinSlot* __restrict__ table, int64_t slots, int64_t max_values, long long* __restrict__ minmax /* [2] */,
                                       unsigned long long* __restrict__ count, long long* __restrict__ values)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < slots; i += stride) {
        long long k = table[i].key;
        if ((unsigned long long)k == EMPTY_KEY) continue;
        atomicMin(minmax, k);
        atomicMax(minmax + 1, k);
        unsigned long long at = atomicAdd(count, 1ULL);
        if ((long long)at < max_values) values[at] = k;
    }
}

// HashBuilderOperator: NEEDS_INPUT -> (finish) LOOKUP_SOURCE_BUILT -> CLOSED
struct JoinBuildOp : tgpu_op {
    std::vector<int32_t> key_channels, output_channels;
    std::vector<DevPage> chunks;     // key column + output columns (+ the filter's extra channels) of every input page
    std::vector<int32_t> col_types;  // types of [key, outputs..., extras...] as first seen (an empty build still needs them)
    // join filter function: the compiled program, buildLayout.size(), and the build channels it reads that are neither key nor output
    // channels (kept after the outputs in every chunk)
    bool has_filter = false;
    DProgram filter;
    int32_t num_build_channels = 0;
    std::vector<int32_t> filter_channels;   // layout channels the filter reads
    std::vector<int32_t> extra_channels;
    int64_t rows = 0;
    bool finishing = false;
    tgpu_lookup* lookup = nullptr;

    explicit JoinBuildOp(tgpu_ctx* c) : tgpu_op(c) {}
    ~JoinBuildOp() override { if (lookup) tgpu_lookup_release(lookup); }

    bool needs_input() override { return !finishing; }

    int add_input(const tgpu_page* page) override
    {
        // HashBuilderOperator.addInput :253-277 -> PagesIndex.addPage :224-256
        if (col_types.empty()) {
            auto type_of = [&](int32_t ch) -> int32_t {
                if (ch < 0 || ch >= page->num_columns) return 0;
                const tgpu_column* c = &page->columns[ch];
                while ((c->type == TGPU_DICT32 || c->type == TGPU_RLE) && c->dictionary) c = c->dictionary;
                return c->type;
            };
            for (int32_t ch : key_channels) col_types.push_back(type_of(ch));
            for (int32_t ch : output_channels) col_types.push_back(type_of(ch));
            for (int32_t ch : extra_channels) col_types.push_back(type_of(ch));
        }
        if (has_filter && page->num_columns != num_build_channels)
            return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "build page has %d channels, the join filter's build layout %d", page->num_columns, num_build_channels);
        if (page->num_rows == 0) return TGPU_OK;
        if (rows + page->num_rows > (int64_t)INT32_MAX)
            return tg_fail(ctx, TGPU_ERR_INSUFFICIENT_RESOURCES, "Size of pages index cannot exceed 2 billion entries");   // PagesIndex.java:247-250
        bool device = (page->flags & TGPU_PAGE_DEVICE) != 0;
        DevPage p;
        p.rows = page->num_rows;
        auto take = [&](int32_t ch) -> int {
            if (ch < 0 || ch >= page->num_columns) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "channel %d out of range", ch);
            DevColumn c;
            TG_TRY(tg_ingest_column(ctx, &page->columns[ch], device, &c));
            p.cols.push_back(std::move(c));
            return TGPU_OK;
        };
        for (int32_t ch : key_channels) TG_TRY(take(ch));
        for (int32_t ch : output_channels) TG_TRY(take(ch));
        for (int32_t ch : extra_channels) TG_TRY(take(ch));
        if (!device) TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        for (int32_t ch : filter_channels) {
            if (ch >= num_build_channels) break;
            const DevColumn& c = p.cols[kept_at(ch)];
            if (!join_filter_type_ok(c))
                return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "join filters over variable-width / 128-bit / REAL channel %d are not supported on the GPU path", ch);
        }
        rows += p.rows;
        chunks.push_back(std::move(p));
        return TGPU_OK;
    }

    // column of a chunk that holds build channel ch (the filter's build channels are kept once)
    size_t kept_at(int32_t ch) const
    {
        for (size_t b = 0; b < output_channels.size(); b++)
            if (output_channels[b] == ch) return key_channels.size() + b;
        for (size_t k = 0; k < key_channels.size(); k++)
            if (key_channels[k] == ch) return k;
        for (size_t e = 0; e < extra_channels.size(); e++)
            if (extra_channels[e] == ch) return key_channels.size() + output_channels.size() + e;
        return (size_t)-1;
    }

    int concat(DevPage* out)
    {
        if (chunks.size() == 1) { *out = std::move(chunks[0]); chunks.clear(); return TGPU_OK; }
        DevPage r;
        r.rows = rows;
        size_t ncols = key_channels.size() + output_channels.size() + extra_channels.size();
        r.cols.resize(ncols);
        for (size_t c = 0; c < ncols && !chunks.empty(); c++) {
            std::vector<const DevColumn*> parts;
            for (auto& ch : chunks) parts.push_back(&ch.cols[c]);
            TG_TRY(tg_concat_columns(ctx, parts, &r.cols[c]));
        }
        chunks.clear();
        *out = std::move(r);
        return TGPU_OK;
    }

    int finish() override
    {
        // HashBuilderOperator.finish :286-308 -> finishInput :310-333 -> PagesIndex.createLookupSourceSupplier :523-542
        if (finishing) return TGPU_OK;   // re-entrant
        std::unique_ptr<tgpu_lookup> lk(new tgpu_lookup());
        lk->ctx = ctx;
        lk->positions = rows;
        lk->num_output = (int32_t)output_channels.size();
        DevPage all;
        TG_TRY(concat(&all));
        const size_t nk = key_channels.size();
        if (rows == 0) {
            all.cols.resize(nk + output_channels.size() + extra_channels.size());
            for (size_t c = 0; c < all.cols.size(); c++) all.cols[c].type = c < col_types.size() && col_types[c] ? col_types[c] : TGPU_INT64;
        }
        // one fixed-width channel -> the table is keyed by the value itself; anything else -> by the row hash + verification
        lk->generic = nk != 1 || all.cols[0].type == TGPU_UTF8 || all.cols[0].type == TGPU_INT128 || all.cols[0].type == TGPU_FLOAT32;      // (no 64-bit canonical key; REAL keys compare as floats in rowkeys.cuh)
        lk->store.rows = rows;
        if (lk->generic) {
            for (size_t c = 0; c < nk; c++) lk->build_keys.push_back(all.cols[c]);
            std::vector<const DevColumn*> kp;
            for (auto& c : lk->build_keys) kp.push_back(&c);
            DevColumn fp;
            TG_TRY(make_fingerprint(ctx, kp, rows, &fp));
            lk->store.cols.push_back(std::move(fp));
        }
        else lk->store.cols.push_back(all.cols[0]);
        for (size_t c = nk; c < nk + output_channels.size(); c++) lk->store.cols.push_back(all.cols[c]);
        lk->key_type = lk->store.cols[0].type;
        if (has_filter) {
            lk->has_filter = true;
            lk->filter = filter;
            lk->num_build_channels = num_build_channels;
            lk->filter_channels = filter_channels;
            lk->filter_cols.resize(num_build_channels);
            for (int32_t ch : filter_channels)
                if (ch < num_build_channels) lk->filter_cols[ch] = all.cols[kept_at(ch)];     // shares the buffers
            for (size_t e = 0; e < extra_channels.size(); e++) lk->filter_extra_bytes += all.cols[nk + output_channels.size() + e].memory_bytes();
            TG_TRY(lk->d_filter.alloc(ctx, sizeof(DProgram)));
            TG_CUDA(ctx, cudaMemcpyAsync(lk->d_filter.p, &lk->filter, sizeof(DProgram), cudaMemcpyHostToDevice, ctx->stream));
        }
        int64_t cap = 0;
        auto build_table = [&]() -> int {
            // sizing: IncrementalLoadFactorHashArraySizeSupplier.getHashArraySize :40-47 (capacity is not observable)
            double lf = rows <= (1 << 16) ? 0.25 : rows <= (1 << 20) ? 0.5 : 0.75;
            int64_t need = (int64_t)((double)rows / lf) + 1;
            cap = 8;   // at least one 8-slot line
            while (cap < need) cap <<= 1;
            // line layouts (modes 1 / 2) want lines at most about half full, unless the keys
            // fill their lines evenly: candidates are tried in this order, each judged by the rows that had to leave their home line
            //   mode 2, base capacity  : "dense" - e.g. TPC-H order keys: every line of 32 key values holds exactly its 8 keys
            //   mode 2, 2 x capacity   : a line expects ~4 keys (random subsets of a dense domain: what a hash exchange leaves on a rank)
            //   mode 1, 2 x capacity   : scattered lines, any distribution
            const char* env_mode = getenv("TGPU_JOIN_HASH");
            const DevColumn& bkey = lk->store.cols[0];
            const bool int_key = !lk->generic && key_kind_of(bkey.type) == KEY_INT;
            int hash_mode = env_mode ? atoi(env_mode) : (int_key && rows > 0 ? 2 : 1);
            if (hash_mode == 2 && !(int_key && rows > 0)) hash_mode = 1;
            const char* env_shift = getenv("TGPU_JOIN_CAP_SHIFT");
            const int64_t base_cap = cap;
            unsigned long long span = 0, kmin = 0;
            if (hash_mode == 2) {
                long long* d_range = ctx->d_scratch->join_key_range;
                long long init_range[2] = {INT64_MAX, INT64_MIN};
                TG_CUDA(ctx, cudaMemcpyAsync(d_range, init_range, sizeof(init_range), cudaMemcpyHostToDevice, ctx->stream));
                TG_LAUNCH(ctx, join_key_range_kernel, tg_grid(ctx, rows, 1024, 8), 256, 0, tg_colref(bkey), rows, d_range);
                long long h_range[2];
                TG_CUDA(ctx, cudaMemcpyAsync(h_range, d_range, sizeof(h_range), cudaMemcpyDeviceToHost, ctx->stream));
                TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
                if (h_range[0] > h_range[1]) hash_mode = 1;      // no insertable key at all
                else {
                    span = (unsigned long long)h_range[1] - (unsigned long long)h_range[0];   // kmax - kmin, exact in 64 bits
                    kmin = (unsigned long long)h_range[0];
                }
            }
            int* d_flags = ctx->d_scratch->join_build_flags;
            unsigned int* d_gave_up = ctx->d_scratch->join_gave_up;
            // attempt 0: dense mode 2; attempt 1: roomy mode 2; attempt 2: mode 1 (or whatever the environment pinned)
            for (int attempt = (hash_mode == 2 && !env_shift && !getenv("TGPU_JOIN_NO_DENSE")) ? 0 : 1; ; attempt++) {
                if (hash_mode == 2 && attempt >= 2) hash_mode = 1;
                const int cap_shift = env_shift ? atoi(env_shift) : (hash_mode == 0 ? 0 : (hash_mode == 2 && attempt == 0) ? 0 : 1);
                cap = base_cap << cap_shift;
                if (cap > (1LL << 31)) return tg_fail(ctx, TGPU_ERR_INSUFFICIENT_RESOURCES, "hash array too large");
                lk->geo.mask = (unsigned long long)cap - 1;
                lk->geo.kmin = 0;
                lk->geo.shift = 0;
                if (hash_mode == 2) {
                    // order-preserving lines: the key range [kmin, kmax] is cut into cap / 8 lines of 2^shift key values
                    const unsigned long long lines = (unsigned long long)cap >> 3;
                    int shift = 0;
                    while (shift < 63 && (span >> shift) >= lines) shift++;
                    if ((span >> shift) >= lines) { hash_mode = 1; attempt = 1; continue; }   // a span of 2^63 or more over very few lines
                    lk->geo.kmin = kmin;
                    lk->geo.shift = shift;
                }
                lk->geo.mode = hash_mode;
                TG_TRY(lk->table.alloc(ctx, (size_t)cap * sizeof(JoinSlot)));
                TG_TRY(tg_fill16(ctx, lk->table.as<int4>(), cap, make_int4(0, (int)0x80000000, -1, 0)));   // empty slot
                int init[4] = {-1, 0, 0, 0};
                TG_CUDA(ctx, cudaMemcpyAsync(d_flags, init, sizeof(init), cudaMemcpyHostToDevice, ctx->stream));
                TG_CUDA(ctx, cudaMemsetAsync(d_gave_up, 0, 8, ctx->stream));
                // mode 2 geometries are trials (the keys must suit them): bounded probing, early stop
                const int give_up_lines = hash_mode == 2 ? 16 : 0;
                const unsigned int give_up_limit = (unsigned int)std::min<int64_t>(rows / 1024, 1 << 20);
                if (rows > 0) {
                    TG_LAUNCH(ctx, join_build_kernel, tg_grid(ctx, rows, 256, 8), 256, 0, tg_colref(bkey), key_kind_of(bkey.type), rows,
                              lk->table.as<JoinSlot>(), lk->geo, d_flags, d_flags + 1, (unsigned int*)(d_flags + 2), give_up_lines, give_up_limit, d_gave_up);
                }
                if (hash_mode != 2) break;
                // mode 2 relies on the keys spreading evenly over their range; clustered domains pile up in a few lines.  Dense: at most
                // 1/64 of the rows off their home line; roomy: at most 1/8; and (nearly) no row further than 8 lines away, and every
                // row placed
                int64_t moved = 0, unplaced = 0;
                TG_TRY(tg_read_i64(ctx, d_flags + 2, &moved));
                TG_TRY(tg_read_i64(ctx, d_gave_up, &unplaced));
                const int64_t off_home = moved & 0xFFFFFFFFLL, far = (moved >> 32) & 0xFFFFFFFFLL;
                if ((unplaced & 0xFFFFFFFFLL) == 0 && off_home * (attempt == 0 ? 64 : 8) <= rows && far * 1024 <= rows) break;
            }
            int64_t packed = 0;
            TG_TRY(tg_read_i64(ctx, d_flags, &packed));
            lk->special_head = (int)(packed & 0xFFFFFFFFLL);
            lk->has_dups = (packed >> 32) != 0;
            return TGPU_OK;
        };
        if (!lk->generic) TG_TRY(build_table());
        else {
            // the fingerprint table: every row must sit in a slot whose head row carries ITS key.  Rows that share a 64-bit hash with a
            // different key move on to their next hash function and the table is rebuilt (never needed in practice; never a failure)
            DevBuf attempt;
            TG_TRY(attempt.alloc(ctx, (size_t)std::max<int64_t>(rows, 1)));
            TG_CUDA(ctx, cudaMemsetAsync(attempt.p, 0, (size_t)std::max<int64_t>(rows, 1), ctx->stream));
            for (int round = 0; ; round++) {
                if (round >= 8) return tg_fail(ctx, TGPU_ERR_INSUFFICIENT_RESOURCES, "join keys collide under 8 independent 64-bit hashes");
                if (round > 0) {
                    std::vector<const DevColumn*> kp;
                    for (auto& c : lk->build_keys) kp.push_back(&c);
                    DevColumn fp;
                    TG_TRY(make_fingerprint(ctx, kp, rows, &fp, attempt.as<uint8_t>()));
                    lk->store.cols[0] = std::move(fp);
                }
                TG_TRY(build_table());
                lk->attempts = round + 1;
                if (rows == 0) break;
                int* d_moved = ctx->d_scratch->join_moved;
                TG_CUDA(ctx, cudaMemsetAsync(d_moved, 0, 8, ctx->stream));
                const DevColumn& fp = lk->store.cols[0];
                TG_LAUNCH(ctx, join_verify_build_kernel, tg_grid(ctx, rows, 256, 8), 256, 0, key_cols_of(lk->build_keys), (const long long*)fp.data, fp.validity, rows,
                          lk->table.as<JoinSlot>(), lk->geo, lk->special_head, attempt.as<uint8_t>(), d_moved);
                int64_t moved = 0;
                TG_TRY(tg_read_i64(ctx, d_moved, &moved));
                if ((moved & 0xFFFFFFFFLL) == 0) break;
            }
        }
        if (lk->has_dups) {
            // ArrayPositionLinks: chains in descending row order
            const DevColumn& key = lk->store.cols[0];
            DevBuf keys_in, keys_out;
            TG_TRY(keys_in.alloc(ctx, (size_t)rows * 8));
            TG_TRY(keys_out.alloc(ctx, (size_t)rows * 8));
            TG_LAUNCH(ctx, join_slot_of_row_kernel, tg_grid(ctx, rows, 256, 8), 256, 0, tg_colref(key), key_kind_of(key.type), rows,
                      lk->table.as<JoinSlot>(), lk->geo, (unsigned long long)cap, keys_in.as<unsigned long long>());
            TG_TRY(tg_sort_keys(ctx, keys_in.as<unsigned long long>(), keys_out.as<unsigned long long>(), (int)rows, 0, 64));
            TG_TRY(lk->links.alloc(ctx, (size_t)rows * 4));
            TG_LAUNCH(ctx, join_links_kernel, tg_grid(ctx, rows, 256, 8), 256, 0, keys_out.as<unsigned long long>(), rows, lk->links.as<int>());
            TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        }
        // slot-ordered copy of the build output columns for the fused probe
        bool slot_payload = !getenv("TGPU_JOIN_PAYLOAD_BY_ROW") && rows > 0 && lk->num_output > 0 && lk->num_output <= 4;
        for (int32_t b = 0; b < lk->num_output && slot_payload; b++)
            slot_payload = lk->store.cols[1 + b].elem_size() > 0 && lk->store.cols[1 + b].elem_size() <= 8 && !lk->store.cols[1 + b].validity;
        if (slot_payload) {
            lk->by_slot.resize(lk->num_output);
            for (int32_t b = 0; b < lk->num_output; b++) {
                const DevColumn& c = lk->store.cols[1 + b];
                TG_TRY(lk->by_slot[b].alloc(ctx, (size_t)(cap + 1) * c.elem_size()));
                TG_LAUNCH(ctx, join_payload_by_slot_kernel, tg_grid(ctx, cap + 1, 1024, 8), 256, 0, lk->table.as<JoinSlot>(), cap, lk->special_head, c.data,
                          c.elem_size(), lk->by_slot[b].p);
            }
        }
        // slots that carry the payload of their head row: keyed slots for one output column (packed into 4 or 8 bytes under mode 2 when the
        // data allow it, else 16 bytes), 32-byte wide slots for two
        if (slot_payload && lk->num_output <= 2 && !lk->has_dups && !lk->generic && cap + 1 < (1LL << 31) && !getenv("TGPU_JOIN_NO_WIDE")) {
            const DevColumn& c0 = lk->store.cols[1];
            const DevColumn* c1 = lk->num_output > 1 ? &lk->store.cols[2] : nullptr;
            const int grid = tg_grid(ctx, cap + 1, 1024, 8);
            if (!c1) {
                lk->keyed_bytes = 16;
                if (lk->geo.mode == 2) {
                    DevBuf d_range;
                    TG_TRY(d_range.alloc(ctx, 4 * sizeof(long long)));
                    long long range[4] = {INT64_MAX, INT64_MIN, INT64_MAX, INT64_MIN};
                    TG_CUDA(ctx, cudaMemcpyAsync(d_range.p, range, sizeof(range), cudaMemcpyHostToDevice, ctx->stream));
                    TG_LAUNCH(ctx, join_packed_range_kernel, grid, 256, 0, lk->table.as<JoinSlot>(), cap, lk->geo.kmin, lk->geo.shift, lk->special_head, c0.data,
                              c0.elem_size(), d_range.as<long long>());
                    TG_CUDA(ctx, cudaMemcpyAsync(range, d_range.p, sizeof(range), cudaMemcpyDeviceToHost, ctx->stream));
                    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
                    // an empty range (no occupied slot, or no cell) fits every tier
                    auto fits = [&](long long krel_min, long long krel_max, unsigned long long cell_max) {
                        const bool krel_ok = range[0] > range[1] || (range[0] > krel_min && range[1] <= krel_max);
                        const bool cell_ok = range[2] > range[3] || (unsigned long long)range[3] - (unsigned long long)range[2] <= cell_max;
                        return krel_ok && cell_ok;
                    };
                    lk->keyed_cmin = range[2] > range[3] ? 0ULL : (unsigned long long)range[2];
                    if (fits(PackedSlot4::KREL_MIN, PackedSlot4::KREL_MAX, PackedSlot4::CELL_MAX)) lk->keyed_bytes = 4;
                    else if (fits(PackedSlot8::KREL_MIN, PackedSlot8::KREL_MAX, PackedSlot8::CELL_MAX)) lk->keyed_bytes = 8;
                }
                TG_TRY(lk->keyed.alloc(ctx, (size_t)(cap + 1) * lk->keyed_bytes));
                if (lk->keyed_bytes == 4)
                    TG_LAUNCH(ctx, join_packed_table_kernel<PackedSlot4>, grid, 256, 0, lk->table.as<JoinSlot>(), cap, lk->geo.kmin, lk->geo.shift, lk->special_head,
                              c0.data, c0.elem_size(), lk->keyed_cmin, lk->keyed.as<PackedSlot4>());
                else if (lk->keyed_bytes == 8)
                    TG_LAUNCH(ctx, join_packed_table_kernel<PackedSlot8>, grid, 256, 0, lk->table.as<JoinSlot>(), cap, lk->geo.kmin, lk->geo.shift, lk->special_head,
                              c0.data, c0.elem_size(), lk->keyed_cmin, lk->keyed.as<PackedSlot8>());
                else
                    TG_LAUNCH(ctx, join_wide_table_kernel<KeyedSlot>, grid, 256, 0, lk->table.as<JoinSlot>(), cap, lk->special_head, c0.data, c0.elem_size(),
                              (const void*)nullptr, 0, lk->keyed.as<KeyedSlot>());
            }
            else {
                TG_TRY(lk->wide.alloc(ctx, (size_t)(cap + 1) * sizeof(WideSlot)));
                TG_LAUNCH(ctx, join_wide_table_kernel<WideSlot>, grid, 256, 0, lk->table.as<JoinSlot>(), cap, lk->special_head, c0.data, c0.elem_size(),
                          c1->data, c1->elem_size(), lk->wide.as<WideSlot>());
            }
        }
        TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        lookup = lk.release();
        finishing = true;
        return TGPU_OK;
    }

    int get_output(OwnedPage** out) override { *out = nullptr; return TGPU_OK; }
    // HashBuilderOperator.isFinished: after the lookup source was handed over and released
    bool is_finished() override { return finishing; }
    int64_t memory_bytes() override
    {
        int64_t b = 0;
        for (auto& c : chunks) b += c.memory_bytes();
        if (lookup) b += tgpu_lookup_memory_bytes(lookup);
        return b;
    }
};

// LookupJoinOperator
struct JoinProbeOp : tgpu_op {
    tgpu_lookup* lookup;
    int join_type = 0, single_match = 0;
    std::vector<int32_t> key_channels, output_channels;
    std::vector<OwnedPage*> pending;
    size_t next_out = 0;
    bool finishing = false;
    // fast path: addInput only enqueues the probe kernel; the match count is read (the one host synchronisation of the
    // step) when the output is asked for, so the caller can overlap other work - the next exchange - with the probe
    struct Deferred {
        bool active = false;
        DevPage in;
        std::shared_ptr<DevBuf> match_bits;     // bit i: probe row i matched (32-bit words, Arrow LSB order)
        std::vector<DevColumn> built;
        int64_t n = 0;
    } deferred;
    DevBuf match_counter;     // per operator: the count must survive until get_output
    // LookupJoinPageBuilder.build :144-150 hands probe blocks through as views.  With by_reference set, a HOST probe page
    // only has its join-key channel uploaded; pass-through output columns of the result then carry no device data
    // (data == NULL, tgpu_page_passthrough_channel names the input block) unless rows had to be dropped or repeated
    bool by_reference = false;

    JoinProbeOp(tgpu_ctx* c, tgpu_lookup* lk) : tgpu_op(c), lookup(lk) { lookup->refs++; }
    ~JoinProbeOp() override
    {
        for (size_t i = next_out; i < pending.size(); i++) delete pending[i];
        tgpu_lookup_release(lookup);
    }

    bool needs_input() override { return !finishing && !deferred.active && next_out >= pending.size(); }

    // fused probe + gather (see join_probe_gather_kernel); returns handled=false when the shape needs the general path
    int fast_path(DevPage& in, const DevColumn& key, int64_t n, bool* handled)
    {
        *handled = false;
        
        if (lookup->has_dups && !single_match) return TGPU_OK;
        if (lookup->num_output > 4) return TGPU_OK;
        if (!probe_key_fits_keyed_table(key.type, lookup->key_type)) return TGPU_OK;   // reported by the general path
        for (int32_t b = 0; b < lookup->num_output; b++) {
            const DevColumn& c = lookup->store.cols[1 + b];
            if (c.elem_size() == 0 || c.elem_size() > 8 || c.validity) return TGPU_OK;      // (the fused gather moves 1 / 2 / 4 / 8-byte payloads)
        }
        // which probe rows matched, one bit per row (store_match_word); it is the build columns' validity of a PROBE_OUTER page
        auto match_bits = std::make_shared<DevBuf>();
        TG_TRY(match_bits->alloc(ctx, (size_t)((n + 31) / 32) * 4));
        unsigned int* bits = match_bits->as<unsigned int>();
        GatherCols g;
        memset(&g, 0, sizeof(g));
        g.count = lookup->num_output;
        std::vector<DevColumn> built(lookup->num_output);
        for (int32_t b = 0; b < lookup->num_output; b++) {
            const DevColumn& c = lookup->store.cols[1 + b];
            built[b].type = c.type;
            built[b].length = n;
            built[b].own_data = std::make_shared<DevBuf>();
            TG_TRY(built[b].own_data->alloc(ctx, (size_t)n * c.elem_size()));
            built[b].data = built[b].own_data->p;
            g.elem[b] = c.elem_size();
            g.src[b] = lookup->by_slot.empty() ? c.data : lookup->by_slot[b].p;
            g.dst[b] = built[b].own_data->p;
        }
        g.by_slot = lookup->by_slot.empty() ? 0 : 1;
        if (!match_counter.p) TG_TRY(match_counter.alloc(ctx, 16));       // [0] matches of the page, [1] (int) layout choice of the page
        unsigned long long* d_matches = match_counter.as<unsigned long long>();
        TG_CUDA(ctx, cudaMemsetAsync(d_matches, 0, 16, ctx->stream));     // no matches yet; layout choice 0 = the 16-byte slots
        constexpr int ROWS = 4;
        int grid = tg_grid(ctx, n, 256 * ROWS, 8);
        auto k_fast = join_probe_gather_kernel<ROWS, true>;
        auto k_any = join_probe_gather_kernel<ROWS, false>;
        const JoinSlot* table = lookup->table.as<JoinSlot>();
        TG_TIMED_BEGIN(ctx);
        int64_t done = 0;
        bool fast = key.type == TGPU_INT64 && !key.validity;
        if (fast && !getenv("TGPU_JOIN_GENERIC_KERNELS")) {
            int64_t tiles = n / 1024;
            if (tiles > 0) {
                // TGPU_JOIN_WIDE = always | never | auto (default): auto lets the page's key locality decide whenever the wide layout is the
                // bigger one (payload cells < 16 bytes); with 16 bytes of payload the two layouts hold the same bytes and wide always wins
                const char* we = getenv("TGPU_JOIN_WIDE");
                int payload_bytes = 0;
                for (int c = 0; c < g.count; c++) payload_bytes += g.elem[c];
                // A keyed table (one payload column) serves both kinds of page: the locality vote picks the key-ordered or the random-access
                // shape of the same kernel, and TGPU_JOIN_WIDE=always pins the random-access one
                const long long* keys = (const long long*)key.data;
                const bool layouts_on = !getenv("TGPU_JOIN_NO_WIDE") && !getenv("TGPU_JOIN_SPAN") && !(we && !strcmp(we, "never"));
                const bool have_keyed = lookup->keyed.p && layouts_on;
                const bool have_wide = lookup->wide.p && layouts_on;
                const bool always = (have_wide || have_keyed) && ((we && !strcmp(we, "always")) || payload_bytes >= 16 || !g.by_slot);
                int* d_choice = (int*)(d_matches + 1);
                // the keyed table in its slot type: the random-access shape alone, or the locality vote and both shapes
                auto run_keyed = [&](const auto* keyed) -> int {
                    const unsigned long long cmin = lookup->keyed_cmin;
                    if (always) return launch_wide(ctx, lookup->geo, keys, tiles, keyed, lookup->special_head, cmin, bits, g, d_matches, nullptr);
                    TG_TRY(launch_locality(ctx, lookup->geo, keys, tiles, d_choice));
                    TG_TRY(launch_keyed_ordered(ctx, lookup->geo, keys, tiles, keyed, lookup->special_head, cmin, bits, g, d_matches, d_choice));
                    return launch_wide(ctx, lookup->geo, keys, tiles, keyed, lookup->special_head, cmin, bits, g, d_matches, d_choice);
                };
                if (have_keyed && lookup->keyed_bytes == 4) TG_TRY(run_keyed(lookup->keyed.as<PackedSlot4>()));
                else if (have_keyed && lookup->keyed_bytes == 8) TG_TRY(run_keyed(lookup->keyed.as<PackedSlot8>()));
                else if (have_keyed) TG_TRY(run_keyed(lookup->keyed.as<KeyedSlot>()));
                else if (always)
                    TG_TRY(launch_wide(ctx, lookup->geo, keys, tiles, lookup->wide.as<WideSlot>(), lookup->special_head, 0ULL, bits, g, d_matches, nullptr));
                else if (have_wide) {
                    TG_TRY(launch_locality(ctx, lookup->geo, keys, tiles, d_choice));
                    TG_TRY(launch_lean<true>(ctx, lookup->geo, keys, tiles, (const int4*)table, lookup->special_head, nullptr, bits, g, d_matches));
                    TG_TRY(launch_wide(ctx, lookup->geo, keys, tiles, lookup->wide.as<WideSlot>(), lookup->special_head, 0ULL, bits, g, d_matches, d_choice));
                }
                else
                    TG_TRY(launch_lean<true>(ctx, lookup->geo, keys, tiles, (const int4*)table, lookup->special_head, nullptr, bits, g, d_matches));
                done = tiles * 1024;
            }
        }
        if (done < n) {
            ColRef kr = tg_colref(key);
            GatherCols gt = g;
            if (done > 0) {
                kr.data = (const char*)kr.data + done * 8;
                for (int c = 0; c < gt.count; c++) gt.dst[c] = (char*)gt.dst[c] + done * gt.elem[c];
            }
            int tgrid = tg_grid(ctx, n - done, 256 * ROWS, 8);
            // done is a multiple of 1024: the tail's bitmap starts at a word boundary
            if (fast) TG_LAUNCH(ctx, k_fast, tgrid, 256, 0, kr, KEY_INT, n - done, table, lookup->geo, lookup->special_head, bits + done / 32, gt, d_matches);
            else TG_LAUNCH(ctx, k_any, tgrid, 256, 0, kr, key_kind_of(key.type), n - done, table, lookup->geo, lookup->special_head, bits + done / 32, gt, d_matches);
        }
        TG_TIMED_END(ctx);
        *handled = true;
        deferred.active = true;
        deferred.in = std::move(in);
        deferred.match_bits = match_bits;
        deferred.built = std::move(built);
        deferred.n = n;
        return TGPU_OK;
    }

    // second half of the fast path: read the match count and shape the output page
    // partial ingest of a host page: the join-key channel goes to the device, the others stay placeholders
    int ingest_keys_only(const tgpu_page* page, DevPage* out)
    {
        DevPage p;
        p.rows = page->num_rows;
        p.cols.resize(page->num_columns);
        for (int32_t c = 0; c < page->num_columns; c++) {
            if (page->columns[c].length != page->num_rows) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "column %d has %lld positions, page has %lld", c,
                                                                          (long long)page->columns[c].length, (long long)page->num_rows);
            bool is_key = c == key_channels[0] || reads_probe_channel(c);    // (the join filter's probe channels go up with the key)
            if (is_key) TG_TRY(tg_ingest_column(ctx, &page->columns[c], false, &p.cols[c]));
            else { p.cols[c].type = page->columns[c].type; p.cols[c].length = page->num_rows; }
        }
        TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        *out = std::move(p);
        return TGPU_OK;
    }

    static bool absent(const DevColumn& c) { return c.data == nullptr && c.length > 0; }

    bool reads_probe_channel(int32_t c) const
    {
        if (!lookup->has_filter) return false;
        return std::find(lookup->filter_channels.begin(), lookup->filter_channels.end(), lookup->num_build_channels + c) != lookup->filter_channels.end();
    }

    // ---- join filter function ----
    void* jit_jf_positions = nullptr;   // NVRTC kernels for the current page shape (nullptr: interpreter kernels)
    void* jit_jf_pairs = nullptr;
    std::string jit_jf_key;

    // the join-sources layout of this page (build channels, then probe channels) as the filter kernels read it; checks the channels
    int filter_columns(const DevPage& in, DColumns* cols)
    {
        memset(cols, 0, sizeof(*cols));
        const int nb = lookup->num_build_channels;
        int elems[TGPU_MAX_CHANNELS] = {0};
        uint32_t nullable = 0;
        for (int32_t ch : lookup->filter_channels) {
            const DevColumn* c = nullptr;
            if (ch < nb) c = &lookup->filter_cols[ch];
            else if (ch - nb < (int32_t)in.cols.size()) c = &in.cols[ch - nb];
            else return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "join filter reads channel %d: the layout has %d build and %zu probe channels", ch, nb, in.cols.size());
            if (!join_filter_type_ok(*c))
                return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "join filters over variable-width / 128-bit / REAL channel %d are not supported on the GPU path", ch);
            cols->cols[ch] = tg_colref(*c);
            elems[ch] = c->elem_size();
            if (c->validity) nullable |= 1u << ch;
        }
        if (!tg::jit_available()) { jit_jf_positions = jit_jf_pairs = nullptr; return TGPU_OK; }
        std::string key;
        for (int c = 0; c < TGPU_MAX_CHANNELS; c++) key += (char)('0' + elems[c]);
        key += ":" + std::to_string(nullable);
        if (key == jit_jf_key && jit_jf_positions) return TGPU_OK;
        const std::string src = gen_join_filter_source(lookup->filter, nb, elems, TGPU_MAX_CHANNELS, nullable);
        TG_TRY(tg::jit_get_function(ctx, src, "tg_jf_positions_jit", &jit_jf_positions));
        TG_TRY(tg::jit_get_function(ctx, src, "tg_jf_pairs_jit", &jit_jf_pairs));
        jit_jf_key = key;
        return TGPU_OK;
    }

    int raise_filter_errors()
    {
        int64_t word = 0;
        TG_TRY(tg_read_i64(ctx, ctx->d_scratch->join_filter_flags, &word));
        return tg::expr_raise(ctx, word & 0xFFFFFFFFLL);
    }

    // no position links: the one candidate of each probe row is dropped (jp[i] = -1) when the filter does not accept it
    int filter_positions(DColumns cols, int* jp, int64_t n)
    {
        unsigned int* d_err = ctx->d_scratch->join_filter_flags;
        TG_CUDA(ctx, cudaMemsetAsync(d_err, 0, 8, ctx->stream));
        long long n_arg = n;
        if (jit_jf_positions) {
            void* params[4] = {&cols, &n_arg, &jp, &d_err};
            TG_TRY(tg::jit_launch(ctx, jit_jf_positions, tg_grid(ctx, n, JF_THREADS, tg::jit_blocks_per_sm(jit_jf_positions, JF_THREADS, 0)), JF_THREADS, 0, params));
        }
        else TG_LAUNCH(ctx, join_filter_positions_kernel, tg_grid(ctx, n, JF_THREADS, 8), JF_THREADS, 0, lookup->d_filter.as<DProgram>(), cols,
                       lookup->num_build_channels, n, jp, d_err);
        return raise_filter_errors();
    }

    // with position links: candidate pairs in chain order, the filter's verdict on each, then PageJoiner's choice per probe row.
    // Output rows (probe row, build position or -1) into out_probe / out_build, their number into *total
    int filter_pairs(DColumns cols, const int* jp, int64_t n, const int* links, bool outer, DevBuf* out_probe, DevBuf* out_build, int64_t* total)
    {
        const int grid = tg_grid(ctx, n, 256 * 4, 8);
        DevBuf counts, offsets;
        TG_TRY(counts.alloc(ctx, (size_t)(n + 1) * 4));
        TG_TRY(offsets.alloc(ctx, (size_t)(n + 1) * 8));
        TG_LAUNCH(ctx, join_count_kernel, grid, 256, 0, jp, n, links, 0, 0, counts.as<int>());
        TG_TRY(tg_exclusive_sum(ctx, counts.as<int>(), offsets.as<long long>(), n + 1));
        int64_t m = 0;
        TG_TRY(tg_read_i64(ctx, offsets.as<long long>() + n, &m));
        if (m > (int64_t)INT32_MAX) return tg_fail(ctx, TGPU_ERR_INSUFFICIENT_RESOURCES, "join candidates of one probe page exceed 2^31-1 rows");
        DevBuf pp, pb, verdict;
        TG_TRY(pp.alloc(ctx, (size_t)m * 4));
        TG_TRY(pb.alloc(ctx, (size_t)m * 4));
        TG_TRY(verdict.alloc(ctx, (size_t)m));
        if (m > 0) {
            TG_LAUNCH(ctx, join_fill_kernel, grid, 256, 0, jp, n, links, 0, 0, offsets.as<long long>(), pp.as<int>(), pb.as<int>());
            long long m_arg = m;
            const int* pp_arg = pp.as<int>();
            const int* pb_arg = pb.as<int>();
            unsigned char* v_arg = verdict.as<unsigned char>();
            if (jit_jf_pairs) {
                void* params[5] = {&cols, &m_arg, &pp_arg, &pb_arg, &v_arg};
                TG_TRY(tg::jit_launch(ctx, jit_jf_pairs, tg_grid(ctx, m, JF_THREADS, tg::jit_blocks_per_sm(jit_jf_pairs, JF_THREADS, 0)), JF_THREADS, 0, params));
            }
            else TG_LAUNCH(ctx, join_filter_pairs_kernel, tg_grid(ctx, m, JF_THREADS, 8), JF_THREADS, 0, lookup->d_filter.as<DProgram>(), cols,
                           lookup->num_build_channels, m, pp_arg, pb_arg, verdict.as<uint8_t>());
        }
        unsigned int* d_err = ctx->d_scratch->join_filter_flags;
        TG_CUDA(ctx, cudaMemsetAsync(d_err, 0, 8, ctx->stream));
        DevBuf out_counts, out_off;
        TG_TRY(out_counts.alloc(ctx, (size_t)(n + 1) * 4));
        TG_TRY(out_off.alloc(ctx, (size_t)(n + 1) * 8));
        TG_LAUNCH(ctx, join_filter_select_kernel, tg_grid(ctx, n, 256, 8), 256, 0, offsets.as<long long>(), n, single_match, outer ? 1 : 0, verdict.as<uint8_t>(),
                  out_counts.as<int>(), d_err);
        TG_TRY(tg_exclusive_sum(ctx, out_counts.as<int>(), out_off.as<long long>(), n + 1));
        TG_TRY(raise_filter_errors());
        TG_TRY(tg_read_i64(ctx, out_off.as<long long>() + n, total));
        if (*total == 0) return TGPU_OK;
        if (*total > (int64_t)INT32_MAX) return tg_fail(ctx, TGPU_ERR_INSUFFICIENT_RESOURCES, "join output of one probe page exceeds 2^31-1 rows");
        TG_TRY(out_probe->alloc(ctx, (size_t)*total * 4));
        TG_TRY(out_build->alloc(ctx, (size_t)*total * 4));
        TG_LAUNCH(ctx, join_filter_fill_kernel, tg_grid(ctx, n, 256, 8), 256, 0, offsets.as<long long>(), n, verdict.as<uint8_t>(), pb.as<int>(), outer ? 1 : 0,
                  out_off.as<long long>(), out_probe->as<int>(), out_build->as<int>());
        return TGPU_OK;
    }

    int upload_absent(const tgpu_page* page, DevPage* in)
    {
        bool any = false;
        for (int32_t c = 0; c < page->num_columns; c++) {
            if (!absent(in->cols[c])) continue;
            TG_TRY(tg_ingest_column(ctx, &page->columns[c], false, &in->cols[c]));
            any = true;
        }
        if (any) TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        return TGPU_OK;
    }

    // `host_page`: the input of a by-reference probe (its pass-through channels were not uploaded), else nullptr
    int complete_fast(const tgpu_page* host_page = nullptr)
    {
        deferred.active = false;
        DevPage in = std::move(deferred.in);
        std::shared_ptr<DevBuf> match_bits = std::move(deferred.match_bits);
        std::vector<DevColumn> built = std::move(deferred.built);
        const int64_t n = deferred.n;
        const bool outer = join_type == TGPU_JOIN_PROBE_OUTER;     // (tracking join types never take the fast path)
        int64_t matches = 0;
        TG_TRY(tg_read_i64(ctx, match_counter.as<int64_t>(), &matches));
        DevPage outp;
        if (host_page && !(matches == n || outer) && matches > 0) TG_TRY(upload_absent(host_page, &in));   // rows are dropped: the gather needs them
        if (matches == n || outer) {
            // every probe row yields exactly one output row: probe blocks pass through
            // (LookupJoinPageBuilder.build :144-150 "outputProbeBlocksDirectly")
            outp.rows = n;
            for (int32_t ch : output_channels) outp.cols.push_back(in.cols[ch]);
            // a PROBE_OUTER page with misses: the match bitmap is the build columns' validity as it stands (bits past n are 0)
            std::shared_ptr<DevBuf> validity;
            if (matches < n) validity = match_bits;
            for (auto& c : built) {
                if (validity) { c.own_validity = validity; c.validity = validity->as<uint8_t>(); }
                outp.cols.push_back(std::move(c));
            }
        }
        else {
            if (matches == 0) return TGPU_OK;
            // compact the matched rows (stable): selection list, then sequential-read gathers
            DevBuf flags, sel;
            TG_TRY(flags.alloc(ctx, (size_t)n));
            TG_LAUNCH(ctx, join_match_flags_kernel, tg_grid(ctx, n, 1024, 8), 256, 0, match_bits->as<unsigned int>(), n, flags.as<uint8_t>());
            TG_TRY(tg_flagged_positions(ctx, flags.as<uint8_t>(), n, &sel, &ctx->d_scratch->join_probe_count));
            outp.rows = matches;
            for (int32_t ch : output_channels) {
                DevColumn c;
                TG_TRY(tg_gather_column(ctx, in.cols[ch], sel.as<int32_t>(), matches, false, &c));
                outp.cols.push_back(std::move(c));
            }
            for (auto& b : built) {
                DevColumn c;
                TG_TRY(tg_gather_column(ctx, b, sel.as<int32_t>(), matches, false, &c));
                outp.cols.push_back(std::move(c));
            }
        }
        OwnedPage* o = tg_make_owned_page(std::move(outp));
        if (matches == n || outer) o->passthrough.assign(output_channels.begin(), output_channels.end());   // probe blocks passed through 1:1
        pending.push_back(o);
        return TGPU_OK;
    }

    int add_input(const tgpu_page* page) override
    {
        if (deferred.active) return tg_fail(ctx, TGPU_ERR_ILLEGAL_STATE, "addInput while the previous page's output has not been taken (needsInput() is false)");
        for (size_t i = next_out; i < pending.size(); i++) delete pending[i];
        pending.clear();
        next_out = 0;
        int64_t n = page->num_rows;
        if (n == 0) return TGPU_OK;
        if (n > (int64_t)INT32_MAX) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "page has more than 2^31-1 positions");
        DevPage in;
        const bool lazy = by_reference && !(page->flags & TGPU_PAGE_DEVICE) && !lookup->generic && key_channels.size() == 1;
        if (lazy) TG_TRY(ingest_keys_only(page, &in));
        else TG_TRY(tg_ingest_page(ctx, page, &in));
        if (key_channels[0] < 0 || key_channels[0] >= (int32_t)in.cols.size()) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "probe key channel out of range");
        for (int32_t ch : output_channels)
            if (ch < 0 || ch >= (int32_t)in.cols.size()) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "probe output channel out of range");
        for (int32_t ch : key_channels)
            if (ch < 0 || ch >= (int32_t)in.cols.size()) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "probe key channel out of range");
        const DevColumn& key = in.cols[key_channels[0]];
        if (!lookup->generic && key_channels.size() != 1) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "probe has %zu join channels, build has 1", key_channels.size());
        const bool tracking = join_type == TGPU_JOIN_LOOKUP_OUTER || join_type == TGPU_JOIN_FULL_OUTER;
        DColumns fcols;
        if (lookup->has_filter) TG_TRY(filter_columns(in, &fcols));
        if (!lookup->generic && !tracking && !lookup->has_filter && !getenv("TGPU_JOIN_GENERAL_PATH")) {
            bool handled = false;
            TG_TRY(fast_path(in, key, n, &handled));
            if (handled) return lazy ? complete_fast(page) : TGPU_OK;   // host buffers are the caller's again after this call
        }
        if (lazy) TG_TRY(upload_absent(page, &in));
        // joinPositionCache (JoinProbe.java:112-180)
        auto jp = std::make_shared<DevBuf>();
        TG_TRY(jp->alloc(ctx, (size_t)(n + 1) * 4));
        if (lookup->generic) {
            std::vector<const DevColumn*> kp;
            for (int32_t ch : key_channels) kp.push_back(&in.cols[ch]);
            TG_TRY(lookup_positions_generic(ctx, lookup, kp, n, jp->as<int>()));
        }
        else TG_TRY(lookup_positions(ctx, lookup, key, jp->as<int>()));
        bool outer = join_type == TGPU_JOIN_PROBE_OUTER || join_type == TGPU_JOIN_FULL_OUTER;
        const int* links = lookup->has_dups ? lookup->links.as<int>() : nullptr;
        // a join filter without position links only drops candidates: the expansion below then runs as without a filter
        if (lookup->has_filter && !links) TG_TRY(filter_positions(fcols, jp->as<int>(), n));
        const bool filtered_pairs = lookup->has_filter && links;
        DevBuf out_probe, out_build;
        // match counts -> exclusive scan -> output offsets
        DevBuf counts, offsets;
        int grid = tg_grid(ctx, n, 256 * 4, 8);
        int64_t total = 0;
        if (filtered_pairs) TG_TRY(filter_pairs(fcols, jp->as<int>(), n, links, outer, &out_probe, &out_build, &total));
        else {
            TG_TRY(counts.alloc(ctx, (size_t)(n + 1) * 4));
            TG_TRY(offsets.alloc(ctx, (size_t)(n + 1) * 8));
            TG_LAUNCH(ctx, join_count_kernel, grid, 256, 0, jp->as<int>(), n, links, single_match, outer ? 1 : 0, counts.as<int>());
            TG_TRY(tg_exclusive_sum(ctx, counts.as<int>(), offsets.as<long long>(), n + 1));
            TG_TRY(tg_read_i64(ctx, offsets.as<long long>() + n, &total));
        }
        if (total == 0) return TGPU_OK;
        if (total > (int64_t)INT32_MAX) return tg_fail(ctx, TGPU_ERR_INSUFFICIENT_RESOURCES, "join output of one probe page exceeds 2^31-1 rows");

        DevPage outp;
        outp.rows = total;
        // every probe row produced exactly one row and there are no chains: probe rows map 1:1
        // (LookupJoinPageBuilder.build :144-150 "outputProbeBlocksDirectly")
        bool identity = !filtered_pairs && (total == n) && (!links || single_match);
        const int* build_idx = nullptr;
        bool build_may_be_null = outer;
        if (identity) {
            for (int32_t ch : output_channels) outp.cols.push_back(in.cols[ch]);   // shares ownership, no copy
            build_idx = jp->as<int>();
        }
        else {
            if (!filtered_pairs) {
                TG_TRY(out_probe.alloc(ctx, (size_t)total * 4));
                TG_TRY(out_build.alloc(ctx, (size_t)total * 4));
                TG_LAUNCH(ctx, join_fill_kernel, grid, 256, 0, jp->as<int>(), n, links, single_match, outer ? 1 : 0, offsets.as<long long>(),
                          out_probe.as<int>(), out_build.as<int>());
            }
            for (int32_t ch : output_channels) {
                DevColumn c;
                TG_TRY(tg_gather_column(ctx, in.cols[ch], out_probe.as<int>(), total, false, &c));
                outp.cols.push_back(std::move(c));
            }
            build_idx = out_build.as<int>();
        }
        for (int32_t b = 0; b < lookup->num_output; b++) {
            DevColumn c;
            TG_TRY(tg_gather_column(ctx, lookup->store.cols[1 + b], build_idx, total, build_may_be_null, &c));
            outp.cols.push_back(std::move(c));
        }
        if (tracking && lookup->visited.p)
            TG_LAUNCH(ctx, join_mark_visited_kernel, tg_grid(ctx, total, 1024, 8), 256, 0, build_idx, total, lookup->visited.as<uint8_t>());
        pending.push_back(tg_make_owned_page(std::move(outp)));
        if (tracking) TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));   // the marks must be visible to the outer operator's context
        return TGPU_OK;
    }

    int get_output(OwnedPage** out) override
    {
        *out = nullptr;
        if (deferred.active) TG_TRY(complete_fast());
        if (next_out < pending.size()) *out = pending[next_out++];
        return TGPU_OK;
    }
    int finish() override { finishing = true; return TGPU_OK; }
    bool is_finished() override { return finishing && !deferred.active && next_out >= pending.size(); }
};

// LookupOuterOperator (M/operator/join/LookupOuterOperator.java:170-206): after every probe has finished, the build rows no
// probe emitted, in position order, with NULLs in the probe output channels.  A source operator.
struct JoinOuterOp : tgpu_op {
    tgpu_lookup* lookup;
    std::vector<int32_t> probe_types;
    bool done = false;
    OwnedPage* pending = nullptr;

    JoinOuterOp(tgpu_ctx* c, tgpu_lookup* lk) : tgpu_op(c), lookup(lk) { lookup->refs++; }
    ~JoinOuterOp() override { delete pending; tgpu_lookup_release(lookup); }

    bool needs_input() override { return false; }
    int add_input(const tgpu_page*) override { return tg_fail(ctx, TGPU_ERR_ILLEGAL_STATE, "LookupOuterOperator does not take input"); }

    int produce()
    {
        done = true;
        const int64_t n = lookup->positions;
        if (n == 0) return TGPU_OK;
        DevBuf flags, sel;
        TG_TRY(flags.alloc(ctx, (size_t)n));
        if (lookup->visited.p) TG_LAUNCH(ctx, join_unvisited_flags_kernel, tg_grid(ctx, n, 1024, 8), 256, 0, lookup->visited.as<uint8_t>(), n, flags.as<uint8_t>());
        else TG_CUDA(ctx, cudaMemsetAsync(flags.p, 1, (size_t)n, ctx->stream));     // no tracking probe ever ran: every row is unvisited
        long long* d_count = &ctx->d_scratch->join_outer_count;
        TG_TRY(tg_flagged_positions(ctx, flags.as<uint8_t>(), n, &sel, d_count));
        int64_t m = 0;
        TG_TRY(tg_read_i64(ctx, d_count, &m));
        if (m == 0) return TGPU_OK;
        DevPage outp;
        outp.rows = m;
        // probe channels: all NULL
        auto all_null = std::make_shared<DevBuf>();
        TG_TRY(all_null->alloc(ctx, (size_t)((m + 7) / 8)));
        TG_CUDA(ctx, cudaMemsetAsync(all_null->p, 0, (size_t)((m + 7) / 8), ctx->stream));
        for (int32_t t : probe_types) {
            DevColumn c;
            c.type = t;
            c.length = m;
            c.own_validity = all_null;
            c.validity = all_null->as<uint8_t>();
            size_t es = (size_t)(t == TGPU_UTF8 ? 1 : c.elem_size());
            c.own_data = std::make_shared<DevBuf>();
            TG_TRY(c.own_data->alloc(ctx, std::max<size_t>((size_t)m * es, 8)));
            TG_CUDA(ctx, cudaMemsetAsync(c.own_data->p, 0, std::max<size_t>((size_t)m * es, 8), ctx->stream));
            c.data = c.own_data->p;
            if (t == TGPU_UTF8) {
                c.own_offsets = std::make_shared<DevBuf>();
                TG_TRY(c.own_offsets->alloc(ctx, (size_t)(m + 1) * 4));
                TG_CUDA(ctx, cudaMemsetAsync(c.own_offsets->p, 0, (size_t)(m + 1) * 4, ctx->stream));
                c.offsets = c.own_offsets->as<int32_t>();
            }
            outp.cols.push_back(std::move(c));
        }
        for (int32_t b = 0; b < lookup->num_output; b++) {
            DevColumn c;
            TG_TRY(tg_gather_column(ctx, lookup->store.cols[1 + b], sel.as<int32_t>(), m, false, &c));
            outp.cols.push_back(std::move(c));
        }
        TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        pending = tg_make_owned_page(std::move(outp));
        return TGPU_OK;
    }

    int get_output(OwnedPage** out) override
    {
        *out = nullptr;
        if (!done) TG_TRY(produce());
        *out = pending;
        pending = nullptr;
        return TGPU_OK;
    }
    int finish() override { return TGPU_OK; }
    bool is_finished() override { return done && !pending; }
};

// HashSemiJoinOperator (M/operator/HashSemiJoinOperator.java:155-201) over a lookup built by a HashBuilder on the filtering
// source's join channel (the ChannelSet of SetBuilderOperator): input page + one BOOLEAN column.
struct SemiJoinOp : tgpu_op {
    tgpu_lookup* lookup;
    int32_t probe_channel = 0;
    OwnedPage* pending = nullptr;
    bool finishing = false;

    SemiJoinOp(tgpu_ctx* c, tgpu_lookup* lk) : tgpu_op(c), lookup(lk) { lookup->refs++; }
    ~SemiJoinOp() override { delete pending; tgpu_lookup_release(lookup); }

    bool needs_input() override { return !finishing && !pending; }

    int add_input(const tgpu_page* page) override
    {
        if (pending) return tg_fail(ctx, TGPU_ERR_ILLEGAL_STATE, "addInput while the previous page's output has not been taken");
        int64_t n = page->num_rows;
        if (n == 0) return TGPU_OK;
        DevPage in;
        TG_TRY(tg_ingest_page(ctx, page, &in));
        if (probe_channel < 0 || probe_channel >= (int32_t)in.cols.size()) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "probe join channel out of range");
        const DevColumn& key = in.cols[probe_channel];
        const int float_kind = key.type == TGPU_FLOAT64 ? 1 : key.type == TGPU_FLOAT32 ? 2 : 0;
        DevBuf pos;
        TG_TRY(pos.alloc(ctx, (size_t)n * 4));
        if (lookup->generic) {
            std::vector<const DevColumn*> kp{&key};
            TG_TRY(lookup_positions_generic(ctx, lookup, kp, n, pos.as<int>()));
        }
        else TG_TRY(lookup_positions(ctx, lookup, key, pos.as<int>()));
        DevColumn out;
        out.type = TGPU_INT8;
        out.length = n;
        out.own_data = std::make_shared<DevBuf>();
        TG_TRY(out.own_data->alloc(ctx, (size_t)n));
        out.data = out.own_data->p;
        DevBuf is_null;
        TG_TRY(is_null.alloc(ctx, (size_t)n));
        TG_LAUNCH(ctx, semi_join_kernel, tg_grid(ctx, n, 1024, 8), 256, 0, pos.as<int>(), key.validity, n, lookup->positions == 0 ? 1 : 0,
                  lookup->null_key_rows > 0 ? 1 : 0, out.own_data->as<signed char>(), is_null.as<uint8_t>(), tg_colref(key), float_kind, lookup->nan_key_rows > 0 ? 1 : 0);
        tgpu_column bm;
        memset(&bm, 0, sizeof(bm));
        bm.type = TGPU_INT8;
        bm.flags = TGPU_COL_NULLS_BYTEMAP;
        bm.length = n;
        bm.data = is_null.p;
        bm.validity = is_null.as<uint8_t>();
        DevColumn packed;
        TG_TRY(tg_ingest_column(ctx, &bm, true, &packed));
        out.own_validity = packed.own_validity;
        out.validity = packed.validity;
        DevPage outp;
        outp.rows = n;
        outp.cols = in.cols;            // inputPage.appendColumn(...): the input blocks pass through
        outp.cols.push_back(std::move(out));
        TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        pending = tg_make_owned_page(std::move(outp));
        for (int32_t c = 0; c + 1 < (int32_t)pending->page.cols.size(); c++) pending->passthrough.push_back(c);
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

// rows of the build side whose join key is NULL (HashSemiJoin's containsNull; never matched, so always outer rows)
static int lookup_count_null_keys(tgpu_ctx* ctx, tgpu_lookup* lk)
{
    if (lk->null_key_rows >= 0) return TGPU_OK;
    lk->null_key_rows = 0;
    if (lk->positions == 0) return TGPU_OK;
    const DevColumn* key = lk->generic ? (lk->build_keys.empty() ? nullptr : &lk->build_keys[0]) : (lk->store.cols.empty() ? nullptr : &lk->store.cols[0]);
    if (!key || !key->validity) return TGPU_OK;
    DevBuf cnt;
    TG_TRY(cnt.alloc(ctx, 8));
    TG_CUDA(ctx, cudaMemsetAsync(cnt.p, 0, 8, ctx->stream));
    TG_LAUNCH(ctx, count_nulls_kernel, tg_grid(ctx, lk->positions, 1024, 8), 256, 0, key->validity, lk->positions, cnt.as<unsigned long long>());
    int64_t v = 0;
    TG_TRY(tg_read_i64(ctx, cnt.p, &v));
    lk->null_key_rows = v;
    return TGPU_OK;
}

static int lookup_count_nan_keys(tgpu_ctx* ctx, tgpu_lookup* lk)
{
    if (lk->nan_key_rows >= 0) return TGPU_OK;
    lk->nan_key_rows = 0;
    if (lk->positions == 0) return TGPU_OK;
    const DevColumn* key = lk->generic ? (lk->build_keys.empty() ? nullptr : &lk->build_keys[0]) : (lk->store.cols.empty() ? nullptr : &lk->store.cols[0]);
    const int float_kind = !key ? 0 : key->type == TGPU_FLOAT64 ? 1 : key->type == TGPU_FLOAT32 ? 2 : 0;
    if (!float_kind) return TGPU_OK;
    DevBuf cnt;
    TG_TRY(cnt.alloc(ctx, 8));
    TG_CUDA(ctx, cudaMemsetAsync(cnt.p, 0, 8, ctx->stream));
    TG_LAUNCH(ctx, count_nan_keys_kernel, tg_grid(ctx, lk->positions, 1024, 8), 256, 0, tg_colref(*key), float_kind, lk->positions, cnt.as<unsigned long long>());
    int64_t v = 0;
    TG_TRY(tg_read_i64(ctx, cnt.p, &v));
    lk->nan_key_rows = v;
    return TGPU_OK;
}

}  // namespace

// ------------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------------
extern "C" int tgpu_join_build_create(tgpu_ctx* ctx, const tgpu_join_build_spec* spec, tgpu_op** out)
{
    if (!ctx || !spec || !out) return TGPU_ERR_INVALID_ARGUMENT;
    if (spec->num_key_channels < 1 || spec->num_key_channels > tg::MAX_KEY_COLS)
        return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "GPU hash join supports 1..%d join channels (got %d)", tg::MAX_KEY_COLS, spec->num_key_channels);
    JoinBuildOp* op = new JoinBuildOp(ctx);
    op->key_channels.assign(spec->key_channels, spec->key_channels + spec->num_key_channels);
    op->output_channels.assign(spec->output_channels, spec->output_channels + spec->num_output_channels);
    *out = op;
    return TGPU_OK;
}

extern "C" int tgpu_join_build_create_filtered(tgpu_ctx* ctx, const tgpu_join_build_spec* spec, const tgpu_expr_program* filter, int32_t num_build_channels,
                                               tgpu_op** out)
{
    if (!ctx || !spec || !filter || !out) return TGPU_ERR_INVALID_ARGUMENT;
    DProgram prog;
    TG_TRY(join_filter_compile(ctx, filter, num_build_channels, &prog));
    std::vector<int32_t> used;
    for (int i = 0; i < prog.num_filter_insns; i++) {
        const tg::DOperand* ops[3] = {&prog.insns[i].a, &prog.insns[i].b, &prog.insns[i].c};
        for (auto* o : ops)
            if (o->kind == TGPU_OPND_COLUMN && std::find(used.begin(), used.end(), o->index) == used.end()) used.push_back(o->index);
    }
    std::sort(used.begin(), used.end());
    tgpu_op* base = nullptr;
    TG_TRY(tgpu_join_build_create(ctx, spec, &base));
    std::unique_ptr<JoinBuildOp> op(static_cast<JoinBuildOp*>(base));
    for (int32_t ch : used) {
        if (ch >= num_build_channels) continue;
        if (op->kept_at(ch) == (size_t)-1) op->extra_channels.push_back(ch);
    }
    op->has_filter = true;
    op->filter = prog;
    op->num_build_channels = num_build_channels;
    op->filter_channels = used;
    *out = op.release();
    return TGPU_OK;
}

extern "C" int tgpu_join_build_get_lookup(tgpu_op* build, tgpu_lookup** out)
{
    JoinBuildOp* op = dynamic_cast<JoinBuildOp*>(build);
    if (!op || !out) return TGPU_ERR_INVALID_ARGUMENT;
    if (!op->lookup) return tg_fail(op->ctx, TGPU_ERR_ILLEGAL_STATE, "lookup source is not built yet: call finish() first");
    op->lookup->refs++;
    *out = op->lookup;
    return TGPU_OK;
}

extern "C" void tgpu_lookup_release(tgpu_lookup* lookup)
{
    if (!lookup) return;
    if (--lookup->refs == 0) {
        cudaSetDevice(lookup->ctx->device);
        delete lookup;
    }
}

extern "C" int64_t tgpu_lookup_position_count(const tgpu_lookup* lookup) { return lookup ? lookup->positions : 0; }

extern "C" int64_t tgpu_lookup_memory_bytes(const tgpu_lookup* lookup)
{
    if (!lookup) return 0;
    int64_t b = (int64_t)lookup->table.bytes + (int64_t)lookup->links.bytes + lookup->store.memory_bytes() + lookup->filter_extra_bytes;
    for (auto& s : lookup->by_slot) b += (int64_t)s.bytes;
    b += (int64_t)lookup->wide.bytes + (int64_t)lookup->keyed.bytes;
    return b;
}

extern "C" int tgpu_lookup_has_duplicates(const tgpu_lookup* lookup) { return lookup && lookup->has_dups ? 1 : 0; }

extern "C" int tgpu_join_probe_create(tgpu_ctx* ctx, const tgpu_join_probe_spec* spec, tgpu_lookup* lookup, tgpu_op** out)
{
    if (!ctx || !spec || !lookup || !out) return TGPU_ERR_INVALID_ARGUMENT;
    if (spec->num_key_channels < 1 || spec->num_key_channels > tg::MAX_KEY_COLS)
        return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "GPU hash join supports 1..%d join channels (got %d)", tg::MAX_KEY_COLS, spec->num_key_channels);
    if (spec->join_type < TGPU_JOIN_INNER || spec->join_type > TGPU_JOIN_FULL_OUTER) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "bad join type %d", spec->join_type);
    if (spec->join_type == TGPU_JOIN_LOOKUP_OUTER || spec->join_type == TGPU_JOIN_FULL_OUTER) {
        // OuterLookupSourceSupplier: the visited-positions array is shared by every probe of this lookup source
        TG_CUDA(ctx, cudaSetDevice(ctx->device));
        std::lock_guard<std::mutex> guard(lookup->visited_lock);
        if (!lookup->visited.p && lookup->positions > 0) {
            TG_TRY(lookup->visited.alloc(ctx, (size_t)lookup->positions));
            TG_CUDA(ctx, cudaMemsetAsync(lookup->visited.p, 0, (size_t)lookup->positions, ctx->stream));
            TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        }
    }
    JoinProbeOp* op = new JoinProbeOp(ctx, lookup);
    op->join_type = spec->join_type;
    op->single_match = spec->output_single_match;
    op->key_channels.assign(spec->key_channels, spec->key_channels + spec->num_key_channels);
    op->output_channels.assign(spec->output_channels, spec->output_channels + spec->num_output_channels);
    *out = op;
    return TGPU_OK;
}

extern "C" int tgpu_join_outer_create(tgpu_ctx* ctx, tgpu_lookup* lookup, const int32_t* probe_output_types, int32_t num_probe_outputs, tgpu_op** out)
{
    if (!ctx || !lookup || !out || num_probe_outputs < 0 || (num_probe_outputs > 0 && !probe_output_types)) return TGPU_ERR_INVALID_ARGUMENT;
    JoinOuterOp* op = new JoinOuterOp(ctx, lookup);
    op->probe_types.assign(probe_output_types, probe_output_types + num_probe_outputs);
    *out = op;
    return TGPU_OK;
}

extern "C" int tgpu_semi_join_create(tgpu_ctx* ctx, tgpu_lookup* lookup, int32_t probe_join_channel, tgpu_op** out)
{
    if (!ctx || !lookup || !out) return TGPU_ERR_INVALID_ARGUMENT;
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    if (lookup->generic && lookup->build_keys.size() != 1) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "a semi-join set has one channel");
    if (lookup->has_filter) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "a semi-join set (ChannelSet) has no join filter");
    TG_TRY(lookup_count_null_keys(ctx, lookup));
    TG_TRY(lookup_count_nan_keys(ctx, lookup));
    SemiJoinOp* op = new SemiJoinOp(ctx, lookup);
    op->probe_channel = probe_join_channel;
    *out = op;
    return TGPU_OK;
}

extern "C" int tgpu_lookup_key_domain(tgpu_ctx* ctx, tgpu_lookup* lookup, int64_t max_values, int64_t* min_out, int64_t* max_out, int64_t* distinct_out,
                                      int64_t* values_out, int32_t* has_null_out)
{
    if (!ctx || !lookup || !min_out || !max_out || !distinct_out || max_values < 0 || (max_values > 0 && !values_out)) return TGPU_ERR_INVALID_ARGUMENT;
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    if (lookup->generic || lookup->key_type == TGPU_FLOAT64 || lookup->key_type == TGPU_UTF8)
        return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "key domains are collected for single BIGINT-family join keys only");
    TG_TRY(lookup_count_null_keys(ctx, lookup));
    if (has_null_out) *has_null_out = lookup->null_key_rows > 0;
    const int64_t slots = (int64_t)lookup->geo.mask + 1;
    DevBuf state, vals;
    TG_TRY(state.alloc(ctx, 24));
    TG_TRY(vals.alloc(ctx, (size_t)std::max<int64_t>(max_values, 1) * 8));
    long long init[3] = {INT64_MAX, INT64_MIN, 0};
    TG_CUDA(ctx, cudaMemcpyAsync(state.p, init, 24, cudaMemcpyHostToDevice, ctx->stream));
    if (lookup->table.p && lookup->positions > 0)
        TG_LAUNCH(ctx, join_key_domain_kernel, tg_grid(ctx, slots, 1024, 8), 256, 0, lookup->table.as<JoinSlot>(), slots, max_values, state.as<long long>(),
                  (unsigned long long*)(state.as<long long>() + 2), vals.as<long long>());
    long long res[3];
    TG_CUDA(ctx, cudaMemcpyAsync(res, state.p, 24, cudaMemcpyDeviceToHost, ctx->stream));
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    int64_t distinct = res[2];
    int64_t got = std::min<int64_t>(distinct, max_values);
    if (got > 0) {
        TG_CUDA(ctx, cudaMemcpyAsync(values_out, vals.p, (size_t)got * 8, cudaMemcpyDeviceToHost, ctx->stream));
        TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    if (lookup->special_head >= 0) {       // the key INT64_MIN lives beside the table
        if (distinct < max_values) values_out[distinct] = INT64_MIN;
        distinct++;
        res[0] = INT64_MIN;
        if (res[1] < res[0]) res[1] = INT64_MIN;
    }
    if (distinct <= max_values && distinct > 0) std::sort(values_out, values_out + distinct);
    *min_out = res[0];
    *max_out = res[1];
    *distinct_out = distinct;
    return TGPU_OK;
}

extern "C" int tgpu_join_probe_set_passthrough_by_reference(tgpu_op* op, int32_t enable)
{
    JoinProbeOp* p = dynamic_cast<JoinProbeOp*>(op);
    if (!p) return TGPU_ERR_INVALID_ARGUMENT;
    p->by_reference = enable != 0;
    return TGPU_OK;
}

extern "C" int tgpu_lookup_get_join_positions(tgpu_ctx* ctx, const tgpu_lookup* lookup, const tgpu_page* keys_page, int32_t* out_positions)
{
    if (!ctx || !lookup || !keys_page || !out_positions) return TGPU_ERR_INVALID_ARGUMENT;
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    bool device = (keys_page->flags & TGPU_PAGE_DEVICE) != 0;
    int64_t n = keys_page->num_rows;
    if (lookup->generic) {
        DevPage kp;
        TG_TRY(tg_ingest_page(ctx, keys_page, &kp));
        std::vector<const DevColumn*> refs;
        for (auto& c : kp.cols) refs.push_back(&c);
        if (device) return lookup_positions_generic(ctx, lookup, refs, n, out_positions);
        DevBuf gout;
        TG_TRY(gout.alloc(ctx, (size_t)std::max<int64_t>(n, 1) * 4));
        TG_TRY(lookup_positions_generic(ctx, lookup, refs, n, gout.as<int>()));
        TG_CUDA(ctx, cudaMemcpyAsync(out_positions, gout.p, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
        TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        return TGPU_OK;
    }
    if (keys_page->num_columns != 1) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "exactly one key column expected");
    DevColumn key;
    TG_TRY(tg_ingest_column(ctx, &keys_page->columns[0], device, &key));
    if (device) return lookup_positions(ctx, lookup, key, out_positions);
    DevBuf out;
    TG_TRY(out.alloc(ctx, (size_t)n * 4));
    TG_TRY(lookup_positions(ctx, lookup, key, out.as<int>()));
    TG_CUDA(ctx, cudaMemcpyAsync(out_positions, out.p, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return TGPU_OK;
}

extern "C" int tgpu_lookup_copy_position_links(tgpu_ctx* ctx, const tgpu_lookup* lookup, int32_t* out_links_host)
{
    if (!ctx || !lookup || !out_links_host) return TGPU_ERR_INVALID_ARGUMENT;
    if (!lookup->has_dups) {
        for (int64_t i = 0; i < lookup->positions; i++) out_links_host[i] = -1;
        return TGPU_OK;
    }
    TG_CUDA(ctx, cudaMemcpyAsync(out_links_host, lookup->links.p, (size_t)lookup->positions * 4, cudaMemcpyDeviceToHost, ctx->stream));
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return TGPU_OK;
}

extern "C" int tgpu_jit_selftest_join_filter(const tgpu_expr_program* program, int32_t num_build_channels, const int32_t* channel_types, int32_t num_channels,
                                             uint32_t nullable_mask, int64_t* cubin_bytes, char* source_out, int64_t source_cap)
{
    if (!program || !channel_types || !cubin_bytes || num_channels < 0) return TGPU_ERR_INVALID_ARGUMENT;
    tgpu_ctx fake;
    DProgram prog;
    int st = join_filter_compile(&fake, program, num_build_channels, &prog);
    if (st != TGPU_OK) return st;
    bool used[TGPU_MAX_CHANNELS] = {false};
    tg::fp_mark_columns(prog, 0, prog.num_filter_insns, used);
    for (int c = num_channels; c < TGPU_MAX_CHANNELS; c++)
        if (used[c]) return TGPU_ERR_INVALID_ARGUMENT;     // outside the layout
    return tg::jit_selftest(channel_types, num_channels, [&](const int* elems) {
        return gen_join_filter_source(prog, num_build_channels, elems, std::min<int32_t>(num_channels, TGPU_MAX_CHANNELS), nullable_mask);
    }, cubin_bytes, source_out, source_cap);
}
