// groupby.cu — HashAggregationOperator / GroupByHash / grouped accumulators for sm_90a.
//
// Reference semantics reproduced:
//   - GroupByHash contract (M/operator/GroupByHash.java:118-125): group ids are dense, 0-based and assigned in
//     first-appearance order over the whole input stream; a NULL key is an ordinary group
//     (M/operator/BigintGroupByHash.java:193-200); DOUBLE keys group by IDENTICAL (NaN == NaN, -0 == +0,
//     S/type/DoubleType.java:218-229) and the stored key is the first one seen.
//   - accumulators (M/operator/aggregation/GroupedAggregator.java:77-117 + the @InputFunctions cited in
//     include/trino_gpu.h): state[groupId] op= value, NULL inputs skipped, AggregationMask honoured.
//   - output (InMemoryHashAggregationBuilder.buildResult :229-300): key columns then one column per aggregate
//     (PARTIAL: the intermediate state columns), rows in group-id order.
//   - HashAggregationOperator state machine (M/operator/HashAggregationOperator.java:346-498): accumulate until
//     finish(); a PARTIAL step flushes when its memory exceeds max_partial_bytes (:351-353,478-483).
//
// Two device paths, chosen at run time:
//   S (small)  : one pass, no group-id array in HBM.  Every CTA keeps a shared-memory key table of L slots and
//                per-thread private accumulators [slot][acc][thread] (no atomics, no bank conflicts); a
//                fixed-order in-CTA reduction and a single-CTA merge kernel fold the CTA partials into the
//                operator state, ranking new groups by their first row so ids come out in first-seen order.
//                The optional `pre` program (filter + projections) is evaluated in the same kernel, so
//                projected columns never reach HBM (TPC-H Q1 shape).  Results are run-to-run deterministic.
//   G (general): global open-addressing table {key, gid, first_row}; provisional inserts record the minimum
//                row per new key, new groups are ranked with a prefix sum over "representative row" flags,
//                then accumulators are updated with L2 atomics (RED.ADD.F64 / atomicAdd / atomicMin/Max).
// Keys are packed exactly into one 64-bit word (single key of any fixed width, or several narrow keys with
// one null bit each, <= 63 bits); other key shapes return NOT_SUPPORTED so the caller keeps the Java operator.
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#include <algorithm>
#include <map>

#include "expr.cuh"
#include "jit.cuh"
#include "multisplit.cuh"
#include "strdict.cuh"

#include <atomic>
#include <mutex>

// PartialAggregationController (M/operator/aggregation/partial/PartialAggregationController.java:35-103), shared by the drivers of one
// plan node: a mutex for onFlush, an atomic flag for the readers (the reference's synchronized method + volatile field)
struct tgpu_partial_agg_controller {
    std::mutex mu;
    int64_t max_partial_bytes = 0;
    double threshold = 0;
    std::atomic<bool> disabled{false};
    int64_t total_bytes = 0, total_rows = 0, total_unique = 0;
};

namespace {

using namespace tg;

constexpr unsigned long long EMPTY_KEY = 0x8000000000000000ULL;
constexpr long long NO_ROW = 0x7FFFFFFFFFFFFFFFLL;
constexpr int MAX_KEYS = 4;
constexpr int MAX_SRCS = 32;
constexpr int MAX_ACCS = 40;   // (a FINAL decimal sum alone takes 9: four 128-bit pairs and its non-NULL counter)
constexpr int S_THREADS = TGD_S_THREADS;
static_assert(TGD_MAX_CHANNELS == TGPU_MAX_CHANNELS, "channel limits differ");
constexpr int S_GMAX = 64;             // regular groups the S path can hold (+2 special)
constexpr int S_SPECIAL_NULL = 0;      // special slot for the NULL key (single-key case)
constexpr int S_SPECIAL_SENTINEL = 1;  // special slot for a key whose bits equal EMPTY_KEY

struct SrcRef {
    int32_t is_temp;   // 0: channel of the input page, 1: VM temporary of the pre program
    int32_t index;
    int32_t vtype;     // temps only
    int32_t pad;
};

struct AccDesc {
    int32_t kind;
    int32_t src;       // index into srcs, -1 for ACC_ROWS
    int32_t mask;      // index into srcs of the BOOLEAN mask, or -1
    int32_t pad;
};

struct AggPlan {
    int32_t num_keys;
    int32_t key_src[MAX_KEYS];
    int32_t key_bits[MAX_KEYS];      // payload bits per key in the packed word (multi-key case)
    int32_t key_is_double[MAX_KEYS];
    int32_t num_srcs;
    SrcRef srcs[MAX_SRCS];
    int32_t num_accs;
    AccDesc accs[MAX_ACCS];
    int32_t has_pre;
    int32_t key_hashed;              // keys do not pack into 63 bits: the table is keyed by a 64-bit fingerprint of the tuple,
                                     // every row is verified against the stored key values (path G only)
};

// which accumulators the specialised kernel really maintains: a NONNULL counter over an input that cannot be
// NULL in this page is the row counter of the same mask, so it is dropped from the kernel and read back from the
// ROWS accumulator when the CTA partials are merged.
struct AccMap {
    int32_t compact_count;
    int32_t of_plan[MAX_ACCS];    // plan accumulator -> index in the kernel's compact accumulator space
};


#if defined(__CUDACC__)
struct Fetched {
    long long bits;
    bool is_null;
};

__device__ __forceinline__ Fetched fetch_src(const SrcRef& s, const DColumns& cols, int64_t row, const int64_t* temps, int tstride, uint32_t nullbits)
{
    Fetched f;
    if (s.is_temp) {
        f.bits = temps[s.index * tstride];
        f.is_null = (nullbits >> s.index) & 1;
    }
    else {
        const ColRef& c = cols.cols[s.index];
        f.is_null = !tg_valid(c.validity, row);
        f.bits = tg_load_i64(c, row);
    }
    return f;
}

// IDENTICAL-canonical bits of a key value: -0.0 -> +0.0, every NaN -> one NaN (S/type/DoubleType.java:218-229)
__device__ __forceinline__ unsigned long long canonical_key_bits(long long bits, int is_double)
{
    unsigned long long u = (unsigned long long)bits;
    if (is_double) {
        if ((u << 1) == 0) u = 0;
        if ((u & 0x7FFFFFFFFFFFFFFFULL) > 0x7FF0000000000000ULL) u = 0x7FF8000000000000ULL;
    }
    return u;
}

// canonical packed key of a row.  Returns the special-slot index (0 NULL key, 1 sentinel-valued key) or -1.
// `attempt` (hashed composite keys only): which of the independent 64-bit hash functions of the key tuple to use - a tuple whose
// attempt-0 hash is already owned by a different tuple lives under its attempt-1 hash, and so on (run_general_ids)
__device__ __forceinline__ int pack_key(const AggPlan& plan, const DColumns& cols, int64_t row, const int64_t* temps, int tstride, uint32_t nullbits,
                                        unsigned long long* out, int attempt = 0)
{
    if (plan.num_keys == 1) {
        Fetched f = fetch_src(plan.srcs[plan.key_src[0]], cols, row, temps, tstride, nullbits);
        if (f.is_null) return S_SPECIAL_NULL;
        unsigned long long u = (unsigned long long)f.bits;
        if (plan.key_is_double[0]) {
            if ((u << 1) == 0) u = 0;
            if ((u & 0x7FFFFFFFFFFFFFFFULL) > 0x7FF0000000000000ULL) u = 0x7FF8000000000000ULL;
        }
        if (u == EMPTY_KEY) return S_SPECIAL_SENTINEL;
        *out = u;
        return -1;
    }
    if (plan.key_hashed) {
        unsigned long long h = 0x9E3779B97F4A7C15ULL + (unsigned long long)attempt * 0xD1B54A32D192ED03ULL;
        for (int k = 0; k < plan.num_keys; k++) {
            Fetched f = fetch_src(plan.srcs[plan.key_src[k]], cols, row, temps, tstride, nullbits);
            unsigned long long u = f.is_null ? 0ULL : canonical_key_bits(f.bits, plan.key_is_double[k]);
            h = murmur3_mix(h ^ u) * 31ULL + (f.is_null ? 1ULL : 0ULL);
        }
        if (h == EMPTY_KEY) return S_SPECIAL_SENTINEL;
        *out = h;
        return -1;
    }
    unsigned long long pk = 0;
    int shift = 0;
    for (int k = 0; k < plan.num_keys; k++) {
        Fetched f = fetch_src(plan.srcs[plan.key_src[k]], cols, row, temps, tstride, nullbits);
        int bits = plan.key_bits[k];
        unsigned long long field = f.is_null ? 1ULL : (((unsigned long long)f.bits & ((1ULL << bits) - 1)) << 1);
        pk |= field << shift;
        shift += bits + 1;
    }
    *out = pk;   // <= 63 bits used: can never equal EMPTY_KEY
    return -1;
}

__device__ __forceinline__ bool mask_selected(const AggPlan& plan, int mask, const DColumns& cols, int64_t row, const int64_t* temps, int tstride, uint32_t nullbits)
{
    if (mask < 0) return true;
    Fetched m = fetch_src(plan.srcs[mask], cols, row, temps, tstride, nullbits);
    return !m.is_null && m.bits != 0;
}

// =====================================================================================================
// path S
// =====================================================================================================
// dynamic shared memory layout:
//   unsigned long long tkeys[L]; long long lfirst[L+2]; unsigned long long acc[(L+2)*A*T]; int64 temps[8*T] (pre only)
__global__ void __launch_bounds__(S_THREADS) agg_small_kernel(AggPlan plan, DColumns cols, const DProgram* __restrict__ prog, int64_t n, int L,
                                                             SmallOut out)
{
    extern __shared__ unsigned long long smem_u64[];
    const int A = plan.num_accs;
    const int T = S_THREADS;
    unsigned long long* tkeys = smem_u64;
    long long* lfirst = (long long*)(tkeys + L);
    unsigned long long* acc = (unsigned long long*)(lfirst + L + 2);
    int64_t* temps_base = (int64_t*)(acc + (size_t)(L + 2) * A * T);
    int64_t* temps = temps_base + threadIdx.x;
    const int tid = threadIdx.x;

    for (int i = tid; i < L; i += T) tkeys[i] = EMPTY_KEY;
    for (int i = tid; i < L + 2; i += T) lfirst[i] = NO_ROW;
    for (int s = 0; s < L + 2; s++)
        for (int a = 0; a < A; a++) acc[((size_t)s * A + a) * T + tid] = acc_init(plan.accs[a].kind);
    __shared__ int s_overflow;
    if (tid == 0) s_overflow = 0;
    __syncthreads();

    unsigned long long seen = 0;
    uint32_t err = 0, ignored = 0;
    const long long hi_off = T;   // HI half is the next accumulator: ((s*A + a+1)*T + tid) - ((s*A + a)*T + tid)
    int64_t stride = (int64_t)gridDim.x * T;
    for (int64_t row = (int64_t)blockIdx.x * T + tid; row < n; row += stride) {
        uint32_t nb = 0;
        if (plan.has_pre) {
            if (prog->filter_temp >= 0) {
                nb = vm_run(prog, 0, prog->num_filter_insns, cols, row, temps, T, 0, &ignored);
                err |= ignored;
                int ft = prog->filter_temp;
                bool sel = !((nb >> ft) & 1) && temps[ft * T] != 0;
                if (!sel) continue;
            }
            nb = vm_run(prog, prog->num_filter_insns, prog->num_insns, cols, row, temps, T, nb, &err);
        }
        unsigned long long pk = 0;
        int special = pack_key(plan, cols, row, temps, T, nb, &pk);
        int slot;
        if (special >= 0) slot = L + special;
        else {
            int h = (int)(murmur3_mix(pk) & (unsigned long long)(L - 1));
            slot = -1;
            for (int probe = 0; probe < L; probe++) {
                unsigned long long cur = tkeys[h];
                if (cur == EMPTY_KEY) cur = atomicCAS(&tkeys[h], EMPTY_KEY, pk);
                if (cur == EMPTY_KEY || cur == pk) { slot = h; break; }
                h = (h + 1) & (L - 1);
            }
            if (slot < 0) { s_overflow = 1; break; }   // more distinct keys in this CTA than L: host switches to path G
        }
        if (!((seen >> slot) & 1)) {
            seen |= 1ULL << slot;
            atomicMin(&lfirst[slot], (long long)row);   // rows of one thread ascend: its first hit is its minimum
        }
        int last_src = -2;
        Fetched v;
        v.bits = 0; v.is_null = false;
        for (int a = 0; a < A; a++) {
            const AccDesc& d = plan.accs[a];
            if (d.kind == ACC_SUM_I64_HI) continue;
            if (!mask_selected(plan, d.mask, cols, row, temps, T, nb)) continue;
            if (d.src >= 0 && d.src != last_src) { v = fetch_src(plan.srcs[d.src], cols, row, temps, T, nb); last_src = d.src; }
            if (d.kind != ACC_ROWS && v.is_null) continue;
            acc_update_private(d.kind, &acc[((size_t)slot * A + a) * T + tid], hi_off, v.bits);
        }
    }
    if (err) atomicOr(out.err, err);
    __syncthreads();
    if (s_overflow) {
        if (tid == 0) *out.overflow = 1;
        return;
    }

    // fixed-order reduction of the T private copies of every (slot, acc): lane-sequential then xor tree
    const int warp = tid >> 5, lane = tid & 31, nwarps = T >> 5;
    const size_t b = blockIdx.x;
    for (int pair = warp; pair < (L + 2) * A; pair += nwarps) {
        int s = pair / A, a = pair % A;
        int kind = plan.accs[a].kind;
        if (kind == ACC_SUM_I64_HI) continue;   // reduced together with its LO half
        if (lfirst[s] == NO_ROW) continue;
        const unsigned long long* p = &acc[((size_t)s * A + a) * T];
        if (kind == ACC_SUM_I64_LO) {
            const unsigned long long* ph = p + T;
            unsigned long long lo = 0, hi = 0;
            for (int t = lane; t < T; t += 32) { unsigned long long o = lo; lo += p[t]; hi += ph[t] + (lo < o ? 1 : 0); }
            for (int off = 16; off > 0; off >>= 1) {
                unsigned long long ol = __shfl_xor_sync(0xffffffffu, lo, off), oh = __shfl_xor_sync(0xffffffffu, hi, off);
                unsigned long long o = lo; lo += ol; hi += oh + (lo < o ? 1 : 0);
            }
            if (lane == 0) {
                out.blk_acc[(b * (L + 2) + s) * A + a] = lo;
                out.blk_acc[(b * (L + 2) + s) * A + a + 1] = hi;
            }
        }
        else {
            unsigned long long r = acc_init(kind);
            for (int t = lane; t < T; t += 32) r = acc_combine(kind, r, p[t]);
            for (int off = 16; off > 0; off >>= 1) r = acc_combine(kind, r, __shfl_xor_sync(0xffffffffu, r, off));
            if (lane == 0) out.blk_acc[(b * (L + 2) + s) * A + a] = r;
        }
    }
    for (int s = tid; s < L + 2; s += T) {
        out.blk_first[b * (L + 2) + s] = lfirst[s];
        if (s < L) out.blk_keys[b * L + s] = tkeys[s];
    }
}

// operator state shared by both paths (device resident)
struct AggState {
    int32_t* count;                   // [0] number of groups, [1] gid of NULL-key group or -1, [2] gid of sentinel-key group or -1
    unsigned long long* keys;         // path S: canonical packed key per gid (cap entries)
    unsigned long long* acc;          // [A][cap]
    long long* keyvals;               // [num_keys][cap] raw first-seen key values
    unsigned char* keynull;           // [num_keys][cap]
    int64_t cap;
};

// single-CTA merge of the CTA partials of one page into the operator state (path S)
__global__ void __launch_bounds__(256) agg_small_merge_kernel(AggPlan plan, DColumns cols, int B, int L, SmallOut part, AggState st, int* __restrict__ blk_ps, AccMap map)
{
    __shared__ unsigned long long pkeys[S_GMAX];
    __shared__ long long pfirst[S_GMAX + 2];
    __shared__ int pgid[S_GMAX + 2];       // gid of the page slot (existing or newly assigned)
    __shared__ int pnew[S_GMAX + 2];
    __shared__ int s_fail;
    const int tid = threadIdx.x, T = blockDim.x;
    const int A = plan.num_accs;
    if (*((volatile int*)part.overflow)) return;   // a CTA ran out of key slots: its partials were never written
    for (int i = tid; i < S_GMAX; i += T) pkeys[i] = EMPTY_KEY;
    for (int i = tid; i < S_GMAX + 2; i += T) { pfirst[i] = NO_ROW; pgid[i] = -1; pnew[i] = 0; }
    if (tid == 0) s_fail = 0;
    __syncthreads();
    // 1. distinct keys of the page with their minimum first row
    const int entries = B * (L + 2);
    for (int e = tid; e < entries; e += T) {
        int b = e / (L + 2), s = e % (L + 2);
        long long first = part.blk_first[(size_t)b * (L + 2) + s];
        int ps = -1;
        if (first != NO_ROW) {
            if (s >= L) ps = S_GMAX + (s - L);
            else {
                unsigned long long key = part.blk_keys[(size_t)b * L + s];
                int h = (int)(murmur3_mix(key) & (S_GMAX - 1));
                for (int probe = 0; probe < S_GMAX; probe++) {
                    unsigned long long cur = pkeys[h];
                    if (cur == EMPTY_KEY) cur = atomicCAS(&pkeys[h], EMPTY_KEY, key);
                    if (cur == EMPTY_KEY || cur == key) { ps = h; break; }
                    h = (h + 1) & (S_GMAX - 1);
                }
                if (ps < 0) s_fail = 1;
            }
            if (ps >= 0) atomicMin(&pfirst[ps], first);
        }
        blk_ps[e] = ps;
    }
    __syncthreads();
    if (s_fail) { if (tid == 0) *part.overflow = 1; return; }
    // 2. match page slots against the state
    const int count = st.count[0];
    for (int ps = tid; ps < S_GMAX + 2; ps += T) {
        if (pfirst[ps] == NO_ROW) continue;
        int gid = -1;
        if (ps >= S_GMAX) gid = st.count[1 + (ps - S_GMAX)];
        else {
            unsigned long long key = pkeys[ps];
            for (int g = 0; g < count; g++)
                if (st.keys[g] == key && g != st.count[1] && g != st.count[2]) { gid = g; break; }
        }
        pgid[ps] = gid;
        pnew[ps] = gid < 0 ? 1 : 0;
    }
    __syncthreads();
    // 3. new groups get ids in first-row order
    int my_new = 0;
    for (int ps = tid; ps < S_GMAX + 2; ps += T) my_new += pnew[ps];
    __shared__ int s_total_new;
    if (tid == 0) s_total_new = 0;
    __syncthreads();
    if (my_new) atomicAdd(&s_total_new, my_new);
    __syncthreads();
    const int total_new = s_total_new;
    if ((int64_t)count + total_new > st.cap) { if (tid == 0) *part.overflow = 1; return; }
    for (int ps = tid; ps < S_GMAX + 2; ps += T) {
        if (!pnew[ps]) continue;
        int rank = 0;
        for (int q = 0; q < S_GMAX + 2; q++)
            if (pnew[q] && pfirst[q] < pfirst[ps]) rank++;
        int gid = count + rank;
        pgid[ps] = gid;
        long long row = pfirst[ps];
        if (ps < S_GMAX) st.keys[gid] = pkeys[ps];
        else { st.keys[gid] = EMPTY_KEY; st.count[1 + (ps - S_GMAX)] = gid; }
        for (int k = 0; k < plan.num_keys; k++) {
            const ColRef& c = cols.cols[plan.srcs[plan.key_src[k]].index];   // keys are pass-through channels
            bool isn = !tg_valid(c.validity, row);
            st.keyvals[(size_t)k * st.cap + gid] = isn ? 0 : tg_load_i64(c, row);
            st.keynull[(size_t)k * st.cap + gid] = isn ? 1 : 0;
        }
        for (int a = 0; a < A; a++) st.acc[(size_t)a * st.cap + gid] = acc_init(plan.accs[a].kind);
    }
    __syncthreads();
    // 4. fold CTA partials in CTA order (deterministic)
    for (int pair = tid; pair < (S_GMAX + 2) * A; pair += T) {
        int ps = pair / A, a = pair % A;
        int kind = plan.accs[a].kind;
        if (pfirst[ps] == NO_ROW || kind == ACC_SUM_I64_HI) continue;
        int gid = pgid[ps];
        unsigned long long r = st.acc[(size_t)a * st.cap + gid];
        unsigned long long rh = kind == ACC_SUM_I64_LO ? st.acc[(size_t)(a + 1) * st.cap + gid] : 0;
        for (int b = 0; b < B; b++) {
            for (int s = 0; s < L + 2; s++) {
                if (blk_ps[b * (L + 2) + s] != ps) continue;
                size_t at = ((size_t)b * (L + 2) + s) * map.compact_count + map.of_plan[a];
                if (kind == ACC_SUM_I64_LO) {
                    unsigned long long o = r;
                    r += part.blk_acc[at];
                    rh += part.blk_acc[at + 1] + (r < o ? 1 : 0);
                }
                else r = acc_combine(kind, r, part.blk_acc[at]);
            }
        }
        st.acc[(size_t)a * st.cap + gid] = r;
        if (kind == ACC_SUM_I64_LO) st.acc[(size_t)(a + 1) * st.cap + gid] = rh;
    }
    __syncthreads();
    if (tid == 0) st.count[0] = count + total_new;
}

// =====================================================================================================
// path G
// =====================================================================================================
struct __align__(16) GSlot {
    unsigned long long key;
    int gid;        // -1 until the group is numbered
    int first_row;  // minimum row of the current page that hit this provisional slot
};

struct GSpecial {
    int gid[2];
    int first_row[2];
};

__global__ void g_table_init_kernel(int4* table, int64_t slots)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const int4 empty = make_int4(0, (int)0x80000000, -1, 0x7FFFFFFF);
    for (; i < slots; i += stride) table[i] = empty;
}

// K1: find or provisionally insert the key of every row.  slot_of_row: slot index, or -2-special.
// `budget` new slots may be claimed (reserve-then-claim keeps the load factor bounded); exceeding it sets *overflow.
// `rows` / `attempt`: nullptr = rows [0, n) at attempt 0; else the rows that have to move on to their next hash function
__global__ void __launch_bounds__(256) g_insert_kernel(AggPlan plan, DColumns cols, int64_t n, const int* __restrict__ rows, const unsigned char* __restrict__ attempt,
                                                      GSlot* __restrict__ table, unsigned long long mask,
                                                      GSpecial* __restrict__ special, int* __restrict__ slot_of_row, int* __restrict__ tickets, int budget,
                                                      int* __restrict__ overflow)
{
    int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; idx < n; idx += stride) {
        const int64_t row = rows ? rows[idx] : idx;
        unsigned long long pk = 0;
        int sp = pack_key(plan, cols, row, nullptr, 0, 0, &pk, attempt ? attempt[row] : 0);
        if (sp >= 0) {
            if (special->gid[sp] < 0) atomicMin(&special->first_row[sp], (int)row);
            slot_of_row[row] = -2 - sp;
            continue;
        }
        unsigned long long pos = murmur3_mix(pk) & mask;
        bool have_ticket = false;
        int found = -1;
        while (true) {
            unsigned long long cur = *((volatile unsigned long long*)&table[pos].key);
            if (cur == EMPTY_KEY) {
                if (!have_ticket) {
                    if (atomicAdd(tickets, 1) >= budget) { *overflow = 1; break; }
                    have_ticket = true;
                }
                cur = atomicCAS(&table[pos].key, EMPTY_KEY, pk);
                if (cur == EMPTY_KEY) { found = (int)pos; have_ticket = false; break; }   // ticket consumed
            }
            if (cur == pk) { found = (int)pos; break; }
            pos = (pos + 1) & mask;
        }
        if (have_ticket) atomicSub(tickets, 1);
        slot_of_row[row] = found;   // -1 only on overflow (page is re-run after the table grows)
        if (found >= 0 && *((volatile int*)&table[found].gid) < 0) atomicMin(&table[found].first_row, (int)row);
    }
}

// K2: flag the representative (minimum) row of every group that is new in this page
__global__ void g_flag_kernel(int64_t n, const GSlot* __restrict__ table, const GSpecial* __restrict__ special, const int* __restrict__ slot_of_row,
                              unsigned char* __restrict__ flags)
{
    int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; row < n; row += stride) {
        int s = slot_of_row[row];
        bool rep;
        if (s <= -2) { int sp = -2 - s; rep = special->gid[sp] < 0 && special->first_row[sp] == (int)row; }
        else rep = table[s].gid < 0 && table[s].first_row == (int)row;
        flags[row] = rep ? 1 : 0;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) flags[n] = 0;
}

// K3: number the new groups (next_gid + rank of the representative row) and record their key values
__global__ void g_assign_kernel(AggPlan plan, DColumns cols, int64_t n, GSlot* __restrict__ table, GSpecial* __restrict__ special,
                                const int* __restrict__ slot_of_row, const unsigned char* __restrict__ flags, const int* __restrict__ rank, int next_gid, AggState st)
{
    int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; row < n; row += stride) {
        if (!flags[row]) continue;
        int gid = next_gid + rank[row];
        int s = slot_of_row[row];
        if (s <= -2) special->gid[-2 - s] = gid;
        else table[s].gid = gid;
        for (int k = 0; k < plan.num_keys; k++) {
            const ColRef& c = cols.cols[plan.srcs[plan.key_src[k]].index];
            bool isn = !tg_valid(c.validity, row);
            st.keyvals[(size_t)k * st.cap + gid] = isn ? 0 : tg_load_i64(c, row);
            st.keynull[(size_t)k * st.cap + gid] = isn ? 1 : 0;
        }
        for (int a = 0; a < plan.num_accs; a++) st.acc[(size_t)a * st.cap + gid] = acc_init(plan.accs[a].kind);
    }
}

// K4: group id of every row
__global__ void g_gid_kernel(int64_t n, const GSlot* __restrict__ table, const GSpecial* __restrict__ special, const int* __restrict__ slot_of_row,
                             int* __restrict__ gids)
{
    int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; row < n; row += stride) {
        int s = slot_of_row[row];
        gids[row] = s <= -2 ? special->gid[-2 - s] : table[s].gid;
    }
}

// hashed composite keys: a row's slot must hold ITS key tuple - the tuple stored for the slot's group (existing groups) or the tuple
// of the slot's lowest row in this page (new slots).  A row whose tuple differs shares a 64-bit hash with another tuple: it moves
// on to its next hash function (attempt + 1) and is inserted again - full-key comparison and chaining by rehash, like
// FlatHash.valueIdentical on a control-byte hit (M/operator/FlatHash.java:445-469), never a query failure.
__device__ __forceinline__ bool g_same_tuple(const AggPlan& plan, const DColumns& cols, int64_t row, int64_t other_row)
{
    for (int k = 0; k < plan.num_keys; k++) {
        Fetched a = fetch_src(plan.srcs[plan.key_src[k]], cols, row, nullptr, 0, 0), b = fetch_src(plan.srcs[plan.key_src[k]], cols, other_row, nullptr, 0, 0);
        if (a.is_null != b.is_null) return false;
        if (!a.is_null && canonical_key_bits(a.bits, plan.key_is_double[k]) != canonical_key_bits(b.bits, plan.key_is_double[k])) return false;
    }
    return true;
}

__global__ void g_verify_kernel(AggPlan plan, DColumns cols, int64_t n, const int* __restrict__ rows, const GSlot* __restrict__ table,
                                const int* __restrict__ slot_of_row, AggState st, unsigned char* __restrict__ attempt, int* __restrict__ retry, int* __restrict__ retry_count)
{
    int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; idx < n; idx += stride) {
        const int64_t row = rows ? rows[idx] : idx;
        const int s = slot_of_row[row];
        if (s < 0) continue;                       // special groups, or no slot (table growth pending)
        const GSlot slot = table[s];
        bool same = true;
        if (slot.gid >= 0) {
            for (int k = 0; k < plan.num_keys && same; k++) {
                Fetched f = fetch_src(plan.srcs[plan.key_src[k]], cols, row, nullptr, 0, 0);
                bool sn = st.keynull[(size_t)k * st.cap + slot.gid] != 0;
                same = f.is_null == sn;
                if (same && !sn)
                    same = canonical_key_bits(f.bits, plan.key_is_double[k]) == canonical_key_bits(st.keyvals[(size_t)k * st.cap + slot.gid], plan.key_is_double[k]);
            }
        }
        else if (slot.first_row != (int)row) same = g_same_tuple(plan, cols, row, slot.first_row);
        if (!same) {
            attempt[row] = (unsigned char)(attempt[row] + 1);
            retry[atomicAdd(retry_count, 1)] = (int)row;
        }
    }
}

// accumulate with L2 atomics: state[acc][gid] op= value
__global__ void __launch_bounds__(256) g_accumulate_kernel(AggPlan plan, DColumns cols, int64_t n, const int* __restrict__ gids, AggState st)
{
    int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; row < n; row += stride) {
        int gid = gids[row];
        int last_src = -2;
        Fetched v;
        v.bits = 0; v.is_null = false;
        for (int a = 0; a < plan.num_accs; a++) {
            const AccDesc& d = plan.accs[a];
            if (d.kind == ACC_SUM_I64_HI) continue;
            if (!mask_selected(plan, d.mask, cols, row, nullptr, 0, 0)) continue;
            if (d.src >= 0 && d.src != last_src) { v = fetch_src(plan.srcs[d.src], cols, row, nullptr, 0, 0); last_src = d.src; }
            if (d.kind != ACC_ROWS && v.is_null) continue;
            unsigned long long* p = &st.acc[(size_t)a * st.cap + gid];
            switch (d.kind) {
                case ACC_ROWS: case ACC_NONNULL: atomicAdd(p, 1ULL); break;
                case ACC_SUM_F64: atomicAdd((double*)p, __longlong_as_double(v.bits)); break;
                case ACC_SUM_F64_FROM_I64: atomicAdd((double*)p, (double)v.bits); break;
                case ACC_SUM_I64_LO: {
                    unsigned long long add = (unsigned long long)v.bits;
                    unsigned long long old = atomicAdd(p, add);
                    long long carry = (v.bits < 0 ? -1LL : 0LL) + ((old + add) < old ? 1LL : 0LL);
                    if (carry) atomicAdd(p + st.cap, (unsigned long long)carry);
                    break;
                }
                case ACC_MIN_F64: atomicMin(p, f64_order_key(v.bits)); break;
                case ACC_MAX_F64: atomicMax(p, f64_order_key_max(v.bits)); break;
                case ACC_MIN_I64: atomicMin(p, i64_order_key(v.bits)); break;
                case ACC_MAX_I64: atomicMax(p, i64_order_key(v.bits)); break;
                default: break;
            }
        }
    }
}

// re-insert numbered groups into a bigger table
__global__ void g_rehash_kernel(const GSlot* __restrict__ old_table, int64_t old_slots, GSlot* __restrict__ table, unsigned long long mask)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < old_slots; i += stride) {
        GSlot s = old_table[i];
        if (s.key == EMPTY_KEY || s.gid < 0) continue;
        unsigned long long pos = murmur3_mix(s.key) & mask;
        while (atomicCAS(&table[pos].key, EMPTY_KEY, s.key) != EMPTY_KEY) pos = (pos + 1) & mask;
        table[pos].gid = s.gid;
    }
}

// forget provisional (unnumbered) claims of an aborted K1 run
__global__ void g_reset_provisional_kernel(GSlot* __restrict__ table, int64_t slots, GSpecial* special)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < slots; i += stride)
        if (table[i].gid < 0) table[i].first_row = 0x7FFFFFFF;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        for (int sp = 0; sp < 2; sp++) if (special->gid[sp] < 0) special->first_row[sp] = 0x7FFFFFFF;
    }
}

// S -> G migration: insert the S-path groups (ids already final) into the G table
__global__ void g_migrate_kernel(AggState st, GSlot* __restrict__ table, unsigned long long mask, GSpecial* special)
{
    int count = st.count[0];
    for (int g = threadIdx.x; g < count; g += blockDim.x) {
        if (g == st.count[1]) { special->gid[0] = g; continue; }
        if (g == st.count[2]) { special->gid[1] = g; continue; }
        unsigned long long key = st.keys[g];
        unsigned long long pos = murmur3_mix(key) & mask;
        while (atomicCAS(&table[pos].key, EMPTY_KEY, key) != EMPTY_KEY) pos = (pos + 1) & mask;
        table[pos].gid = g;
    }
}

__global__ void relayout_state_kernel(const unsigned long long* __restrict__ old_acc, const long long* __restrict__ old_keyvals,
                                      const unsigned char* __restrict__ old_keynull, int64_t old_cap, int64_t count, int A, int K, AggState st)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < count; i += stride) {
        for (int a = 0; a < A; a++) st.acc[(size_t)a * st.cap + i] = old_acc[(size_t)a * old_cap + i];
        for (int k = 0; k < K; k++) {
            st.keyvals[(size_t)k * st.cap + i] = old_keyvals[(size_t)k * old_cap + i];
            st.keynull[(size_t)k * st.cap + i] = old_keynull[(size_t)k * old_cap + i];
        }
    }
}


// =====================================================================================================
// path G, fused form (packed integer keys): ONE pass per page.  A row finds or inserts its key slot, lowers the
// slot's first-row stamp (global row number) and applies its accumulators with L2 atomics on state indexed BY SLOT —
// no group-id array, no flag/scan/assign passes.  Dense first-seen ids are only needed when rows are emitted: finish()
// compacts the used slots, sorts them by first-row stamp and gathers the state into id order.
// Rows that cannot claim a slot because the table reached its fill limit are appended to a deferred list and replayed
// after the table has grown (their accumulators are untouched, so nothing is counted twice).
// =====================================================================================================
// Slot records are AoS: {key, first-row stamp, accumulator words...} padded to a power-of-two number of 8-byte words (W),
// so one row touches ONE 32/64/128-byte line for its key, stamp and every accumulator (SoA state would scatter a
// row over 4-5 lines: DRAM read-modify-write bound).
__device__ __forceinline__ unsigned long long* gf_rec(unsigned long long* base, int64_t s, int W) { return base + (size_t)s * W; }

// one thread per 16 bytes of the record array: consecutive threads write consecutive addresses (not one thread per record, word
// by word, whose stores do not coalesce)
__global__ void gf_init_kernel(unsigned long long* __restrict__ recs, int64_t cap, int W, AggPlan plan)
{
    __shared__ unsigned long long init[64];      // W <= 64 (2 + MAX_ACCS words, padded to a power of two)
    if (threadIdx.x < 64) {
        int w = threadIdx.x;
        init[w] = w == 0 ? EMPTY_KEY : w == 1 ? (unsigned long long)NO_ROW : (w - 2 < plan.num_accs ? acc_init(plan.accs[w - 2].kind) : 0ULL);
    }
    __syncthreads();
    const int64_t pairs = (cap + 2) * W / 2;            // W is 4, 8 or 16: records are whole 16-byte pairs
    const int pmask = W / 2 - 1;
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    ulonglong2* out = (ulonglong2*)recs;
    for (; i < pairs; i += stride) {
        int w = (int)(i & pmask) * 2;
        out[i] = make_ulonglong2(init[w], init[w + 1]);
    }
}

// Accumulator words inside a fused-G record differ from the canonical (path S / output) meaning in two places, both to
// turn read-modify-write atomics into fire-and-forget reductions and to touch fewer words per row:
//   ACC_NONNULL      holds the number of NULL inputs (usually never incremented); non-null = ROWS(same mask) - that
//   ACC_SUM_I64_LO/HI hold L = sum of the low 32-bit halves and H = sum of (v >> 32): value = H * 2^32 + L, no carry
//                    hand-off between the two words, so both are plain RED.ADD
// gf_gather_kernel converts back when the state is laid out in group-id order.
__device__ __forceinline__ void gf_accumulate(const AggPlan& plan, const DColumns& cols, int64_t row, unsigned long long* __restrict__ acc)
{
    int last_src = -2;
    Fetched v;
    v.bits = 0; v.is_null = false;
    for (int a = 0; a < plan.num_accs; a++) {
        const AccDesc& d = plan.accs[a];
        if (d.kind == ACC_SUM_I64_HI) continue;
        if (!mask_selected(plan, d.mask, cols, row, nullptr, 0, 0)) continue;
        if (d.src >= 0 && d.src != last_src) { v = fetch_src(plan.srcs[d.src], cols, row, nullptr, 0, 0); last_src = d.src; }
        unsigned long long* p = acc + a;
        if (d.kind == ACC_NONNULL) {
            if (v.is_null) atomicAdd(p, 1ULL);
            continue;
        }
        if (d.kind != ACC_ROWS && v.is_null) continue;
        switch (d.kind) {
            case ACC_ROWS: atomicAdd(p, 1ULL); break;
            case ACC_SUM_F64: atomicAdd((double*)p, __longlong_as_double(v.bits)); break;
            case ACC_SUM_F64_FROM_I64: atomicAdd((double*)p, (double)v.bits); break;
            case ACC_SUM_I64_LO:
                atomicAdd(p, (unsigned long long)v.bits & 0xFFFFFFFFULL);
                if ((v.bits >> 32) != 0) atomicAdd(p + 1, (unsigned long long)(v.bits >> 32));
                break;
            case ACC_MIN_F64: atomicMin(p, f64_order_key(v.bits)); break;
            case ACC_MAX_F64: atomicMax(p, f64_order_key_max(v.bits)); break;
            case ACC_MIN_I64: atomicMin(p, i64_order_key(v.bits)); break;
            case ACC_MAX_I64: atomicMax(p, i64_order_key(v.bits)); break;
            default: break;
        }
    }
}

// canonical accumulator words -> fused-G record words (S -> G migration)
__device__ __forceinline__ void gf_encode(const AggPlan& plan, unsigned long long* acc)
{
    for (int a = 0; a < plan.num_accs; a++) {
        const AccDesc& d = plan.accs[a];
        if (d.kind == ACC_NONNULL) {
            for (int r = 0; r < plan.num_accs; r++)
                if (plan.accs[r].kind == ACC_ROWS && plan.accs[r].mask == d.mask) acc[a] = acc[r] - acc[a];
        }
        else if (d.kind == ACC_SUM_I64_LO) {
            unsigned long long lo = acc[a], hi = acc[a + 1];
            acc[a] = lo & 0xFFFFFFFFULL;
            acc[a + 1] = (hi << 32) | (lo >> 32);
        }
    }
}

// fused-G record words -> canonical accumulator words
__device__ __forceinline__ void gf_decode(const AggPlan& plan, unsigned long long* acc)
{
    for (int a = 0; a < plan.num_accs; a++) {
        const AccDesc& d = plan.accs[a];
        if (d.kind == ACC_NONNULL) {
            for (int r = 0; r < plan.num_accs; r++)
                if (plan.accs[r].kind == ACC_ROWS && plan.accs[r].mask == d.mask) acc[a] = acc[r] - acc[a];
        }
        else if (d.kind == ACC_SUM_I64_LO) {
            unsigned long long L = acc[a];
            long long H = (long long)acc[a + 1];
            unsigned long long lo = L + ((unsigned long long)H << 32);
            long long hi = (H >> 32) + (lo < L ? 1 : 0);
            acc[a] = lo;
            acc[a + 1] = (unsigned long long)hi;
        }
    }
}

// `rows` == nullptr: rows [first, first + n) of `cols`; else the deferred row list.  `stamp_rows`: cols is a slice-ordered copy of the
// page, stamp_rows[row] is the row's position in the page (first-row stamps must follow page order)
__global__ void __launch_bounds__(256) gf_page_kernel(AggPlan plan, DColumns cols, int64_t n, const int* __restrict__ rows, int64_t first,
                                                     const int* __restrict__ stamp_rows, long long page_base,
                                                     unsigned long long* __restrict__ recs, int64_t cap, int W, int* __restrict__ tickets, int budget,
                                                     int* __restrict__ deferred)
{
    const unsigned long long mask = (unsigned long long)cap - 1;
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        int64_t row = rows ? rows[i] : first + i;
        unsigned long long pk = 0;
        int sp = pack_key(plan, cols, row, nullptr, 0, 0, &pk);
        int64_t s = -1;
        if (sp >= 0) s = cap + sp;
        else {
            unsigned long long pos = murmur3_mix(pk) & mask;
            bool have_ticket = false;
            while (true) {
                unsigned long long* kp = gf_rec(recs, (int64_t)pos, W);
                unsigned long long cur = *((volatile unsigned long long*)kp);
                if (cur == EMPTY_KEY) {
                    if (!have_ticket) {
                        if (atomicAdd(tickets, 1) >= budget) { atomicSub(tickets, 1); break; }
                        have_ticket = true;
                    }
                    cur = atomicCAS(kp, EMPTY_KEY, pk);
                    if (cur == EMPTY_KEY) { s = (int64_t)pos; have_ticket = false; break; }
                }
                if (cur == pk) { s = (int64_t)pos; break; }
                pos = (pos + 1) & mask;
            }
            if (have_ticket) atomicSub(tickets, 1);
        }
        if (s < 0) { deferred[atomicAdd(tickets + 1, 1)] = (int)row; continue; }
        unsigned long long* r = gf_rec(recs, s, W);
        long long stamp = page_base + (stamp_rows ? (long long)stamp_rows[row] : row);
        if (*((volatile long long*)(r + 1)) > stamp) {
            long long old = atomicMin((long long*)(r + 1), stamp);
            if (old == NO_ROW && s >= cap) atomicAdd(tickets + 2, 1);   // a special (NULL / sentinel key) group came to life
        }
        gf_accumulate(plan, cols, row, r + 2);
    }
}

// Locality pass for tables that do not fit the L2: the slot index's top bits name a contiguous slice of the table, rows are
// grouped by slice (stable, so first-row stamps keep their meaning) and gf_page_kernel then runs slice by slice with its
// read-modify-write traffic staying in the L2 instead of costing a random DRAM sector pair per row and accumulator.
__global__ void __launch_bounds__(256) gf_slice_ids_kernel(AggPlan plan, DColumns cols, int64_t n, int64_t cap, int shift, uint8_t* __restrict__ ids,
                                                          unsigned int* __restrict__ counts /* [64] */)
{
    __shared__ unsigned int sh[64];
    if (threadIdx.x < 64) sh[threadIdx.x] = 0;
    __syncthreads();
    const unsigned long long mask = (unsigned long long)cap - 1;
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        unsigned long long pk = 0;
        int sp = pack_key(plan, cols, i, nullptr, 0, 0, &pk);
        int id = sp >= 0 ? 0 : (int)((murmur3_mix(pk) & mask) >> shift);
        ids[i] = (uint8_t)id;
        unsigned int peers = __match_any_sync(__activemask(), id);
        if ((int)(__ffs(peers) - 1) == (int)(threadIdx.x & 31)) atomicAdd(&sh[id], __popc(peers));
    }
    __syncthreads();
    if (threadIdx.x < 64 && sh[threadIdx.x]) atomicAdd(&counts[threadIdx.x], sh[threadIdx.x]);
}

__global__ void gf_iota_kernel(int* __restrict__ out, int64_t n)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) out[i] = (int)i;
}

// per-chunk histogram form of gf_slice_ids_kernel for the multi-split scatter (chunks as in multisplit.cuh, CTA granularity)
__global__ void __launch_bounds__(XT) gf_slice_hist_kernel(AggPlan plan, DColumns cols, int64_t n, int64_t chunk, int64_t cap, int shift, int S,
                                                          uint8_t* __restrict__ ids, unsigned int* __restrict__ hist /* [chunks][S] */)
{
    // thread-private byte counters (one row of 256 bytes per slice: no atomics, no warp votes - the __match_any_sync + atomicAdd form
    // spent ~56 cycles per warp row), folded into 32-bit totals before a byte can wrap
    __shared__ unsigned int sh[XMAXP];
    __shared__ uint8_t priv[XMAXP * XT];
    for (int i = threadIdx.x; i < S; i += XT) sh[i] = 0;
    for (int i = threadIdx.x; i < XMAXP * XT / 4; i += XT) ((unsigned int*)priv)[i] = 0;
    __syncthreads();
    int since_fold = 0;
    auto fold = [&]() {
        // my 64 counters -> the CTA totals (each thread folds its own column, rotated so that the threads of a warp hit different counters)
        for (int k = 0; k < XMAXP; k++) {
            const int q = (k + threadIdx.x) & (XMAXP - 1);
            if (q < S) {
                const unsigned int c = priv[q * XT + threadIdx.x];
                if (c) { atomicAdd(&sh[q], c); priv[q * XT + threadIdx.x] = 0; }
            }
        }
    };
    const unsigned long long mask = (unsigned long long)cap - 1;
    const int64_t begin = (int64_t)blockIdx.x * chunk, end = min(n, begin + chunk);
    // U rows in flight per thread; a single BIGINT key without NULLs (and no pre-stage) is read straight from its column
    constexpr int U = 8;
    const SrcRef k0 = plan.srcs[plan.key_src[0]];
    const bool plain = plan.num_keys == 1 && !plan.has_pre && !k0.is_temp && !plan.key_is_double[0] && cols.cols[k0.index].elem == 8 && !cols.cols[k0.index].validity;
    const long long* __restrict__ key0 = (const long long*)cols.cols[plain ? k0.index : 0].data;
    for (int64_t base = begin; base < end; base += (int64_t)U * XT) {
        int idv[U];
        if (plain && base + (int64_t)U * XT <= end) {
            long long v[U];
#pragma unroll
            for (int u = 0; u < U; u++) v[u] = key0[base + u * XT + threadIdx.x];
#pragma unroll
            for (int u = 0; u < U; u++)
                idv[u] = (unsigned long long)v[u] == EMPTY_KEY ? 0 : (int)((murmur3_mix((unsigned long long)v[u]) & mask) >> shift);
        }
        else {
#pragma unroll
            for (int u = 0; u < U; u++) {
                int64_t row = base + u * XT + threadIdx.x;
                idv[u] = -1;
                if (row < end) {
                    unsigned long long pk = 0;
                    int sp = pack_key(plan, cols, row, nullptr, 0, 0, &pk);
                    idv[u] = sp >= 0 ? 0 : (int)((murmur3_mix(pk) & mask) >> shift);
                }
            }
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
            int64_t row = base + u * XT + threadIdx.x;
            if (row < end) {
                ids[row] = (uint8_t)idv[u];
                priv[idv[u] * XT + threadIdx.x]++;
            }
        }
        if (++since_fold == 31) {              // 31 trips x 8 rows = 248 < 256
            fold();
            since_fold = 0;
        }
    }
    fold();
    __syncthreads();
    for (int i = threadIdx.x; i < S; i += XT) hist[(size_t)blockIdx.x * S + i] = sh[i];
}

// table growth: move every used record into the bigger table
__global__ void gf_rehash_kernel(const unsigned long long* __restrict__ orecs, int64_t ocap, unsigned long long* __restrict__ recs, int64_t cap, int W, int A)
{
    const unsigned long long mask = (unsigned long long)cap - 1;
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < ocap + 2; i += stride) {
        const unsigned long long* o = orecs + (size_t)i * W;
        int64_t dst;
        if (i >= ocap) dst = cap + (i - ocap);      // special records keep their place after the table
        else {
            unsigned long long k = o[0];
            if (k == EMPTY_KEY) continue;
            unsigned long long pos = murmur3_mix(k) & mask;
            while (atomicCAS(gf_rec(recs, (int64_t)pos, W), EMPTY_KEY, k) != EMPTY_KEY) pos = (pos + 1) & mask;
            dst = (int64_t)pos;
        }
        unsigned long long* r = gf_rec(recs, dst, W);
        for (int w = 1; w < 2 + A; w++) r[w] = o[w];
    }
}

// S -> fused-G migration: groups numbered so far keep their order by getting stamps below every real row
__global__ void gf_migrate_kernel(AggState st, AggPlan plan, unsigned long long* __restrict__ recs, int64_t cap, int W)
{
    const unsigned long long mask = (unsigned long long)cap - 1;
    int count = st.count[0];
    for (int g = threadIdx.x; g < count; g += blockDim.x) {
        int64_t dst;
        if (g == st.count[1]) dst = cap;
        else if (g == st.count[2]) dst = cap + 1;
        else {
            unsigned long long k = st.keys[g];
            unsigned long long pos = murmur3_mix(k) & mask;
            while (atomicCAS(gf_rec(recs, (int64_t)pos, W), EMPTY_KEY, k) != EMPTY_KEY) pos = (pos + 1) & mask;
            dst = (int64_t)pos;
        }
        unsigned long long* r = gf_rec(recs, dst, W);
        r[1] = (unsigned long long)((long long)g - (long long)count - 1);   // negative, ascending with the existing id
        unsigned long long w[MAX_ACCS];
        for (int a = 0; a < plan.num_accs; a++) w[a] = st.acc[(size_t)a * st.cap + g];
        gf_encode(plan, w);
        for (int a = 0; a < plan.num_accs; a++) r[2 + a] = w[a];
    }
}

__global__ void gf_used_flags_kernel(const unsigned long long* __restrict__ recs, int64_t n, int W, unsigned char* __restrict__ flags)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) flags[i] = (long long)recs[(size_t)i * W + 1] != NO_ROW ? 1 : 0;
}

__global__ void gf_sort_keys_kernel(const unsigned long long* __restrict__ recs, int W, const int* __restrict__ slots, int64_t G, unsigned long long* __restrict__ out)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < G; i += stride) out[i] = recs[(size_t)slots[i] * W + 1] ^ 0x8000000000000000ULL;   // signed order -> unsigned order
}

// gather the slot records into group-id order (the SoA layout build_output reads)
__global__ void gf_gather_kernel(AggPlan plan, const int* __restrict__ ordered_slots, int64_t G, const unsigned long long* __restrict__ recs, int64_t cap, int W,
                                 AggState st)
{
    int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; g < G; g += stride) {
        int64_t s = ordered_slots[g];
        const unsigned long long* r = recs + (size_t)s * W;
        unsigned long long w[MAX_ACCS];
        for (int a = 0; a < plan.num_accs; a++) w[a] = r[2 + a];
        gf_decode(plan, w);
        for (int a = 0; a < plan.num_accs; a++) st.acc[(size_t)a * st.cap + g] = w[a];
        if (plan.num_keys == 1) {
            bool isnull = s == cap;
            unsigned long long k = s == cap + 1 ? EMPTY_KEY : (s < cap ? r[0] : 0ULL);
            st.keyvals[g] = (long long)k;
            st.keynull[g] = isnull ? 1 : 0;
        }
        else {
            unsigned long long pk = r[0];
            int shift = 0;
            for (int k = 0; k < plan.num_keys; k++) {
                int bits = plan.key_bits[k];
                unsigned long long field = (pk >> shift) & ((2ULL << bits) - 1);
                bool isnull = field & 1ULL;
                long long v = (long long)(field >> 1);
                if (bits < 64 && (v >> (bits - 1)) & 1) v |= ~((1LL << bits) - 1);   // sign-extend
                st.keyvals[(size_t)k * st.cap + g] = isnull ? 0 : v;
                st.keynull[(size_t)k * st.cap + g] = isnull ? 1 : 0;
                shift += bits + 1;
            }
        }
    }
}

// =====================================================================================================
// output
// =====================================================================================================
struct OutSpec {
    int32_t count;                   // output columns after the keys
    int32_t kind[48];                // 0 int64 from acc a0; 1 f64 sum nullable by count a1; 2 avg = sum a0 / count a1; 3 i128 sum (a0 lo, a0+1 hi) nullable by a1;
                                     // 4 min/max f64 decode nullable by a1; 5 min/max i64 decode nullable by a1; 6 f64 sum never null (avg partial sum)
                                     // 7 decimal sum -> INT128 (two words per row: high, low), 8 its overflow count (INT64): a0 = 128-bit sum of the
                                     //   high words (or of the short-decimal values when a2 < 0), a2 / a3 = sums of the low word's upper / lower
                                     //   32 bits, a4 = sum of the incoming overflow counts (state input) or -1; a1 = non-NULL rows;
                                     //   9 = 7 for a FINAL / SINGLE step: raises "Decimal overflow" instead of carrying the count on
                                     // 10 / 11 decimal average -> INT128 / INT64: the same total divided by the row count a5 (a plain counter when
                                     //   a5 < 0: a1), rounded HALF_UP (DecimalAverageAggregation.average); NULL when the count is 0
    int32_t a0[48], a1[48], a2[48], a3[48], a4[48], a5[48];
    void* data[48];
    unsigned char* nullmap[48];      // 1 = NULL
};

// REAL group-by keys run as their exact DOUBLE widening (IDENTICAL over floats and over their doubles agree: NaN with NaN, -0.0 with +0.0,
// S/type/RealType.java:172-185) and are narrowed back on output.  NaN payloads move by bit shifts, so the first-seen raw bits survive.
__global__ void agg_widen_real_kernel(const unsigned int* __restrict__ in, int64_t n, unsigned long long* __restrict__ out)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        const unsigned int b = in[i];
        if ((b & 0x7FFFFFFFu) > 0x7F800000u) out[i] = ((unsigned long long)(b >> 31) << 63) | 0x7FF0000000000000ULL | ((unsigned long long)(b & 0x7FFFFFu) << 29);
        else out[i] = (unsigned long long)__double_as_longlong((double)__uint_as_float(b));
    }
}

__global__ void agg_narrow_real_kernel(const unsigned long long* __restrict__ in, int64_t n, unsigned int* __restrict__ out)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        const unsigned long long b = in[i];
        if ((b & 0x7FFFFFFFFFFFFFFFULL) > 0x7FF0000000000000ULL) out[i] = ((unsigned int)(b >> 63) << 31) | 0x7F800000u | (unsigned int)((b >> 29) & 0x7FFFFFu);
        else out[i] = __float_as_uint((float)__longlong_as_double((long long)b));
    }
}

// ---- long DECIMAL (Int128ArrayBlock) support: the group-by proper only ever sees 64-bit channels ----------------------------------
// An INT128 input column is split into four BIGINT columns once per page: high word, low word (as bits), and the low word's upper and
// lower 32 bits as non-negative numbers.  Keys use (high, low); DecimalSumAggregation sums high (signed) and the two low halves with the
// existing carry-free 128-bit accumulators, and the output kernel reassembles sum = S_high * 2^64 + S_upper * 2^32 + S_lower.
__global__ void agg_split_int128_kernel(const long long* __restrict__ src, int64_t n, long long* __restrict__ high, long long* __restrict__ low,
                                        long long* __restrict__ low_upper, long long* __restrict__ low_lower)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        const longlong2 v = ((const longlong2*)src)[i];          // x = high, y = low (S/block/Int128ArrayBlock.java:123-133)
        high[i] = v.x;
        low[i] = v.y;
        low_upper[i] = (long long)((unsigned long long)v.y >> 32);
        low_lower[i] = (long long)((unsigned long long)v.y & 0xFFFFFFFFULL);
    }
}

__global__ void agg_join_int128_kernel(const long long* __restrict__ high, const long long* __restrict__ low, int64_t n, long long* __restrict__ out)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) ((longlong2*)out)[i] = make_longlong2(high[i], low[i]);
}

// 256-bit two's complement accumulator for the reassembly (four 64-bit limbs, least significant first)
struct Wide256 { unsigned long long w[4]; };
__device__ __forceinline__ void wide_add_shifted(Wide256& t, unsigned long long lo, long long hi, int shift_words32)
{
    // the signed 128-bit value (hi:lo), sign-extended to 256 bits, shifted left by 32 * shift_words32 bits (0, 1, 2 or 4)
    unsigned long long v[4] = {lo, (unsigned long long)hi, (unsigned long long)(hi >> 63), (unsigned long long)(hi >> 63)};
    unsigned long long s[4];
    const int words = shift_words32 >> 1;                 // whole 64-bit limbs
    const bool half = (shift_words32 & 1) != 0;           // plus 32 bits
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const int src = i - words;
        unsigned long long cur = src >= 0 ? v[src] : 0, prev = src - 1 >= 0 ? v[src - 1] : 0;
        s[i] = half ? (cur << 32) | (prev >> 32) : cur;
    }
    unsigned long long carry = 0;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        unsigned long long a = t.w[i], b = s[i];
        unsigned long long r = a + b;
        unsigned long long c1 = r < a ? 1 : 0;
        unsigned long long r2 = r + carry;
        unsigned long long c2 = r2 < r ? 1 : 0;
        t.w[i] = r2;
        carry = c1 + c2;
    }
}

__global__ void agg_output_kernel(AggState st, int64_t count, OutSpec spec, unsigned int* __restrict__ err_out, unsigned int* __restrict__ any_null)
{
    int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    unsigned int nulls0 = 0, nulls1 = 0, err = 0;
    for (; g < count; g += stride) {
        for (int c = 0; c < spec.count; c++) {
            unsigned long long x = st.acc[(size_t)spec.a0[c] * st.cap + g];
            unsigned long long cnt = spec.a1[c] >= 0 ? st.acc[(size_t)spec.a1[c] * st.cap + g] : 1;
            long long outv = 0;
            bool isn = false;
            switch (spec.kind[c]) {
                case 0: outv = (long long)x; break;
                case 1: isn = cnt == 0; outv = (long long)x; break;
                case 2:
                    isn = cnt == 0;
                    if (!isn) outv = __double_as_longlong(__ddiv_rn(__longlong_as_double((long long)x), (double)(long long)cnt));
                    break;
                case 3: {
                    isn = cnt == 0;
                    long long hi = (long long)st.acc[(size_t)(spec.a0[c] + 1) * st.cap + g];
                    long long lo = (long long)x;
                    if (hi != (lo >> 63)) err |= TG_ERR_BIT_OVERFLOW;   // Math.addExact would have thrown
                    outv = lo;
                    break;
                }
                case 4: isn = cnt == 0; outv = f64_from_order_key(x); break;
                case 5: isn = cnt == 0; outv = (long long)(x ^ 0x8000000000000000ULL); break;
                case 7: case 8: case 9: case 10: case 11: {
                    // DecimalSumAggregation: state = (sum mod 2^128 as a signed 128-bit value, overflow) with
                    // total = signed128(sum) + overflow * 2^128 (addWithOverflow, S/type/Int128Math.java)
                    isn = cnt == 0;
                    Wide256 t = {{0, 0, 0, 0}};
                    auto pair = [&](int a, unsigned long long* lo, long long* hi) {
                        *lo = st.acc[(size_t)a * st.cap + g];
                        *hi = (long long)st.acc[(size_t)(a + 1) * st.cap + g];
                    };
                    unsigned long long lo; long long hi;
                    pair(spec.a0[c], &lo, &hi);
                    wide_add_shifted(t, lo, hi, spec.a2[c] >= 0 ? 2 : 0);          // short decimals: the values themselves
                    if (spec.a2[c] >= 0) { pair(spec.a2[c], &lo, &hi); wide_add_shifted(t, lo, hi, 1); }
                    if (spec.a3[c] >= 0) { pair(spec.a3[c], &lo, &hi); wide_add_shifted(t, lo, hi, 0); }
                    if (spec.a4[c] >= 0) { pair(spec.a4[c], &lo, &hi); wide_add_shifted(t, lo, hi, 4); }
                    // upper 128 bits + 1 if the low 128 bits read as a negative number
                    long long overflow = (long long)t.w[2] + (((long long)t.w[1]) < 0 ? 1 : 0);
                    const bool upper_fits = (long long)t.w[3] == ((long long)t.w[2] >> 63);
                    if (!upper_fits) err |= TG_ERR_BIT_OVERFLOW;                    // (|total| >= 2^191: nothing sane gets here)
                    if (spec.kind[c] == 8) { outv = overflow; isn = false; break; }
                    if (spec.kind[c] >= 10) {
                        // average = total / count, HALF_UP (Int128Math.divideRoundUp; with overflow != 0 the BigDecimal path of
                        // DecimalAverageAggregation.average :152-175 - the same exact quotient)
                        const unsigned long long n_rows = spec.a5[c] >= 0 ? st.acc[(size_t)spec.a5[c] * st.cap + g] : cnt;
                        isn = n_rows == 0;
                        long long rh = 0;
                        unsigned long long rl = 0;
                        if (!isn) {
                            const bool neg = ((long long)t.w[3]) < 0;
                            unsigned long long m[4] = {t.w[0], t.w[1], t.w[2], t.w[3]};
                            if (neg) {                                               // magnitude
                                unsigned long long carry = 1;
#pragma unroll
                                for (int i = 0; i < 4; i++) { unsigned long long v = ~m[i] + carry; carry = (carry && v == 0) ? 1 : 0; m[i] = v; }
                            }
                            unsigned long long q[4], rem = 0;
#pragma unroll
                            for (int i = 3; i >= 0; i--) {
                                unsigned __int128 cur = ((unsigned __int128)rem << 64) | m[i];
                                q[i] = (unsigned long long)(cur / n_rows);
                                rem = (unsigned long long)(cur % n_rows);
                            }
                            if ((unsigned __int128)rem * 2 >= (unsigned __int128)n_rows) {           // HALF_UP on the magnitude
#pragma unroll
                                for (int i = 0; i < 4; i++) { q[i] += 1; if (q[i] != 0) break; }
                            }
                            // the quotient must fit the result: overflow == 0 -> inside +-10^38 (overflows(result)), else 128 bits (Int128.valueOf)
                            const unsigned long long MAXH = 0x4B3B4CA85A86C47AULL, MAXL = 0x098A224000000000ULL;
                            bool bad = q[2] != 0 || q[3] != 0;
                            if (overflow == 0) bad = bad || q[1] > MAXH || (q[1] == MAXH && q[0] >= MAXL);
                            else bad = bad || (q[1] >> 63) != 0;
                            if (spec.kind[c] == 11) bad = bad || q[1] != 0 || (q[0] >> 63) != 0;             // toLongExact
                            if (bad) err |= TG_ERR_BIT_OVERFLOW;
                            rl = q[0];
                            rh = (long long)q[1];
                            if (neg) { rl = ~rl + 1; rh = (long long)(~(unsigned long long)rh + (rl == 0 ? 1 : 0)); }
                        }
                        if (spec.kind[c] == 11) { outv = (long long)rl; break; }
                        ((long long*)spec.data[c])[2 * g] = isn ? 0 : rh;
                        ((long long*)spec.data[c])[2 * g + 1] = isn ? 0 : (long long)rl;
                        spec.nullmap[c][g] = isn ? 1 : 0;
                        if (isn) { if (c < 32) nulls0 |= 1u << c; else nulls1 |= 1u << (c - 32); }
                        continue;
                    }
                    if (!isn && spec.kind[c] == 9) {
                        // outputDecimal :127-146: overflow != 0 or |value| >= 10^38 -> NUMERIC_VALUE_OUT_OF_RANGE "Decimal overflow"
                        const long long vh = (long long)t.w[1];
                        const unsigned long long vl = t.w[0];
                        // |v| as unsigned 128 bits
                        unsigned long long al = vl, ah = (unsigned long long)vh;
                        if (vh < 0) { al = ~vl + 1; ah = ~(unsigned long long)vh + (al == 0 ? 1 : 0); }
                        const unsigned long long MAXH = 0x4B3B4CA85A86C47AULL, MAXL = 0x098A224000000000ULL;    // 10^38
                        if (overflow != 0 || ah > MAXH || (ah == MAXH && al >= MAXL)) err |= TG_ERR_BIT_OVERFLOW;
                    }
                    ((long long*)spec.data[c])[2 * g] = isn ? 0 : (long long)t.w[1];
                    ((long long*)spec.data[c])[2 * g + 1] = isn ? 0 : (long long)t.w[0];
                    spec.nullmap[c][g] = isn ? 1 : 0;
                    if (isn) { if (c < 32) nulls0 |= 1u << c; else nulls1 |= 1u << (c - 32); }
                    continue;
                }
                default: outv = (long long)x; break;
            }
            ((long long*)spec.data[c])[g] = isn ? 0 : outv;
            spec.nullmap[c][g] = isn ? 1 : 0;
            if (isn) { if (c < 32) nulls0 |= 1u << c; else nulls1 |= 1u << (c - 32); }
        }
    }
    if (err) atomicOr(err_out, err);
    if (nulls0) atomicOr(any_null, nulls0);
    if (nulls1) atomicOr(any_null + 1, nulls1);
}

// typed key column from the 64-bit first-seen key values
__global__ void agg_key_output_kernel(const long long* __restrict__ keyvals, const unsigned char* __restrict__ keynull, int64_t count, int elem,
                                      void* __restrict__ out, unsigned char* __restrict__ nullmap)
{
    int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; g < count; g += stride) {
        long long v = keyvals[g];
        switch (elem) {
            case 8: ((long long*)out)[g] = v; break;
            case 4: ((int*)out)[g] = (int)v; break;
            case 2: ((short*)out)[g] = (short)v; break;
            default: ((signed char*)out)[g] = (signed char)v; break;
        }
        nullmap[g] = keynull[g];
    }
}

__global__ void nullmap_pack_kernel(const unsigned char* __restrict__ is_null, int64_t n, unsigned char* __restrict__ bitmap, unsigned int* __restrict__ any)
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
        bitmap[b] = (unsigned char)v;
    }
    if (seen && any) atomicOr(any, 1u);
}

// SkipAggregationBuilder.buildOutputPage (M/operator/aggregation/partial/SkipAggregationBuilder.java:103-131): every row is its own
// group, so the intermediate state of an aggregate is a function of that one row - count: 0/1, sum/min/max: the value or NULL,
// avg: (0/1, value).  One thread per row, all aggregates in one pass; null bytes are packed into bitmaps by nullmap_pack_kernel.
#define SKIP_MAX_FNS 24
struct SkipFn {
    int32_t function, in_ch, mask_ch, in_is_double;
    void* out0;
    unsigned char* null0;      // 1 byte per row (sum / min / max), else null
    void* out1;                // avg: the DOUBLE sum; decimal sum / avg: the overflow count
    void* out2;                // decimal avg: the row count
};
struct SkipSpec {
    int32_t count;
    SkipFn f[SKIP_MAX_FNS];
};

__global__ void __launch_bounds__(256) agg_skip_kernel(DColumns cols, int64_t n, SkipSpec spec)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        for (int a = 0; a < spec.count; a++) {
            const SkipFn& f = spec.f[a];
            bool on = true;
            if (f.mask_ch >= 0) {
                const ColRef& m = cols.cols[f.mask_ch];
                on = tg_valid(m.validity, i) && tg_load_i64(m, i) != 0;       // AggregationMask: NULL or false drops the row
            }
            long long bits = 0, bits_high = 0;
            if (f.in_ch >= 0) {
                const ColRef& c = cols.cols[f.in_ch];
                if (!tg_valid(c.validity, i)) on = false;
                else if (c.elem == 16) { bits_high = ((const long long*)c.data)[2 * i]; bits = ((const long long*)c.data)[2 * i + 1]; }
                else { bits = tg_load_i64(c, i); bits_high = bits >> 63; }
            }
            switch (f.function) {
                case TGPU_AGG_SUM_DECIMAL: case TGPU_AGG_AVG_DECIMAL:
                    ((long long*)f.out0)[2 * i] = on ? bits_high : 0;
                    ((long long*)f.out0)[2 * i + 1] = on ? bits : 0;
                    f.null0[i] = on ? 0 : 1;
                    ((long long*)f.out1)[i] = 0;
                    if (f.function == TGPU_AGG_AVG_DECIMAL) ((long long*)f.out2)[i] = on ? 1 : 0;
                    break;
                case TGPU_AGG_COUNT_STAR: case TGPU_AGG_COUNT:
                    ((long long*)f.out0)[i] = on ? 1 : 0;
                    break;
                case TGPU_AGG_AVG: {
                    ((long long*)f.out0)[i] = on ? 1 : 0;
                    double v = f.in_is_double ? __longlong_as_double(bits) : (double)bits;
                    ((double*)f.out1)[i] = on ? v : 0.0;
                    break;
                }
                default:                                                       // sum / min / max: the value itself (raw bits for DOUBLE)
                    ((long long*)f.out0)[i] = on ? bits : 0;
                    f.null0[i] = on ? 0 : 1;
                    break;
            }
        }
    }
}

#endif  // __CUDACC__


// =====================================================================================================
// NVRTC specialisation of path S: straight-line typed code for the row program (filter + projections +
// key packing + accumulator updates) plugged into agg_small_body<P> of device_lib.cuh.
// =====================================================================================================
static void appendf(std::string& s, const char* fmt, ...)
{
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    s += buf;
}

static std::string gen_operand(const DOperand& o)
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

// `elems[c]` = element size of input channel c (0 = not a fixed-width column); bit c of nullable_mask = channel c has a validity bitmap
// rows in flight per thread of the fused general kernel (TGPU_AGG_G_ROWS: 1, 2, 4 or 8; experiments)
static int general_rows_per_thread()
{
    const char* e = getenv("TGPU_AGG_G_ROWS");
    const int r = e ? atoi(e) : TGD_G_ROWS;
    return r == 1 || r == 2 || r == 4 || r == 8 ? r : TGD_G_ROWS;
}

static std::string gen_agg_small_source(const AggPlan& plan, const DProgram* prog, const int* elems, int num_channels, int L, int min_blocks,
                                        uint32_t nullable_mask, AccMap* map, bool vec = false)
{
    std::string s;
    bool used[TGPU_MAX_CHANNELS] = {false};
    for (int i = 0; i < plan.num_srcs; i++)
        if (!plan.srcs[i].is_temp) used[plan.srcs[i].index] = true;
    // never-NULL analysis of the temporaries (straight-line program: one pass)
    bool temp_nullable[TGPU_MAX_TEMPS];
    for (int t = 0; t < TGPU_MAX_TEMPS; t++) temp_nullable[t] = true;
    auto opnd_nullable = [&](const DOperand& o) {
        switch (o.kind) {
            case TGPU_OPND_COLUMN: return ((nullable_mask >> o.index) & 1) != 0;
            case TGPU_OPND_TEMP: return temp_nullable[o.index];
            case TGPU_OPND_CONST: return false;
            default: return true;
        }
    };
    if (prog) {
        for (int i = 0; i < prog->num_insns; i++) {
            const DInsn& in = prog->insns[i];
            const DOperand* ops[3] = {&in.a, &in.b, &in.c};
            for (auto* o : ops)
                if (o->kind == TGPU_OPND_COLUMN) used[o->index] = true;
            bool n;
            switch (in.op) {
                case TGPU_EX_IS_NULL: case TGPU_EX_IS_NOT_NULL: n = false; break;
                case TGPU_EX_MOV: case TGPU_EX_NEG: case TGPU_EX_NOT: case TGPU_EX_CAST_BIGINT_TO_DOUBLE: case TGPU_EX_CAST_DOUBLE_TO_BIGINT: case TGPU_EX_IN:
                    n = opnd_nullable(in.a); break;
                case TGPU_EX_BETWEEN: n = opnd_nullable(in.a) || opnd_nullable(in.b) || opnd_nullable(in.c); break;
                default: n = opnd_nullable(in.a) || opnd_nullable(in.b); break;
            }
            temp_nullable[in.dst] = n;
        }
    }
    auto src_nullable = [&](int src) {
        const SrcRef& r = plan.srcs[src];
        return r.is_temp ? temp_nullable[r.index] : (((nullable_mask >> r.index) & 1) != 0);
    };
    // compact accumulator space
    int compact = 0;
    int kinds[MAX_ACCS];
    for (int a = 0; a < plan.num_accs; a++) map->of_plan[a] = -1;
    for (int a = 0; a < plan.num_accs; a++) {
        const AccDesc& d = plan.accs[a];
        if (d.kind == ACC_NONNULL && !src_nullable(d.src)) continue;   // aliased below
        kinds[compact] = d.kind;
        map->of_plan[a] = compact++;
    }
    for (int a = 0; a < plan.num_accs; a++) {
        if (map->of_plan[a] >= 0) continue;
        const AccDesc& d = plan.accs[a];
        for (int r = 0; r < plan.num_accs; r++)
            if (plan.accs[r].kind == ACC_ROWS && plan.accs[r].mask == d.mask) map->of_plan[a] = map->of_plan[r];
    }
    map->compact_count = compact;

    appendf(s, "struct Prog {\n  static constexpr int L = %d, A = %d, R = 4, GR = %d;\n  static constexpr bool VEC = %s, SPECIALS = %s;\n", L, compact, general_rows_per_thread(),
            vec ? "true" : "false", plan.num_keys == 1 ? "true" : "false");
    s += "  __device__ static __forceinline__ int acc_kind(int a) {\n    switch (a) {\n";
    for (int a = 0; a < compact; a++) appendf(s, "      case %d: return %d;\n", a, kinds[a]);
    s += "      default: return 0;\n    }\n  }\n";
    s += "  struct Regs {\n";
    for (int c = 0; c < num_channels && c < TGPU_MAX_CHANNELS; c++)
        if (used[c]) appendf(s, "    long long c%d; bool c%dn;\n", c, c);
    s += "  };\n";
    for (int i = 0; i < plan.num_srcs; i++) appendf(s, "  long long v%d; bool vn%d;\n", i, i);
    // all global loads of a row, nothing else: the body issues them for R rows back to back
    s += "  __device__ __forceinline__ void load(const DColumns& cols, long long row, Regs& r) {\n";
    for (int c = 0; c < num_channels && c < TGPU_MAX_CHANNELS; c++) {
        if (!used[c]) continue;
        appendf(s, "    r.c%d = tg_load_elem<%d>(cols.cols[%d].data, row);", c, elems[c], c);
        if ((nullable_mask >> c) & 1) appendf(s, " r.c%dn = !tg_valid(cols.cols[%d].validity, row);\n", c, c);
        else appendf(s, " r.c%dn = false;\n", c);
    }
    s += "  }\n";
    // the same for FOUR CONSECUTIVE rows starting at a multiple of 4 (VEC kernels: every column base is 16-byte aligned): one or two
    // 16-byte loads per wide column, one 4-byte load per INT8 column, the four validity bits from one byte
    s += "  __device__ __forceinline__ void load4(const DColumns& cols, long long row0, Regs (&r)[4]) {\n";
    for (int c = 0; c < num_channels && c < TGPU_MAX_CHANNELS; c++) {
        if (!used[c]) continue;
        switch (elems[c]) {
            case 8:
                appendf(s, "    { const longlong2* p = (const longlong2*)((const char*)cols.cols[%d].data + row0 * 8); longlong2 a = p[0], b = p[1];"
                           " r[0].c%d = a.x; r[1].c%d = a.y; r[2].c%d = b.x; r[3].c%d = b.y; }\n", c, c, c, c, c);
                break;
            case 4:
                appendf(s, "    { int4 a = *(const int4*)((const char*)cols.cols[%d].data + row0 * 4); r[0].c%d = a.x; r[1].c%d = a.y; r[2].c%d = a.z; r[3].c%d = a.w; }\n",
                        c, c, c, c, c);
                break;
            case 2:
                appendf(s, "    { short4 a = *(const short4*)((const char*)cols.cols[%d].data + row0 * 2); r[0].c%d = a.x; r[1].c%d = a.y; r[2].c%d = a.z; r[3].c%d = a.w; }\n",
                        c, c, c, c, c);
                break;
            default:
                appendf(s, "    { char4 a = *(const char4*)((const char*)cols.cols[%d].data + row0); r[0].c%d = a.x; r[1].c%d = a.y; r[2].c%d = a.z; r[3].c%d = a.w; }\n",
                        c, c, c, c, c);
                break;
        }
        if ((nullable_mask >> c) & 1)
            appendf(s, "    { const uint8_t* v = cols.cols[%d].validity; unsigned int b = v ? ((unsigned int)v[row0 >> 3] >> (row0 & 7)) : 0xfu;"
                       " r[0].c%dn = !(b & 1); r[1].c%dn = !(b & 2); r[2].c%dn = !(b & 4); r[3].c%dn = !(b & 8); }\n", c, c, c, c, c);
        else appendf(s, "    r[0].c%dn = r[1].c%dn = r[2].c%dn = r[3].c%dn = false;\n", c, c, c, c);
    }
    s += "  }\n";
    s += "  __device__ __forceinline__ bool row(const Regs& r, unsigned long long* pk, int* special, unsigned int* err) {\n";
    for (int c = 0; c < num_channels && c < TGPU_MAX_CHANNELS; c++)
        if (used[c]) appendf(s, "    const long long c%d = r.c%d; const bool c%dn = r.c%dn;\n", c, c, c, c);
    if (prog) {
        for (int t = 0; t < TGPU_MAX_TEMPS; t++) appendf(s, "    long long t%d = 0; bool tn%d = true;\n", t, t);
        for (int i = 0; i < prog->num_insns; i++) {
            const DInsn& in = prog->insns[i];
            if (i == prog->num_filter_insns && prog->filter_temp >= 0)
                appendf(s, "    if (tn%d || t%d == 0) return false;\n", prog->filter_temp, prog->filter_temp);
            if (in.op == TGPU_EX_IN) {
                int li = (int)in.b.imm;
                appendf(s, "    { Value a = %s; bool hit = false;\n", gen_operand(in.a).c_str());
                for (int k = 0; k < prog->in_count[li]; k++) {
                    unsigned long long c = (unsigned long long)prog->in_values[prog->in_offset[li] + k];
                    if (in.vtype == TGPU_V_DOUBLE) appendf(s, "      hit |= __longlong_as_double(a.bits) == __longlong_as_double((long long)0x%llxULL);\n", c);
                    else appendf(s, "      hit |= a.bits == (long long)0x%llxULL;\n", c);
                }
                appendf(s, "      t%d = hit ? 1 : 0; tn%d = a.is_null; }\n", in.dst, in.dst);
            }
            else {
                appendf(s, "    { Value x = vm_apply(%d, %d, %s, %s, %s, err); t%d = x.bits; tn%d = x.is_null; }\n", in.op, in.vtype,
                        gen_operand(in.a).c_str(), gen_operand(in.b).c_str(), gen_operand(in.c).c_str(), in.dst, in.dst);
            }
        }
        if (prog->num_filter_insns == prog->num_insns && prog->filter_temp >= 0)
            appendf(s, "    if (tn%d || t%d == 0) return false;\n", prog->filter_temp, prog->filter_temp);
    }
    for (int i = 0; i < plan.num_srcs; i++) {
        if (plan.srcs[i].is_temp) appendf(s, "    v%d = t%d; vn%d = tn%d;\n", i, plan.srcs[i].index, i, plan.srcs[i].index);
        else appendf(s, "    v%d = c%d; vn%d = c%dn;\n", i, plan.srcs[i].index, i, plan.srcs[i].index);
    }
    if (plan.num_keys == 1) {
        int k = plan.key_src[0];
        appendf(s, "    if (vn%d) { *special = 0; return true; }\n    unsigned long long u = (unsigned long long)v%d;\n", k, k);
        if (plan.key_is_double[0])
            s += "    if ((u << 1) == 0) u = 0;\n    if ((u & 0x7FFFFFFFFFFFFFFFULL) > 0x7FF0000000000000ULL) u = 0x7FF8000000000000ULL;\n";
        s += "    if (u == TGD_EMPTY_KEY) { *special = 1; return true; }\n    *pk = u;\n";
    }
    else {
        s += "    unsigned long long k = 0;\n";
        int shift = 0;
        for (int kk = 0; kk < plan.num_keys; kk++) {
            int src = plan.key_src[kk], bits = plan.key_bits[kk];
            appendf(s, "    k |= (vn%d ? 1ULL : ((((unsigned long long)v%d) & 0x%llxULL) << 1)) << %d;\n", src, src, (1ULL << bits) - 1, shift);
            shift += bits + 1;
        }
        s += "    *pk = k;\n";
    }
    s += "    return true;\n  }\n";
    s += "  __device__ __forceinline__ void accumulate(unsigned long long* acc, int T) {\n";
    for (int a = 0; a < plan.num_accs; a++) {
        const AccDesc& d = plan.accs[a];
        if (d.kind == ACC_SUM_I64_HI) continue;
        if (d.kind == ACC_NONNULL && !src_nullable(d.src)) continue;
        std::string cond = "true";
        if (d.mask >= 0) { char b[64]; snprintf(b, sizeof(b), "(!vn%d && v%d != 0)", d.mask, d.mask); cond = b; }
        if (d.kind != ACC_ROWS && src_nullable(d.src)) { char b[64]; snprintf(b, sizeof(b), " && !vn%d", d.src); cond += b; }
        if (d.kind == ACC_ROWS) appendf(s, "    if (%s) acc_update_private(%d, acc + %d * T, T, 0);\n", cond.c_str(), d.kind, map->of_plan[a]);
        else appendf(s, "    if (%s) acc_update_private(%d, acc + %d * T, T, v%d);\n", cond.c_str(), d.kind, map->of_plan[a], d.src);
    }
    s += "  }\n";
    // the same accumulators as reductions on a fused-G slot record (plan order, the record encoding of gf_accumulate: NONNULL counts the
    // NULL inputs, the 128-bit integer sum is two carry-free 64-bit sums of the value's halves)
    s += "  __device__ __forceinline__ void accumulate_global(unsigned long long* acc) {\n";
    for (int a = 0; a < plan.num_accs; a++) {
        const AccDesc& d = plan.accs[a];
        if (d.kind == ACC_SUM_I64_HI) continue;
        std::string cond = "true";
        if (d.mask >= 0) { char b[64]; snprintf(b, sizeof(b), "(!vn%d && v%d != 0)", d.mask, d.mask); cond = b; }
        const bool nullable = d.src >= 0 && src_nullable(d.src);
        if (d.kind == ACC_NONNULL) {
            if (nullable) appendf(s, "    if (%s && vn%d) atomicAdd(acc + %d, 1ULL);\n", cond.c_str(), d.src, a);
            continue;
        }
        if (d.kind != ACC_ROWS && nullable) { char b[64]; snprintf(b, sizeof(b), " && !vn%d", d.src); cond += b; }
        switch (d.kind) {
            case ACC_ROWS: appendf(s, "    if (%s) atomicAdd(acc + %d, 1ULL);\n", cond.c_str(), a); break;
            case ACC_SUM_F64: appendf(s, "    if (%s) atomicAdd((double*)(acc + %d), __longlong_as_double(v%d));\n", cond.c_str(), a, d.src); break;
            case ACC_SUM_F64_FROM_I64: appendf(s, "    if (%s) atomicAdd((double*)(acc + %d), (double)v%d);\n", cond.c_str(), a, d.src); break;
            case ACC_SUM_I64_LO:
                // (values that fit 32 unsigned bits have nothing to add to the high word: one reduction less per row)
                appendf(s, "    if (%s) { atomicAdd(acc + %d, (unsigned long long)v%d & 0xFFFFFFFFULL); if ((v%d >> 32) != 0) atomicAdd(acc + %d, (unsigned long long)(v%d >> 32)); }\n",
                        cond.c_str(), a, d.src, d.src, a + 1, d.src);
                break;
            case ACC_MIN_F64: appendf(s, "    if (%s) atomicMin(acc + %d, f64_order_key(v%d));\n", cond.c_str(), a, d.src); break;
            case ACC_MAX_F64: appendf(s, "    if (%s) atomicMax(acc + %d, f64_order_key_max(v%d));\n", cond.c_str(), a, d.src); break;
            case ACC_MIN_I64: appendf(s, "    if (%s) atomicMin(acc + %d, i64_order_key(v%d));\n", cond.c_str(), a, d.src); break;
            case ACC_MAX_I64: appendf(s, "    if (%s) atomicMax(acc + %d, i64_order_key(v%d));\n", cond.c_str(), a, d.src); break;
            default: break;
        }
    }
    s += "  }\n};\n";
    appendf(s, "extern \"C\" __global__ void __launch_bounds__(%d, %d) tg_agg_small_jit(DColumns cols, long long n, SmallOut out) {\n", S_THREADS, min_blocks);
    s += "  extern __shared__ unsigned long long smem_u64[];\n  Prog p;\n  agg_small_body(p, cols, n, out, smem_u64);\n}\n";
    {
        const char* e = getenv("TGPU_AGG_G_MINB");
        appendf(s, "extern \"C\" __global__ void __launch_bounds__(256, %d) tg_agg_general_jit(DColumns cols, long long n, const int* rows, long long first, const int* stamp_rows,\n",
                e ? atoi(e) : 4);
    }
    s += ""
         "    long long page_base, unsigned long long* recs, long long cap, int W, int* tickets, int budget_per_way, int* deferred, unsigned int* err_out) {\n"
         "  Prog p;\n  agg_general_body(p, cols, n, rows, first, stamp_rows, page_base, recs, cap, W, tickets, budget_per_way, deferred, err_out);\n}\n";
    return s;
}

// =====================================================================================================
// host side
// =====================================================================================================
struct AggFnPlan {
    int function;
    int in_elem_is_double;
    int acc_main = -1, acc_count = -1;   // indices into plan.accs
    int acc2 = -1, acc3 = -1, acc4 = -1; // decimal sum: the low word's upper / lower 32-bit sums, the incoming overflow counts
    int acc5 = -1;                       // decimal average from states: the sum of the incoming row counts
    int result_type = 0;                 // decimal average: TGPU_INT64 (short decimal) or TGPU_INT128
};

struct AggOp : tgpu_op {
    // spec
    std::vector<int32_t> key_channels;       // channels of the (projected) input
    std::vector<tgpu_agg_fn> fns;
    int step = TGPU_STEP_SINGLE;
    int64_t expected_groups = 0, max_partial_bytes = 0;
    bool has_pre = false;
    DProgram host_prog;
    DevBuf d_prog;
    std::vector<tgpu_projection> projections;
    std::vector<tgpu_expr_insn> pre_insns;            // deep copy of the caller's program (its pointers die after create)
    std::vector<std::vector<int64_t>> pre_in_values;
    int32_t pre_filter_temp = -1, pre_num_filter_insns = 0;
    tgpu_op* inner_fp = nullptr;                      // unfused FilterAndProject feeding the general path
    int32_t prog_max_channel = -1;
    bool gids_only = false;                  // tgpu_groupby_hash_* handle
    // variable-width keys: one string dictionary per UTF8 key column; the group-by runs on the 30-bit ids (strdict.cuh)
    std::vector<std::shared_ptr<StringDict>> key_dicts;
    std::vector<uint8_t> key_real;       // REAL keys: the group-by runs on their DOUBLE widening (encode_string_keys), the output narrows them back
    // global aggregation default rows (HashAggregationOperator.getGlobalAggregationOutput :537-567)
    std::vector<int32_t> global_group_ids;
    int32_t group_id_key = -1;               // index into key_channels of the $group_id key
    std::vector<int32_t> input_types;        // tgpu_type of every aggregation-input channel (only needed to shape the default rows)
    bool saw_group = false;                  // a group was ever created (across PARTIAL flushes)

    // resolved at the first page (needs column types)
    bool planned = false;
    AggPlan plan;
    std::vector<int> key_types;
    std::vector<int> src_channel;            // aggregation-input channel of every plan source
    std::vector<AggFnPlan> fnplans;
    std::vector<int> fn_input_types;         // tgpu_type of each aggregate's input (first state column for FINAL)

    // state
    bool use_general = false;
    DevBuf st_count, st_keys, st_acc, st_keyvals, st_keynull;
    int64_t st_cap = 0;
    int64_t group_count = 0;
    // path S scratch
    struct JitVariant { void* fn = nullptr; AccMap map; };
    std::map<uint64_t, JitVariant> jit_variants;   // keyed by (L, which channels carry a validity bitmap)
    std::map<uint64_t, void*> jit_g_variants;      // fused general kernel, keyed by the page layout (element widths, validity bitmaps)
    std::vector<int> jit_elems;
    DevBuf f_tickets;
    int s_L = 0, s_grid = 0;
    size_t s_smem = 0, s_per_slot = 0, s_fixed = 0;
    DevBuf blk_keys, blk_first, blk_acc, blk_ps;
    // path G
    DevBuf g_table, g_special;
    int64_t g_slots = 0;
    // path G, fused form
    bool fused_general = false;
    DevBuf f_recs;
    int64_t f_cap = 0, f_used = 0, f_specials = 0, rows_seen = 0;

    bool finishing = false, finished = false, flushing = false;
    std::vector<OwnedPage*> pending;
    size_t next_out = 0;

    // long DECIMAL channels (TGPU_INT128): split into four BIGINT channels appended behind the page's own (prepare_wide)
    std::vector<int32_t> spec_key_channels;     // groupByChannels as the caller numbered them (key_channels is rewritten by prepare_wide)
    bool wide_ready = false;
    int wide_base = -1;                         // first virtual channel = number of real channels of the page
    std::vector<int> wide_channels;             // the INT128 channels the plan reads, ascending
    std::vector<char> wide_key_high;            // per (expanded) group-by key: 1 = the high word of an INT128 key, the next key is its low word

    // adaptive partial aggregation: one "builder" spans the pages between two flushes (HashAggregationOperator.aggregationBuilder)
    tgpu_partial_agg_controller* controller = nullptr;
    bool builder_open = false, skip_mode = false;
    int64_t builder_bytes = 0, builder_rows = 0, builder_unique = 0;     // aggregationInputBytesProcessed / ...RowsProcessed / ...UniqueRowsProduced
    int64_t rows_skipped = 0;                                              // AggregationMetrics: input rows processed with partial aggregation disabled
    tgpu_op* skip_fp = nullptr;                                            // the pre-stage as its own FilterAndProject, for skipped builders of a fused operator

    explicit AggOp(tgpu_ctx* c) : tgpu_op(c) {}
    ~AggOp() override
    {
        for (size_t i = next_out; i < pending.size(); i++) delete pending[i];
        delete inner_fp;
        delete skip_fp;
    }

    AggState state() const
    {
        AggState s;
        s.count = st_count.as<int32_t>();
        s.keys = st_keys.as<unsigned long long>();
        s.acc = st_acc.as<unsigned long long>();
        s.keyvals = st_keyvals.as<long long>();
        s.keynull = st_keynull.as<unsigned char>();
        s.cap = st_cap;
        return s;
    }

    // sources are identified by the channel of the aggregation input they stand for (a projection output when a
    // pre-stage is fused), so the accumulator layout is the same with and without the fused pre-stage
    int add_src(int is_temp, int index, int vtype, int agg_channel)
    {
        for (int i = 0; i < plan.num_srcs; i++)
            if (src_channel[i] == agg_channel) return i;
        if (plan.num_srcs >= MAX_SRCS) return -1;
        plan.srcs[plan.num_srcs] = SrcRef{is_temp, index, vtype, 0};
        src_channel.push_back(agg_channel);
        return plan.num_srcs++;
    }

    // value source of a channel of the aggregation input (a projection output when `pre` is set)
    int src_of_channel(int ch, int* type_out, const DevPage& in)
    {
        if (!has_pre) {
            if (ch < 0 || ch >= (int)in.cols.size()) return -1;
            *type_out = in.cols[ch].type;
            return add_src(0, ch, 0, ch);
        }
        if (ch < 0 || ch >= (int)projections.size()) return -1;
        const tgpu_projection& p = projections[ch];
        if (p.kind == 0) {
            if (p.index < 0 || p.index >= (int)in.cols.size()) return -1;
            *type_out = in.cols[p.index].type;
            return add_src(0, p.index, 0, ch);
        }
        *type_out = p.vtype == TGPU_V_DOUBLE ? TGPU_FLOAT64 : p.vtype == TGPU_V_BOOLEAN ? TGPU_INT8 : TGPU_INT64;
        return add_src(1, p.index, p.vtype, ch);
    }

    int add_acc(int kind, int src, int mask)
    {
        for (int i = 0; i < plan.num_accs; i++)
            if (plan.accs[i].kind == kind && plan.accs[i].src == src && plan.accs[i].mask == mask) return i;
        int need = kind == ACC_SUM_I64_LO ? 2 : 1;
        if (plan.num_accs + need > MAX_ACCS) return -1;
        int at = plan.num_accs;
        plan.accs[at] = AccDesc{kind, src, mask, 0};
        if (need == 2) plan.accs[at + 1] = AccDesc{ACC_SUM_I64_HI, src, mask, 0};
        plan.num_accs += need;
        return at;
    }

    // channel of an ingested page that feeds group-by key k (a pass-through projection when the pre-stage is fused)
    int key_input_channel(int k) const
    {
        int ch = key_channels[k];
        if (!has_pre) return ch;
        if (ch < 0 || ch >= (int)projections.size() || projections[ch].kind != 0) return -1;
        return projections[ch].index;
    }

    int wide_virtual(int ch, int word) const
    {
        for (size_t i = 0; i < wide_channels.size(); i++)
            if (wide_channels[i] == ch) return wide_base + 4 * (int)i + word;
        return -1;
    }

    // TGPU_INT128 channels -> four BIGINT channels each (high, low, low's upper 32 bits, low's lower 32 bits) appended behind the real
    // channels; on the first page the group-by keys of that type become (high, low) key pairs.  The kernels never see a 128-bit value.
    int prepare_wide(DevPage* pg)
    {
        const bool from_state = step == TGPU_STEP_FINAL || step == TGPU_STEP_INTERMEDIATE;
        if (!wide_ready) {
            std::vector<int> want;
            auto note = [&](int ch) { if (ch >= 0 && ch < (int)pg->cols.size() && pg->cols[ch].type == TGPU_INT128) want.push_back(ch); };
            bool any_wide = false;
            for (auto& c : pg->cols) any_wide = any_wide || c.type == TGPU_INT128;
            if (any_wide && has_pre)
                return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "a fused pre-stage over pages with 128-bit channels is not supported: run the FilterAndProject operator in front");
            for (int ch : key_channels) note(ch);
            for (auto& f : fns) {
                note(f.input_channel);
                if (f.function != TGPU_AGG_SUM_DECIMAL && f.function != TGPU_AGG_AVG_DECIMAL && f.function != TGPU_AGG_COUNT && f.function != TGPU_AGG_COUNT_STAR && f.input_channel >= 0 &&
                    f.input_channel < (int)pg->cols.size() && pg->cols[f.input_channel].type == TGPU_INT128)
                    return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "aggregate function %d over a 128-bit channel (only count and the decimal sum are built)", f.function);
            }
            (void)from_state;
            std::sort(want.begin(), want.end());
            want.erase(std::unique(want.begin(), want.end()), want.end());
            wide_channels = want;
            wide_base = (int)pg->cols.size();
            if (wide_base + 4 * (int)wide_channels.size() > TGPU_MAX_CHANNELS)
                return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "too many channels once the 128-bit ones are split (%d)", wide_base + 4 * (int)wide_channels.size());
            // INT128 keys -> (high, low)
            std::vector<int32_t> keys;
            std::vector<std::shared_ptr<StringDict>> dicts;
            wide_key_high.clear();
            int new_group_id_key = group_id_key;
            for (size_t k = 0; k < key_channels.size(); k++) {
                const int ch = key_channels[k];
                if ((int)k == group_id_key) new_group_id_key = (int)keys.size();
                if (wide_virtual(ch, 0) >= 0) {
                    keys.push_back(wide_virtual(ch, 0)); wide_key_high.push_back(1); dicts.push_back(nullptr);
                    keys.push_back(wide_virtual(ch, 1)); wide_key_high.push_back(0); dicts.push_back(nullptr);
                }
                else {
                    keys.push_back(ch); wide_key_high.push_back(0);
                    dicts.push_back(k < key_dicts.size() ? key_dicts[k] : nullptr);
                }
            }
            key_channels = keys;
            key_dicts = dicts;
            group_id_key = new_group_id_key;
            wide_ready = true;
        }
        if (wide_channels.empty()) return TGPU_OK;
        if ((int)pg->cols.size() != wide_base) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "page has %zu channels, the first one had %d", pg->cols.size(), wide_base);
        const int64_t n = pg->rows;
        for (int ch : wide_channels) {
            const DevColumn src = pg->cols[ch];
            if (src.type != TGPU_INT128) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "channel %d changed its type between pages", ch);
            DevColumn part[4];
            for (auto& c : part) {
                c.type = TGPU_INT64;
                c.length = n;
                c.own_data = std::make_shared<DevBuf>();
                TG_TRY(c.own_data->alloc(ctx, (size_t)std::max<int64_t>(n, 1) * 8));
                c.data = c.own_data->p;
                c.own_validity = src.own_validity;
                c.validity = src.validity;
            }
            if (n > 0)
                TG_LAUNCH(ctx, agg_split_int128_kernel, tg_grid(ctx, n, 1024, 8), 256, 0, (const long long*)src.data, n, part[0].own_data->as<long long>(),
                          part[1].own_data->as<long long>(), part[2].own_data->as<long long>(), part[3].own_data->as<long long>());
            for (auto& c : part) pg->cols.push_back(std::move(c));
        }
        return TGPU_OK;
    }

    // UTF8 key columns of the page -> INT32 dictionary ids, in place (FlatHash keeps the bytes in AppendOnlyVariableWidthData; here
    // the dictionary does, and the group-by proper sees fixed-width keys)
    int encode_string_keys(DevPage* pg)
    {
        const int nk = (int)key_channels.size();
        if ((int)key_dicts.size() < nk) key_dicts.resize(nk);
        if ((int)key_real.size() < nk) key_real.resize(nk, 0);
        bool any_real = false;
        for (auto& c : pg->cols) any_real = any_real || c.type == TGPU_FLOAT32;
        if (any_real) {
            if (has_pre) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "a fused pre-stage over pages with REAL channels is not supported: run the FilterAndProject operator in front");
            for (auto& f : fns)
                if (f.function != TGPU_AGG_COUNT_STAR && f.input_channel >= 0 && f.input_channel < (int)pg->cols.size() && pg->cols[f.input_channel].type == TGPU_FLOAT32)
                    return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "aggregate function %d over a REAL channel: keep the Java accumulator", f.function);
        }
        std::map<int, int> done;      // channel -> first key that encoded it
        for (int k = 0; k < nk; k++) {
            int ch = key_input_channel(k);
            if (ch < 0 || ch >= (int)pg->cols.size()) continue;      // reported by make_plan
            auto first = done.find(ch);
            if (first != done.end()) { key_dicts[k] = key_dicts[first->second]; key_real[k] = key_real[first->second]; continue; }
            if (pg->cols[ch].type == TGPU_FLOAT32) {
                if (planned && !key_real[k]) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "group-by channel %d became REAL after the first page", ch);
                const DevColumn& src = pg->cols[ch];
                DevColumn wide;
                wide.type = TGPU_FLOAT64;
                wide.length = src.length;
                wide.own_data = std::make_shared<DevBuf>();
                TG_TRY(wide.own_data->alloc(ctx, (size_t)std::max<int64_t>(src.length, 1) * 8));
                wide.data = wide.own_data->p;
                wide.own_validity = src.own_validity;
                wide.validity = src.validity;
                if (src.length > 0)
                    TG_LAUNCH(ctx, agg_widen_real_kernel, tg_grid(ctx, src.length, 1024, 8), 256, 0, (const unsigned int*)src.data, src.length, wide.own_data->as<unsigned long long>());
                pg->cols[ch] = std::move(wide);
                key_real[k] = 1;
                done[ch] = k;
                continue;
            }
            if (key_real[k]) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "group-by channel %d was REAL in an earlier page and is type %d now", ch, pg->cols[ch].type);
            const bool is_string = pg->cols[ch].type == TGPU_UTF8;
            if (!is_string && !key_dicts[k]) continue;
            if (!is_string) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "group-by channel %d was variable-width in an earlier page and is type %d now", ch, pg->cols[ch].type);
            if (planned && !key_dicts[k]) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "group-by channel %d became variable-width after the first page", ch);
            if (!key_dicts[k]) key_dicts[k] = std::make_shared<StringDict>(ctx);
            DevColumn ids;
            TG_TRY(key_dicts[k]->encode(pg->cols[ch], &ids));
            pg->cols[ch] = std::move(ids);
            done[ch] = k;
        }
        return TGPU_OK;
    }

    int make_plan(const DevPage& in)
    {
        memset(&plan, 0, sizeof(plan));
        src_channel.clear();
        plan.has_pre = has_pre ? 1 : 0;
        int nk = (int)key_channels.size();
        if (nk < 1) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "global aggregation (no GROUP BY keys) stays on the Java AggregationOperator");
        if (nk > MAX_KEYS) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "more than %d group-by keys", MAX_KEYS);
        plan.num_keys = nk;
        int total_bits = 0;
        key_types.clear();
        for (int k = 0; k < nk; k++) {
            int type = 0;
            int s = src_of_channel(key_channels[k], &type, in);
            if (s < 0) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "group-by channel %d out of range", key_channels[k]);
            if (plan.srcs[s].is_temp) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "group-by keys must be pass-through channels of the fused pre-stage");
            int bits = type == TGPU_INT64 || type == TGPU_FLOAT64 ? 64 : type == TGPU_INT32 ? 32 : type == TGPU_INT16 ? 16 : type == TGPU_INT8 ? 8 : 0;
            if (k < (int)key_dicts.size() && key_dicts[k] && type == TGPU_INT32) bits = 30;     // dictionary ids of a variable-width key (< SD_MAX_IDS)
            if (!bits) return tg_fail(ctx, TGPU_ERR_ILLEGAL_STATE, "variable-width group-by key reached the planner unencoded");
            plan.key_src[k] = s;
            plan.key_bits[k] = bits;
            plan.key_is_double[k] = type == TGPU_FLOAT64;
            key_types.push_back(type);
            total_bits += bits + 1;
        }
        plan.key_hashed = (nk > 1 && total_bits > 63) ? 1 : 0;
        fnplans.clear();
        fn_input_types.clear();
        bool from_state = step == TGPU_STEP_FINAL || step == TGPU_STEP_INTERMEDIATE;
        for (auto& f : fns) {
            AggFnPlan fp;
            fp.function = f.function;
            int mask = -1;
            if (f.mask_channel >= 0) {
                int mt = 0;
                mask = src_of_channel(f.mask_channel, &mt, in);
                if (mask < 0) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "mask channel out of range");
            }
            int type = TGPU_INT64, src = -1, src2 = -1, type2 = 0;
            if (f.function == TGPU_AGG_SUM_DECIMAL || f.function == TGPU_AGG_AVG_DECIMAL) {
                // DecimalSumAggregation.java:44-146.  Raw input: a short decimal (BIGINT) is summed in 128 bits as BIGINT sums are; a long
                // decimal arrives as its four BIGINT parts (prepare_wide).  State input: the INT128 sum column likewise, plus the overflow
                // column at input_channel + 1.
                const bool wide = wide_virtual(f.input_channel, 0) >= 0;
                int t = 0;
                if (wide) {
                    const int s_high = src_of_channel(wide_virtual(f.input_channel, 0), &t, in);
                    const int s_upper = src_of_channel(wide_virtual(f.input_channel, 2), &t, in);
                    const int s_lower = src_of_channel(wide_virtual(f.input_channel, 3), &t, in);
                    if (s_high < 0 || s_upper < 0 || s_lower < 0) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "too many distinct aggregate inputs");
                    fp.acc_main = add_acc(ACC_SUM_I64_LO, s_high, mask);
                    fp.acc2 = add_acc(ACC_SUM_I64_LO, s_upper, mask);
                    fp.acc3 = add_acc(ACC_SUM_I64_LO, s_lower, mask);
                    fp.acc_count = add_acc(ACC_NONNULL, s_high, mask);
                    if (fp.acc2 < 0 || fp.acc3 < 0) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "too many accumulators");
                    type = TGPU_INT128;
                }
                else {
                    if (from_state) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "the decimal sum state is an INT128 channel followed by a BIGINT overflow channel");
                    src = src_of_channel(f.input_channel, &type, in);
                    if (src < 0) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "aggregate input channel %d out of range", f.input_channel);
                    if (type != TGPU_INT64) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "a decimal sum reads BIGINT (short decimal) or INT128 channels, not type %d", type);
                    fp.acc_main = add_acc(ACC_SUM_I64_LO, src, mask);
                    fp.acc_count = add_acc(ACC_NONNULL, src, mask);
                }
                if (from_state) {
                    const int s_over = src_of_channel(f.input_channel + 1, &t, in);
                    if (s_over < 0 || t != TGPU_INT64) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "the decimal sum state needs its BIGINT overflow channel");
                    fp.acc4 = add_acc(ACC_SUM_I64_LO, s_over, -1);
                    if (fp.acc4 < 0) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "too many accumulators");
                    if (f.function == TGPU_AGG_AVG_DECIMAL) {
                        const int s_rows = src_of_channel(f.input_channel + 2, &t, in);
                        if (s_rows < 0 || t != TGPU_INT64) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "the decimal average state needs its BIGINT row-count channel");
                        fp.acc5 = add_acc(ACC_SUM_I64_LO, s_rows, -1);
                        if (fp.acc5 < 0) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "too many accumulators");
                    }
                }
                if (f.function == TGPU_AGG_AVG_DECIMAL) {
                    fp.result_type = f.reserved == TGPU_INT64 || f.reserved == TGPU_INT128 ? f.reserved : (wide && !from_state ? TGPU_INT128 : from_state ? 0 : TGPU_INT64);
                    if (!fp.result_type) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "a FINAL decimal average needs tgpu_agg_fn.reserved = TGPU_INT64 or TGPU_INT128 (the result type)");
                }
                fp.in_elem_is_double = 0;
                fn_input_types.push_back(type);
                if (fp.acc_main < 0 || fp.acc_count < 0) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "too many accumulators");
                fnplans.push_back(fp);
                continue;
            }
            if (f.function != TGPU_AGG_COUNT_STAR || from_state) {
                src = src_of_channel(f.input_channel, &type, in);
                if (src < 0) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "aggregate input channel %d out of range", f.input_channel);
                if (type == TGPU_UTF8) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "aggregates over variable-width inputs are not supported");
                if (type == TGPU_FLOAT32) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "aggregate function %d over a REAL channel: keep the Java accumulator", f.function);
            }
            bool dbl = type == TGPU_FLOAT64;
            fp.in_elem_is_double = dbl;
            fn_input_types.push_back(type);
            if (!from_state) {
                switch (f.function) {
                    case TGPU_AGG_COUNT_STAR: fp.acc_main = add_acc(ACC_ROWS, -1, mask); break;
                    case TGPU_AGG_COUNT: fp.acc_main = add_acc(ACC_NONNULL, src, mask); break;
                    case TGPU_AGG_SUM:
                        fp.acc_main = add_acc(dbl ? ACC_SUM_F64 : ACC_SUM_I64_LO, src, mask);
                        fp.acc_count = add_acc(ACC_NONNULL, src, mask);
                        break;
                    case TGPU_AGG_AVG:
                        fp.acc_main = add_acc(dbl ? ACC_SUM_F64 : ACC_SUM_F64_FROM_I64, src, mask);
                        fp.acc_count = add_acc(ACC_NONNULL, src, mask);
                        break;
                    case TGPU_AGG_MIN: case TGPU_AGG_MAX:
                        fp.acc_main = add_acc(f.function == TGPU_AGG_MIN ? (dbl ? ACC_MIN_F64 : ACC_MIN_I64) : (dbl ? ACC_MAX_F64 : ACC_MAX_I64), src, mask);
                        fp.acc_count = add_acc(ACC_NONNULL, src, mask);
                        break;
                    default: return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "aggregate function %d", f.function);
                }
            }
            else {
                // combine functions over the intermediate state columns (layout in include/trino_gpu.h)
                switch (f.function) {
                    case TGPU_AGG_COUNT_STAR: case TGPU_AGG_COUNT: fp.acc_main = add_acc(ACC_SUM_I64_LO, src, -1); break;
                    case TGPU_AGG_SUM:
                        fp.acc_main = add_acc(dbl ? ACC_SUM_F64 : ACC_SUM_I64_LO, src, -1);
                        fp.acc_count = add_acc(ACC_NONNULL, src, -1);
                        break;
                    case TGPU_AGG_AVG:
                        src2 = src_of_channel(f.input_channel + 1, &type2, in);
                        if (src2 < 0) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "avg state needs two channels");
                        fp.acc_count = add_acc(ACC_SUM_I64_LO, src, -1);
                        fp.acc_main = add_acc(ACC_SUM_F64, src2, -1);
                        break;
                    case TGPU_AGG_MIN: case TGPU_AGG_MAX:
                        fp.acc_main = add_acc(f.function == TGPU_AGG_MIN ? (dbl ? ACC_MIN_F64 : ACC_MIN_I64) : (dbl ? ACC_MAX_F64 : ACC_MAX_I64), src, -1);
                        fp.acc_count = add_acc(ACC_NONNULL, src, -1);
                        break;
                    default: return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "aggregate function %d", f.function);
                }
            }
            if (fp.acc_main < 0 || (fp.acc_count == -1 && false)) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "too many accumulators");
            fnplans.push_back(fp);
        }
        if (plan.num_srcs > MAX_SRCS) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "too many distinct aggregate inputs");
        // every non-null counter can fall back on the row counter of its mask when its input has no NULLs in a page
        for (int a = 0, n0 = plan.num_accs; a < n0; a++)
            if (plan.accs[a].kind == ACC_NONNULL && add_acc(ACC_ROWS, -1, plan.accs[a].mask) < 0)
                return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "too many accumulators");
        // accumulators sorted by source so the kernels fetch every source once per row
        // (indices are referenced by fnplans: keep positions, the kernels only cache the last source)
        planned = true;
        return TGPU_OK;
    }

    int alloc_state(int64_t cap)
    {
        int A = plan.num_accs > 0 ? plan.num_accs : 1, K = plan.num_keys;
        DevBuf n_keys, n_acc, n_kv, n_kn;
        TG_TRY(n_keys.alloc(ctx, (size_t)cap * 8));
        TG_TRY(n_acc.alloc(ctx, (size_t)cap * 8 * A));
        TG_TRY(n_kv.alloc(ctx, (size_t)cap * 8 * K));
        TG_TRY(n_kn.alloc(ctx, (size_t)cap * K));
        if (st_cap > 0 && group_count > 0) {
            AggState ns;
            ns.count = st_count.as<int32_t>();
            ns.keys = n_keys.as<unsigned long long>();
            ns.acc = n_acc.as<unsigned long long>();
            ns.keyvals = n_kv.as<long long>();
            ns.keynull = n_kn.as<unsigned char>();
            ns.cap = cap;
            TG_CUDA(ctx, cudaMemcpyAsync(ns.keys, st_keys.p, (size_t)std::min(cap, st_cap) * 8, cudaMemcpyDeviceToDevice, ctx->stream));
            TG_LAUNCH(ctx, relayout_state_kernel, tg_grid(ctx, group_count, 256, 8), 256, 0, st_acc.as<unsigned long long>(), st_keyvals.as<long long>(),
                      st_keynull.as<unsigned char>(), st_cap, group_count, plan.num_accs, K, ns);
        }
        st_keys = std::move(n_keys);
        st_acc = std::move(n_acc);
        st_keyvals = std::move(n_kv);
        st_keynull = std::move(n_kn);
        st_cap = cap;
        return TGPU_OK;
    }

    int init_state()
    {
        TG_TRY(st_count.alloc(ctx, 64));
        int32_t init[4] = {0, -1, -1, 0};
        TG_CUDA(ctx, cudaMemcpyAsync(st_count.p, init, sizeof(init), cudaMemcpyHostToDevice, ctx->stream));
        group_count = 0;
        st_cap = 0;
        TG_TRY(alloc_state(S_GMAX + 2));
        use_general = gids_only;
        // path S configuration.  Per-thread private accumulators cost (L+2) x A x 8 bytes of shared memory per
        // thread, so the number of key slots per CTA (L) trades directly against resident warps: start with L = 4
        // (most warps in flight) and escalate 4 -> 8 -> 16 -> 32 when a CTA meets more distinct keys than fit;
        // beyond that the general path takes over.
        int A = plan.num_accs > 0 ? plan.num_accs : 1;
        bool jit = jit_available();
        if (jit) {
            // the specialised kernel drops non-null counters of inputs that cannot be NULL: size for the common case
            int opt = 0;
            for (int a = 0; a < plan.num_accs; a++) opt += plan.accs[a].kind != ACC_NONNULL;
            A = opt > 0 ? opt : 1;
        }
        s_per_slot = (size_t)A * S_THREADS * 8;
        s_fixed = (size_t)(has_pre && !jit ? TGPU_MAX_TEMPS * S_THREADS * 8 : 0) + 1024;
        s_L = 0;
        s_grid = 0;
        if (!set_small_L(4)) use_general = true;
        if (plan.key_hashed) use_general = true;   // the shared-memory path needs exactly packed keys
        if (expected_groups > S_GMAX * 4) use_general = true;   // planner expects many groups: skip the S attempt
        return TGPU_OK;
    }

    // ---- path S -----------------------------------------------------------------------------------
    size_t smem_limit() const { return (ctx->smem_optin > 0 ? ctx->smem_optin : 227 * 1024) - 2048; }

    bool set_small_L(int L)
    {
        size_t need = s_fixed + (size_t)(L + 2) * s_per_slot + (size_t)L * 8 + (size_t)(L + 2) * 8;
        if (L > 32 || need > smem_limit()) return false;
        s_L = L;
        s_smem = need;
        s_grid = 0;   // CTA partial buffers are re-sized for the new L
        return true;
    }

    int run_small(const DevPage& in, const DColumns& cols, bool* overflowed)
    {
        int64_t n = in.rows;
        int L = s_L, A = plan.num_accs;
        // (the specialised kernel of a multi-key plan carries no accumulator sets for the special groups)
        const size_t jit_smem = jit_available() && plan.num_keys > 1 ? s_smem - 2 * s_per_slot : s_smem;
        // at most 3 CTAs per SM: the fourth would cap the kernel at 64 registers, and Q1 spills there
        int ctas_per_sm = (int)std::max<size_t>(1, std::min<size_t>(3, (smem_limit() + 2048) / (jit_smem + 1024)));
        if (const char* e = getenv("TGPU_AGG_S_MINB")) ctas_per_sm = std::max(1, std::min(4, atoi(e)));
        int grid = tg_grid(ctx, n, S_THREADS * 4, ctas_per_sm);
        if (grid != s_grid) {
            TG_TRY(blk_keys.alloc(ctx, (size_t)grid * L * 8));
            TG_TRY(blk_first.alloc(ctx, (size_t)grid * (L + 2) * 8));
            TG_TRY(blk_acc.alloc(ctx, (size_t)grid * (L + 2) * (A > 0 ? A : 1) * 8));
            TG_TRY(blk_ps.alloc(ctx, (size_t)grid * (L + 2) * 4));
            s_grid = grid;
        }
        int* d_overflow = (int*)(ctx->d_scratch + 6);
        unsigned int* d_err = (unsigned int*)(ctx->d_scratch + 6) + 1;
        TG_CUDA(ctx, cudaMemsetAsync(d_overflow, 0, 8, ctx->stream));
        SmallOut so;
        so.blk_keys = blk_keys.as<unsigned long long>();
        so.blk_first = blk_first.as<long long>();
        so.blk_acc = blk_acc.as<unsigned long long>();
        so.overflow = d_overflow;
        so.err = d_err;
        // the kernel specialised for this row program (NVRTC, cached); the interpreter kernel when NVRTC is not there
        AccMap map;
        void* jit_fn = nullptr;
        if (jit_available()) {
            uint32_t nullable = 0;
            int elems[TGPU_MAX_CHANNELS] = {0};
            for (size_t c = 0; c < in.cols.size() && c < TGPU_MAX_CHANNELS; c++) {
                elems[c] = in.cols[c].elem_size();
                if (in.cols[c].validity) nullable |= 1u << c;
            }
            if (jit_elems.empty()) jit_elems.assign(elems, elems + TGPU_MAX_CHANNELS);
            for (size_t c = 0; c < in.cols.size() && c < TGPU_MAX_CHANNELS; c++)
                if (jit_elems[c] != elems[c]) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "channel %zu changed its type between pages", c);
            // four consecutive rows per thread through 16-byte loads when every column starts on a 16-byte boundary (always true for
            // library-owned and cudaMalloc'ed columns; a caller's sliced device column may not be)
            bool vec = !getenv("TGPU_AGG_S_NO_VEC");
            for (size_t c = 0; c < in.cols.size() && c < TGPU_MAX_CHANNELS; c++)
                vec = vec && ((uintptr_t)in.cols[c].data & 15) == 0;
            uint64_t vkey = ((uint64_t)L << 32) | nullable | (vec ? 1ULL << 63 : 0);
            auto it = jit_variants.find(vkey);
            if (it == jit_variants.end()) {
                JitVariant v;
                std::string src = gen_agg_small_source(plan, has_pre ? &host_prog : nullptr, elems, (int)in.cols.size(), L, ctas_per_sm, nullable, &v.map, vec);
                // a generated program that does not compile is a bug, not a fallback case
                TG_TRY(jit_get_function(ctx, src, "tg_agg_small_jit", &v.fn));
                it = jit_variants.emplace(vkey, v).first;
            }
            jit_fn = it->second.fn;
            map = it->second.map;
        }
        else {
            map.compact_count = A;
            for (int a = 0; a < MAX_ACCS; a++) map.of_plan[a] = a;
        }
        TG_TIMED_BEGIN(ctx);
        if (jit_fn) {
            long long n_arg = n;
            DColumns cols_arg = cols;
            void* params[3] = {&cols_arg, &n_arg, &so};
            const int sets = plan.num_keys == 1 ? L + 2 : L;       // (Prog::SPECIALS)
            size_t smem = (size_t)L * 8 + (size_t)(L + 2) * 8 + (size_t)sets * map.compact_count * S_THREADS * 8;
            if (smem + 2048 > (ctx->smem_optin > 0 ? ctx->smem_optin : 227 * 1024)) { *overflowed = true; return TGPU_OK; }   // too many live accumulators for path S
            TG_TRY(jit_launch(ctx, jit_fn, grid, S_THREADS, smem, params));
        }
        else {
            TG_CUDA(ctx, cudaFuncSetAttribute(agg_small_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)s_smem));
            TG_LAUNCH(ctx, agg_small_kernel, grid, S_THREADS, s_smem, plan, cols, has_pre ? d_prog.as<DProgram>() : nullptr, n, L, so);
        }
        TG_TIMED_END(ctx);
        TG_LAUNCH(ctx, agg_small_merge_kernel, 1, 256, 0, plan, cols, grid, L, so, state(), blk_ps.as<int>(), map);
        // one small readback per page: overflow flag + error bits, then the group count
        int64_t word = 0;
        TG_TRY(tg_read_i64(ctx, d_overflow, &word));
        if ((uint32_t)(word >> 32)) TG_TRY(raise((uint32_t)(word >> 32)));
        *overflowed = (word & 0xFFFFFFFFLL) != 0;
        if (!*overflowed) {
            int64_t cnt = 0;
            TG_TRY(tg_read_i64(ctx, st_count.p, &cnt));
            group_count = (int32_t)(cnt & 0xFFFFFFFFLL);
        }
        return TGPU_OK;
    }

    int raise(uint32_t errbits)
    {
        if (errbits & TG_ERR_BIT_DIV_ZERO) return tg_fail(ctx, TGPU_ERR_DIVISION_BY_ZERO, "Division by zero");
        if (errbits & TG_ERR_BIT_OVERFLOW) return tg_fail(ctx, TGPU_ERR_NUMERIC_VALUE_OUT_OF_RANGE, "bigint arithmetic overflow");
        return TGPU_OK;
    }

    // ---- path G -----------------------------------------------------------------------------------
    int g_alloc_table(int64_t slots)
    {
        DevBuf nt;
        TG_TRY(nt.alloc(ctx, (size_t)slots * sizeof(GSlot)));
        TG_LAUNCH(ctx, g_table_init_kernel, tg_grid(ctx, slots, 1024, 8), 256, 0, nt.as<int4>(), slots);
        if (g_slots > 0)
            TG_LAUNCH(ctx, g_rehash_kernel, tg_grid(ctx, g_slots, 1024, 8), 256, 0, g_table.as<GSlot>(), g_slots, nt.as<GSlot>(), (unsigned long long)slots - 1);
        g_table = std::move(nt);
        g_slots = slots;
        return TGPU_OK;
    }

    // the fused pre-stage as a stand-alone FilterAndProject operator (the reference's own operator chain)
    int make_pre_filter_project(tgpu_op** out)
    {
        std::vector<tgpu_in_list> lists(pre_in_values.size());
        for (size_t i = 0; i < lists.size(); i++) { lists[i].count = (int32_t)pre_in_values[i].size(); lists[i].values = pre_in_values[i].data(); }
        tgpu_expr_program prog;
        memset(&prog, 0, sizeof(prog));
        prog.num_insns = (int32_t)pre_insns.size();
        prog.insns = pre_insns.data();
        prog.filter_temp = pre_filter_temp;
        prog.num_filter_insns = pre_num_filter_insns;
        prog.num_projections = (int32_t)projections.size();
        prog.projections = projections.data();
        prog.num_in_lists = (int32_t)lists.size();
        prog.in_lists = lists.data();
        return tgpu_filter_project_create(ctx, &prog, out);
    }

    int switch_to_general()
    {
        use_general = true;
        if (has_pre) {
            // the general path works on materialised projection outputs: un-fuse the pre-stage into its own
            // FilterAndProject (the reference's own operator chain) and re-point every source at its output channel
            TG_TRY(make_pre_filter_project(&inner_fp));
            for (int i = 0; i < plan.num_srcs; i++) plan.srcs[i] = SrcRef{0, src_channel[i], 0, 0};
            plan.has_pre = 0;
            has_pre = false;
        }
        if (fused_ok() && !getenv("TGPU_AGG_MULTIPASS")) return gf_start();
        TG_TRY(g_special.alloc(ctx, sizeof(GSpecial)));
        GSpecial init;
        init.gid[0] = init.gid[1] = -1;
        init.first_row[0] = init.first_row[1] = 0x7FFFFFFF;
        TG_CUDA(ctx, cudaMemcpyAsync(g_special.p, &init, sizeof(init), cudaMemcpyHostToDevice, ctx->stream));
        TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        int64_t want = expected_groups > 0 ? expected_groups : 1024;
        int64_t slots = 1 << 16;
        while (slots * 3 / 4 < want + group_count) slots <<= 1;    // arraySize(expected, 0.75)
        if (slots > (1LL << 30)) return tg_fail(ctx, TGPU_ERR_INSUFFICIENT_RESOURCES, "Size of hash table cannot exceed 1 billion entries");
        g_slots = 0;
        TG_TRY(g_alloc_table(slots));
        if (group_count > 0)
            TG_LAUNCH(ctx, g_migrate_kernel, 1, 256, 0, state(), g_table.as<GSlot>(), (unsigned long long)g_slots - 1, g_special.as<GSpecial>());
        return TGPU_OK;
    }

    // assigns group ids for the page into d_gids (int32[n]); updates group_count
    int run_general_ids(const DevPage& in, const DColumns& cols, int* d_gids)
    {
        int64_t n = in.rows;
        if (n > (int64_t)INT32_MAX) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "page has more than 2^31-1 positions");
        DevBuf slot_of_row, flags, rank, tmp;
        TG_TRY(slot_of_row.alloc(ctx, (size_t)n * 4));
        TG_TRY(flags.alloc(ctx, (size_t)n + 1));
        TG_TRY(rank.alloc(ctx, (size_t)(n + 1) * 4));
        int* d_tickets = (int*)(ctx->d_scratch + 8);
        int* d_overflow = d_tickets + 1;
        int* d_retry_count = (int*)(ctx->d_scratch + 18);
        int grid = tg_grid(ctx, n, 256, 8);
        DevBuf attempt, retry_a, retry_b;
        if (plan.key_hashed) TG_TRY(attempt.alloc(ctx, (size_t)n));
        while (true) {
            // hashed composite keys: rows settle under the first of their hash functions whose slot holds their own key tuple
            if (plan.key_hashed) TG_CUDA(ctx, cudaMemsetAsync(attempt.p, 0, (size_t)n, ctx->stream));
            const int* rows = nullptr;
            int64_t todo = n;
            bool overflow = false;
            int64_t claimed = 0;
            for (int round = 0; ; round++) {
                if (round >= 8) return tg_fail(ctx, TGPU_ERR_INSUFFICIENT_RESOURCES, "group-by keys collide under 8 independent 64-bit hashes");
                int64_t max_fill = g_slots * 3 / 4;
                int64_t budget = max_fill - group_count - claimed;
                TG_CUDA(ctx, cudaMemsetAsync(d_tickets, 0, 8, ctx->stream));
                TG_LAUNCH(ctx, g_insert_kernel, tg_grid(ctx, todo, 256, 8), 256, 0, plan, cols, todo, rows, plan.key_hashed ? attempt.as<unsigned char>() : nullptr,
                          g_table.as<GSlot>(), (unsigned long long)g_slots - 1, g_special.as<GSpecial>(),
                          slot_of_row.as<int>(), d_tickets, (int)std::min<int64_t>(std::max<int64_t>(budget, 0), INT32_MAX), d_overflow);
                int64_t word = 0;
                TG_TRY(tg_read_i64(ctx, d_tickets, &word));
                overflow = (word >> 32) != 0;
                claimed += word & 0xFFFFFFFFLL;
                if (overflow || !plan.key_hashed) break;
                DevBuf& retry = (round & 1) ? retry_b : retry_a;
                TG_TRY(retry.alloc(ctx, (size_t)todo * 4));
                TG_CUDA(ctx, cudaMemsetAsync(d_retry_count, 0, 8, ctx->stream));
                TG_LAUNCH(ctx, g_verify_kernel, tg_grid(ctx, todo, 256, 8), 256, 0, plan, cols, todo, rows, g_table.as<GSlot>(), slot_of_row.as<int>(), state(),
                          attempt.as<unsigned char>(), retry.as<int>(), d_retry_count);
                int64_t left = 0;
                TG_TRY(tg_read_i64(ctx, d_retry_count, &left));
                left &= 0xFFFFFFFFLL;
                if (left == 0) break;
                rows = retry.as<int>();
                todo = left;
            }
            if (!overflow) break;
            // BigintGroupByHash.tryRehash :239-290: double (here: x4) and retry the page
            int64_t slots = g_slots * 4;
            if (slots > (1LL << 30)) return tg_fail(ctx, TGPU_ERR_INSUFFICIENT_RESOURCES, "Size of hash table cannot exceed 1 billion entries");
            TG_TRY(g_alloc_table(slots));
            TG_LAUNCH(ctx, g_reset_provisional_kernel, 1, 32, 0, g_table.as<GSlot>(), (int64_t)0, g_special.as<GSpecial>());
        }
        TG_LAUNCH(ctx, g_flag_kernel, grid, 256, 0, n, g_table.as<GSlot>(), g_special.as<GSpecial>(), slot_of_row.as<int>(), flags.as<unsigned char>());
        size_t tmp_bytes = 0;
        cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, flags.as<unsigned char>(), rank.as<int>(), n + 1, ctx->stream);
        TG_TRY(tmp.alloc(ctx, tmp_bytes));
        TG_CUDA(ctx, cub::DeviceScan::ExclusiveSum(tmp.p, tmp_bytes, flags.as<unsigned char>(), rank.as<int>(), n + 1, ctx->stream));
        TG_CUDA(ctx, cudaMemcpyAsync(ctx->h_scratch, rank.as<int>() + n, 4, cudaMemcpyDeviceToHost, ctx->stream));
        TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        int32_t total_new = *(int32_t*)ctx->h_scratch;
        if (group_count + total_new > st_cap) {
            int64_t cap = st_cap;
            while (cap < group_count + total_new) cap *= 2;
            TG_TRY(alloc_state(cap));
        }
        if (total_new > 0)
            TG_LAUNCH(ctx, g_assign_kernel, grid, 256, 0, plan, cols, n, g_table.as<GSlot>(), g_special.as<GSpecial>(), slot_of_row.as<int>(),
                      flags.as<unsigned char>(), rank.as<int>(), (int)group_count, state());
        TG_LAUNCH(ctx, g_gid_kernel, grid, 256, 0, n, g_table.as<GSlot>(), g_special.as<GSpecial>(), slot_of_row.as<int>(), d_gids);
        group_count += total_new;
        return TGPU_OK;
    }

    int run_general(const DevPage& in, const DColumns& cols)
    {
        if (fused_general) return run_fused_general(in, cols);
        DevBuf gids;
        TG_TRY(gids.alloc(ctx, (size_t)in.rows * 4));
        TG_TRY(run_general_ids(in, cols, gids.as<int>()));
        if (plan.num_accs > 0)
            TG_LAUNCH(ctx, g_accumulate_kernel, tg_grid(ctx, in.rows, 256, 8), 256, 0, plan, cols, in.rows, gids.as<int>(), state());
        return TGPU_OK;
    }


    // ---- path G, fused form -------------------------------------------------------------------------
    bool fused_ok() const
    {
        if (gids_only || plan.key_hashed) return false;
        for (int k = 0; k < plan.num_keys; k++)
            if (plan.key_is_double[k]) return false;   // first-seen raw value (-0.0 vs +0.0) needs the representative row
        return true;
    }

    int gf_words() const
    {
        int need = 2 + (plan.num_accs > 0 ? plan.num_accs : 0);
        int w = 4;
        while (w < need) w <<= 1;
        return w;
    }

    int gf_alloc(int64_t cap, DevBuf* recs)
    {
        int W = gf_words();
        TG_TRY(recs->alloc(ctx, (size_t)(cap + 2) * W * 8));
        TG_LAUNCH(ctx, gf_init_kernel, tg_grid(ctx, (cap + 2) * W / 2, 1024, 8), 256, 0, recs->as<unsigned long long>(), cap, W, plan);
        return TGPU_OK;
    }

    int gf_start()
    {
        int64_t want = expected_groups > 0 ? expected_groups : 1024;
        int64_t cap = 1 << 16;
        const char* e_load = getenv("TGPU_AGG_G_SIZE_PCT");     // initial sizing only: the fill limit stays 3/4 (tryRehash)
        const int64_t pct = e_load ? atoi(e_load) : 50;     // probe sequences (and the warp-wide lock step over them) are short at <= 1/2 full
        while (cap * pct / 100 < want + group_count) cap <<= 1;
        if (cap > (1LL << 30)) return tg_fail(ctx, TGPU_ERR_INSUFFICIENT_RESOURCES, "Size of hash table cannot exceed 1 billion entries");
        TG_TRY(gf_alloc(cap, &f_recs));
        f_cap = cap;
        f_used = 0;
        if (group_count > 0) {
            TG_LAUNCH(ctx, gf_migrate_kernel, 1, 256, 0, state(), plan, f_recs.as<unsigned long long>(), f_cap, gf_words());
            f_used = group_count;   // migrated specials counted here too: they only ever under-use the budget
        }
        fused_general = true;
        return TGPU_OK;
    }

    int gf_grow()
    {
        int64_t ncap = f_cap * 4;
        if (ncap > (1LL << 30)) return tg_fail(ctx, TGPU_ERR_INSUFFICIENT_RESOURCES, "Size of hash table cannot exceed 1 billion entries");
        DevBuf nr;
        TG_TRY(gf_alloc(ncap, &nr));
        TG_LAUNCH(ctx, gf_rehash_kernel, tg_grid(ctx, f_cap + 2, 1024, 8), 256, 0, f_recs.as<unsigned long long>(), f_cap, nr.as<unsigned long long>(), ncap, gf_words(),
                  plan.num_accs);
        f_recs = std::move(nr);
        f_cap = ncap;
        return TGPU_OK;
    }

    // the fused general kernel specialised for this plan (NVRTC; same row program as the path-S kernel), or nullptr without NVRTC
    int general_jit_function(const DColumns& cols, void** fn)
    {
        *fn = nullptr;
        if (!jit_available() || getenv("TGPU_AGG_GENERAL_INTERPRETED")) return TGPU_OK;
        // the page layout the general path sees (the projection's output once the pre-stage was un-fused): element widths + NULL-ability
        int elems[TGPU_MAX_CHANNELS];
        uint64_t key = 0;
        for (int c = 0; c < TGPU_MAX_CHANNELS; c++) {
            elems[c] = cols.cols[c].data ? cols.cols[c].elem : 0;
            key = key * 0x100000001B3ULL + (uint64_t)(elems[c] * 2 + (cols.cols[c].validity ? 1 : 0));
        }
        uint32_t nullable = 0;
        for (int c = 0; c < TGPU_MAX_CHANNELS; c++)
            if (cols.cols[c].validity) nullable |= 1u << c;
        auto it = jit_g_variants.find(key);
        if (it == jit_g_variants.end()) {
            AccMap unused;
            std::string src = gen_agg_small_source(plan, has_pre ? &host_prog : nullptr, elems, TGPU_MAX_CHANNELS, 4, 2, nullable, &unused);
            void* f = nullptr;
            TG_TRY(jit_get_function(ctx, src, "tg_agg_general_jit", &f));
            it = jit_g_variants.emplace(key, f).first;
        }
        *fn = it->second;
        return TGPU_OK;
    }

    // one pass of the fused general kernel over `todo` rows (`rows` == nullptr: rows [first, first + todo) of the page), replaying deferred
    // rows after growth
    int run_fused_rows(const DColumns& cols, const int* rows, int64_t todo, int64_t first = 0, const int* stamp_rows = nullptr)
    {
        DevBuf deferred, replay;
        TG_TRY(deferred.alloc(ctx, (size_t)std::max<int64_t>(todo, 1) * 4));
        void* jit_fn = nullptr;
        TG_TRY(general_jit_function(cols, &jit_fn));
        constexpr int WAYS = TGD_TICKET_WAYS;
        if (!f_tickets.p) TG_TRY(f_tickets.alloc(ctx, (WAYS + 4) * 4));
        int* d_tickets = f_tickets.as<int>();    // interpreted kernel: [0] claims, [1] deferred rows, [2] specials born; specialised: [0, WAYS) claims, [WAYS] deferred, [WAYS+1] specials, [WAYS+2] error bits
        std::vector<int32_t> counters(WAYS + 4);
        while (true) {
            int64_t budget = f_cap * 3 / 4 - f_used;
            TG_CUDA(ctx, cudaMemsetAsync(d_tickets, 0, (WAYS + 4) * 4, ctx->stream));
            int grid = tg_grid(ctx, todo, 256, 8);
            TG_TIMED_BEGIN(ctx);
            if (jit_fn) {
                DColumns cols_arg = cols;
                long long n_arg = todo, first_arg = first, base_arg = (long long)rows_seen, cap_arg = f_cap;
                const int* rows_arg = rows;
                const int* stamps_arg = stamp_rows;
                unsigned long long* recs_arg = f_recs.as<unsigned long long>();
                int w_arg = gf_words(), per_way = (int)std::min<int64_t>(std::max<int64_t>(budget, 0) / WAYS, INT32_MAX);
                int* tickets_arg = d_tickets;
                int* deferred_arg = deferred.as<int>();
                unsigned int* err_arg = (unsigned int*)(d_tickets + WAYS + 2);
                void* params[13] = {&cols_arg, &n_arg, &rows_arg, &first_arg, &stamps_arg, &base_arg, &recs_arg, &cap_arg, &w_arg, &tickets_arg, &per_way, &deferred_arg, &err_arg};
                grid = (int)std::min<int64_t>(tg_div_up(todo, 256 * general_rows_per_thread()), (int64_t)ctx->sm_count * std::max(1, jit_blocks_per_sm(jit_fn, 256, 0)));
                TG_TRY(jit_launch(ctx, jit_fn, std::max(grid, 1), 256, 0, params));
            }
            else
                TG_LAUNCH(ctx, gf_page_kernel, grid, 256, 0, plan, cols, todo, rows, first, stamp_rows, (long long)rows_seen, f_recs.as<unsigned long long>(), f_cap,
                          gf_words(), d_tickets, (int)std::min<int64_t>(std::max<int64_t>(budget, 0), INT32_MAX), deferred.as<int>());
            TG_TIMED_END(ctx);
            TG_CUDA(ctx, cudaMemcpyAsync(counters.data(), d_tickets, (WAYS + 4) * 4, cudaMemcpyDeviceToHost, ctx->stream));
            TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
            int64_t left;
            if (jit_fn) {
                for (int w = 0; w < WAYS; w++) f_used += counters[w];
                f_specials += counters[WAYS + 1];
                left = counters[WAYS];
                TG_TRY(raise((uint32_t)counters[WAYS + 2]));
            }
            else {
                f_used += counters[0];
                f_specials += counters[2];
                left = counters[1];
            }
            if (left == 0) break;
            // BigintGroupByHash.tryRehash :239-290 (here x4), then replay the rows that found the table full
            TG_TRY(gf_grow());
            replay = std::move(deferred);
            TG_TRY(deferred.alloc(ctx, (size_t)left * 4));
            rows = replay.as<int>();
            todo = left;
        }
        return TGPU_OK;
    }

    // Sliced pass over a slice-ORDERED COPY of the page: the channels the plan reads (and the page row numbers, for the stamps) are
    // moved into slice order by the stable multi-split, so every slice launch streams its rows instead of gathering them through a
    // row list (which cost a 2-sector DRAM fetch per value).  *done = false: shape not handled, use the row-list form.
    // (tests/test_gpu_groupby.py::test_general_path_physical_slices_match_oracle; the fused single-launch form below took over the default)
    int run_physical_slices(const DevPage& in, const DColumns& cols, int64_t n, int log_slices, int log_cap, bool* done)
    {
        *done = false;
        const int S = 1 << log_slices;
        bool used[TGPU_MAX_CHANNELS] = {false};
        for (int i = 0; i < plan.num_srcs; i++) {
            if (plan.srcs[i].is_temp) return TGPU_OK;
            if (plan.srcs[i].index < 0 || plan.srcs[i].index >= (int)in.cols.size()) return TGPU_OK;
            used[plan.srcs[i].index] = true;
        }
        struct Lane { int elem; const void* src; int col; bool nulls; DevBuf buf; };
        std::vector<Lane> lanes;
        for (int c = 0; c < (int)in.cols.size() && c < TGPU_MAX_CHANNELS; c++) {
            if (!used[c]) continue;
            if (in.cols[c].elem_size() == 0) return TGPU_OK;
            lanes.push_back(Lane{in.cols[c].elem_size(), in.cols[c].data, c, false, DevBuf()});
            if (in.cols[c].validity) lanes.push_back(Lane{0, in.cols[c].validity, c, true, DevBuf()});
        }
        lanes.push_back(Lane{XCHG_ROW_NUMBER, nullptr, -1, false, DevBuf()});
        if ((int)lanes.size() > XMAXC || S > XMAXP) return TGPU_OK;
        const XchgGeom geom = xchg_geom(ctx, n, S, true);     // CTA tiles: any number of slices up to 64, row-number lane supported
        DevBuf ids, hist, block_off, d_totals;
        TG_TRY(ids.alloc(ctx, (size_t)n));
        TG_TRY(hist.alloc(ctx, (size_t)geom.nchunks * S * 4));
        TG_TRY(block_off.alloc(ctx, (size_t)geom.nchunks * S * 8));
        TG_TRY(d_totals.alloc(ctx, (size_t)S * 8));
        TG_LAUNCH(ctx, gf_slice_hist_kernel, geom.grid, XT, 0, plan, cols, n, geom.chunk, f_cap, log_cap - log_slices, S, ids.as<uint8_t>(), hist.as<unsigned int>());
        TG_LAUNCH(ctx, xchg_offsets_kernel, S, 256, 0, hist.as<unsigned int>(), geom.nchunks, S, block_off.as<long long>(), d_totals.as<long long>());
        std::vector<long long> counts(S), off(S + 1, 0);
        TG_CUDA(ctx, cudaMemcpyAsync(counts.data(), d_totals.p, (size_t)S * 8, cudaMemcpyDeviceToHost, ctx->stream));
        TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        for (int q = 0; q < S; q++) off[q + 1] = off[q] + counts[q];
        if (off[S] != n) return tg_fail(ctx, TGPU_ERR_ILLEGAL_STATE, "slice counts %lld != rows %lld", off[S], (long long)n);
        std::vector<char*> h_dst(lanes.size() * S);
        for (size_t l = 0; l < lanes.size(); l++) {
            size_t es = lanes[l].elem == XCHG_ROW_NUMBER ? 4 : lanes[l].elem ? (size_t)lanes[l].elem : 1;
            TG_TRY(lanes[l].buf.alloc(ctx, (size_t)n * es));
            for (int q = 0; q < S; q++) h_dst[l * S + q] = (char*)lanes[l].buf.p + (size_t)off[q] * es;
        }
        DevBuf d_dst;
        TG_TRY(d_dst.alloc(ctx, h_dst.size() * sizeof(char*)));
        TG_CUDA(ctx, cudaMemcpyAsync(d_dst.p, h_dst.data(), h_dst.size() * sizeof(char*), cudaMemcpyHostToDevice, ctx->stream));
        XchgCols xc;
        memset(&xc, 0, sizeof(xc));
        xc.count = (int32_t)lanes.size();
        for (size_t l = 0; l < lanes.size(); l++) { xc.elem[l] = lanes[l].elem; xc.src[l] = lanes[l].src; }
        xc.dst = d_dst.as<char*>();
        // (rows of a slice may arrive in any order: their page row numbers travel in the stamp lane)
        TG_TRY(xchg_launch_scatter(ctx, geom, ids.as<uint8_t>(), n, S, block_off.as<long long>(), xc, nullptr, 0, nullptr, !getenv("TGPU_AGG_STABLE_SCATTER")));
        // the slice-ordered page: same channel numbers, data and validity of the channels the plan reads replaced by the copies
        DColumns pcols = cols;
        std::vector<DevColumn> packed_keep;
        const int* stamp_rows = nullptr;
        for (auto& lane : lanes) {
            if (lane.elem == XCHG_ROW_NUMBER) { stamp_rows = lane.buf.as<int>(); continue; }
            if (!lane.nulls) { pcols.cols[lane.col].data = lane.buf.p; continue; }
            tgpu_column bm;
            memset(&bm, 0, sizeof(bm));
            bm.type = TGPU_INT8;
            bm.flags = TGPU_COL_NULLS_BYTEMAP;
            bm.length = n;
            bm.data = lane.buf.p;
            bm.validity = lane.buf.as<uint8_t>();
            DevColumn packed;
            TG_TRY(tg_ingest_column(ctx, &bm, true, &packed));
            pcols.cols[lane.col].validity = packed.validity;
            packed_keep.push_back(std::move(packed));
        }
        // ONE launch over the slice-ordered copy: a grid-stride pass keeps every CTA in the same neighbourhood of the row array, i.e. in
        // the same table slice, so the slice's records stay in the L2 without a launch (and a host round trip) per slice
        TG_TRY(run_fused_rows(pcols, nullptr, n, 0, stamp_rows));
        TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));   // the copies are released below: the last slice launch must be done with them
        *done = true;
        return TGPU_OK;
    }

    int run_fused_general(const DevPage& in, const DColumns& cols)
    {
        int64_t n = in.rows;
        if (n > (int64_t)INT32_MAX) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "page has more than 2^31-1 positions");
        // table much larger than the L2 and a page worth reordering: visit the table slice by slice
        const size_t table_bytes = (size_t)f_cap * gf_words() * 8;
        // (thresholds can be lowered from the environment so that the parity tests reach this path with small inputs)
        const char* e_bytes = getenv("TGPU_AGG_SLICE_MIN_BYTES");
        const char* e_target = getenv("TGPU_AGG_SLICE_BYTES");
        const size_t min_bytes = e_bytes ? (size_t)atoll(e_bytes) : ((size_t)96 << 20);
        const size_t slice_bytes = e_target ? (size_t)atoll(e_target) : ((size_t)16 << 20);
        if (!getenv("TGPU_AGG_NO_SLICES") && table_bytes >= min_bytes && n >= (e_bytes ? 1 : (1 << 20))) {
            int log_slices = 1;
            while (log_slices < 6 && (table_bytes >> log_slices) > slice_bytes) log_slices++;
            const int S = 1 << log_slices;
            int log_cap = 0;
            while ((1LL << log_cap) < f_cap) log_cap++;
            if (!getenv("TGPU_AGG_ROWLIST_SLICES")) {
                bool done = false;
                TG_TRY(run_physical_slices(in, cols, n, log_slices, log_cap, &done));
                if (done) {
                    rows_seen += n;
                    group_count = f_used + f_specials;
                    return TGPU_OK;
                }
            }
            DevBuf ids, ids_sorted, rows_in, rows_sorted, tmp;
            TG_TRY(ids.alloc(ctx, (size_t)n));
            TG_TRY(ids_sorted.alloc(ctx, (size_t)n));
            TG_TRY(rows_in.alloc(ctx, (size_t)n * 4));
            TG_TRY(rows_sorted.alloc(ctx, (size_t)n * 4));
            unsigned int* d_counts = (unsigned int*)(ctx->d_scratch + 32);   // 64 counters
            TG_CUDA(ctx, cudaMemsetAsync(d_counts, 0, 64 * 4, ctx->stream));
            TG_LAUNCH(ctx, gf_slice_ids_kernel, tg_grid(ctx, n, 256, 8), 256, 0, plan, cols, n, f_cap, log_cap - log_slices, ids.as<uint8_t>(), d_counts);
            TG_LAUNCH(ctx, gf_iota_kernel, tg_grid(ctx, n, 1024, 8), 256, 0, rows_in.as<int>(), n);
            size_t tmp_bytes = 0;
            cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, ids.as<uint8_t>(), ids_sorted.as<uint8_t>(), rows_in.as<int>(), rows_sorted.as<int>(), (int)n, 0, log_slices, ctx->stream);
            TG_TRY(tmp.alloc(ctx, tmp_bytes));
            TG_CUDA(ctx, cub::DeviceRadixSort::SortPairs(tmp.p, tmp_bytes, ids.as<uint8_t>(), ids_sorted.as<uint8_t>(), rows_in.as<int>(), rows_sorted.as<int>(), (int)n, 0,
                                                         log_slices, ctx->stream));
            unsigned int counts[64];
            TG_CUDA(ctx, cudaMemcpyAsync(ctx->h_scratch, d_counts, 64 * 4, cudaMemcpyDeviceToHost, ctx->stream));
            TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
            memcpy(counts, ctx->h_scratch, sizeof(counts));
            int64_t off = 0;
            for (int q = 0; q < S; q++) {
                if (counts[q]) TG_TRY(run_fused_rows(cols, rows_sorted.as<int>() + off, counts[q]));
                off += counts[q];
            }
            if (off != n) return tg_fail(ctx, TGPU_ERR_ILLEGAL_STATE, "slice counts %lld != rows %lld", (long long)off, (long long)n);
        }
        else TG_TRY(run_fused_rows(cols, nullptr, n));
        rows_seen += n;
        group_count = f_used + f_specials;
        return TGPU_OK;
    }

    // compact used slots, order them by first-row stamp, gather the state into group-id order
    int gf_finalize()
    {
        int64_t total = f_cap + 2;
        DevBuf flags, slots, tmp;
        TG_TRY(flags.alloc(ctx, (size_t)total));
        TG_TRY(slots.alloc(ctx, (size_t)total * 4));
        TG_LAUNCH(ctx, gf_used_flags_kernel, tg_grid(ctx, total, 1024, 8), 256, 0, f_recs.as<unsigned long long>(), total, gf_words(), flags.as<unsigned char>());
        long long* d_count = (long long*)(ctx->d_scratch + 22);
        size_t tmp_bytes = 0;
        thrust::counting_iterator<int> iota(0);
        cub::DeviceSelect::Flagged(nullptr, tmp_bytes, iota, flags.as<unsigned char>(), slots.as<int>(), d_count, (int)total, ctx->stream);
        TG_TRY(tmp.alloc(ctx, tmp_bytes));
        TG_CUDA(ctx, cub::DeviceSelect::Flagged(tmp.p, tmp_bytes, iota, flags.as<unsigned char>(), slots.as<int>(), d_count, (int)total, ctx->stream));
        int64_t G = 0;
        TG_TRY(tg_read_i64(ctx, d_count, &G));
        group_count = G;
        if (G == 0) return TGPU_OK;
        DevBuf k_in, k_out, s_out, tmp2;
        TG_TRY(k_in.alloc(ctx, (size_t)G * 8));
        TG_TRY(k_out.alloc(ctx, (size_t)G * 8));
        TG_TRY(s_out.alloc(ctx, (size_t)G * 4));
        TG_LAUNCH(ctx, gf_sort_keys_kernel, tg_grid(ctx, G, 1024, 8), 256, 0, f_recs.as<unsigned long long>(), gf_words(), slots.as<int>(), G, k_in.as<unsigned long long>());
        tmp_bytes = 0;
        cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, k_in.as<unsigned long long>(), k_out.as<unsigned long long>(), slots.as<int>(), s_out.as<int>(), (int)G, 0, 64, ctx->stream);
        TG_TRY(tmp2.alloc(ctx, tmp_bytes));
        TG_CUDA(ctx, cub::DeviceRadixSort::SortPairs(tmp2.p, tmp_bytes, k_in.as<unsigned long long>(), k_out.as<unsigned long long>(), slots.as<int>(), s_out.as<int>(), (int)G, 0, 64, ctx->stream));
        if (G > st_cap) {
            int64_t keep = group_count;
            group_count = 0;            // nothing to carry over: the dense arrays are rebuilt from the slots
            TG_TRY(alloc_state(G));
            group_count = keep;
        }
        TG_LAUNCH(ctx, gf_gather_kernel, tg_grid(ctx, G, 256, 8), 256, 0, plan, s_out.as<int>(), G, f_recs.as<unsigned long long>(), f_cap, gf_words(), state());
        return TGPU_OK;
    }

    // ---- Operator protocol --------------------------------------------------------------------------
    bool needs_input() override { return !finishing && !flushing && next_out >= pending.size(); }

    int fill_cols(const DevPage& in, DColumns* cols)
    {
        memset(cols, 0, sizeof(*cols));
        if (in.cols.size() > TGPU_MAX_CHANNELS) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "more than %d channels", TGPU_MAX_CHANNELS);
        for (size_t c = 0; c < in.cols.size(); c++) cols->cols[c] = tg_colref(in.cols[c]);
        return TGPU_OK;
    }

    int add_input(const tgpu_page* page) override
    {
        if (page->num_rows == 0) return TGPU_OK;
        if (!builder_open) {
            // HashAggregationOperator.addInput :358-372: the controller is consulted when a builder is created
            builder_open = true;
            skip_mode = controller && controller->disabled.load(std::memory_order_acquire);
            builder_bytes = builder_rows = builder_unique = 0;
        }
        builder_rows += page->num_rows;
        if (skip_mode) return add_input_skipped(page);
        if (use_general && inner_fp) {
            if (controller) builder_bytes += reference_page_bytes(page);
            return add_via_filter_project(page);
        }
        DevPage in;
        TG_TRY(tg_ingest_page(ctx, page, &in));
        if (controller) builder_bytes += reference_page_bytes(in);
        TG_TRY(prepare_wide(&in));
        TG_TRY(encode_string_keys(&in));
        if (!planned) {
            TG_TRY(make_plan(in));
            TG_TRY(init_state());
            if (use_general) {
                TG_TRY(switch_to_general());
                if (inner_fp) return add_via_filter_project(page);
            }
        }
        if (has_pre && prog_max_channel >= (int)in.cols.size())
            return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "pre-stage reads channel %d, page has %zu", prog_max_channel, in.cols.size());
        DColumns cols;
        TG_TRY(fill_cols(in, &cols));
        if (!use_general) {
            while (true) {
                bool overflowed = false;
                TG_TRY(run_small(in, cols, &overflowed));
                if (!overflowed) return after_page();
                // the state is untouched by an overflowed pass: retry the page with more key slots per CTA
                if (group_count + 2 <= S_GMAX && set_small_L(s_L * 2)) continue;
                break;
            }
            TG_TRY(switch_to_general());
            if (inner_fp) return add_via_filter_project(page);
        }
        TG_TRY(run_general(in, cols));
        return after_page();
    }

    // Page.getSizeInBytes() of the same page on the Java side: value bytes plus one isNull byte per position (LongArrayBlock.getSizeInBytes,
    // S/block/LongArrayBlock.java:93-96), variable width adds the 4-byte offset (S/block/VariableWidthBlock.java:137-140)
    static int64_t reference_column_bytes(int type, int64_t n, int64_t utf8_bytes)
    {
        switch (type) {
            case TGPU_INT64: case TGPU_FLOAT64: return 9 * n;
            case TGPU_INT32: return 5 * n;
            case TGPU_INT16: return 3 * n;
            case TGPU_INT8: return 2 * n;
            case TGPU_UTF8: return utf8_bytes + 5 * n;
            default: return 9 * n;
        }
    }
    static int64_t reference_page_bytes(const DevPage& in)
    {
        int64_t b = 0;
        for (auto& c : in.cols) b += reference_column_bytes(c.type, c.length, c.data_bytes);
        return b;
    }
    static int64_t reference_page_bytes(const tgpu_page* page)
    {
        int64_t b = 0;
        for (int c = 0; c < page->num_columns; c++) {
            const tgpu_column& col = page->columns[c];
            int type = col.type == TGPU_DICT32 || col.type == TGPU_RLE ? (col.dictionary ? col.dictionary->type : TGPU_INT64) : col.type;
            // (variable-width bytes of a device page are not known without a read-back: the offsets and null bytes stand for the column)
            b += reference_column_bytes(type, col.length, 0);
        }
        return b;
    }

    // One page through a skipped builder (SkipAggregationBuilder.processPage / buildResult): the output is parked in `pending`, so
    // needs_input() is false until the caller has taken it (isFull() == currentPage != null)
    int add_input_skipped(const tgpu_page* page)
    {
        const bool from_state = step == TGPU_STEP_INTERMEDIATE;
        tgpu_op* fp = inner_fp;
        if (has_pre) {
            if (!skip_fp) TG_TRY(make_pre_filter_project(&skip_fp));
            fp = skip_fp;
        }
        std::vector<std::unique_ptr<OwnedPage>> projected;
        DevPage raw;
        std::vector<const DevPage*> pages;
        if (fp) {
            builder_bytes += reference_page_bytes(page);
            TG_TRY(fp->add_input(page));
            while (true) {
                OwnedPage* o = nullptr;
                TG_TRY(fp->get_output(&o));
                if (!o) break;
                projected.emplace_back(o);
                pages.push_back(&o->page);
            }
        }
        else {
            TG_TRY(tg_ingest_page(ctx, page, &raw));
            builder_bytes += reference_page_bytes(raw);
            pages.push_back(&raw);
        }
        rows_skipped += page->num_rows;
        for (const DevPage* in : pages) {
            const int64_t n = in->rows;
            if (n == 0) continue;
            DevPage outp;
            outp.rows = n;
            auto channel = [&](int ch, const DevColumn** c) -> int {
                if (ch < 0 || ch >= (int)in->cols.size()) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "aggregation channel %d out of range", ch);
                *c = &in->cols[ch];
                return TGPU_OK;
            };
            for (int ch : spec_key_channels) {
                const DevColumn* c = nullptr;
                TG_TRY(channel(ch, &c));
                outp.cols.push_back(*c);                  // the block itself (page.getBlock(hashChannels[i]))
            }
            SkipSpec spec;
            memset(&spec, 0, sizeof(spec));
            std::vector<std::pair<size_t, std::shared_ptr<DevBuf>>> nullmaps;      // (output column, byte map)
            auto new_col = [&](int type, void** data) -> int {
                DevColumn c;
                c.type = type;
                c.length = n;
                c.own_data = std::make_shared<DevBuf>();
                TG_TRY(c.own_data->alloc(ctx, (size_t)n * (type == TGPU_INT128 ? 16 : 8)));
                c.data = c.own_data->p;
                *data = c.own_data->p;
                outp.cols.push_back(std::move(c));
                return TGPU_OK;
            };
            for (auto& f : fns) {
                if (from_state) {
                    // INTERMEDIATE: a one-row group's combined state is the incoming state
                    const DevColumn* c = nullptr;
                    TG_TRY(channel(f.input_channel, &c));
                    outp.cols.push_back(*c);
                    if (f.function == TGPU_AGG_AVG || f.function == TGPU_AGG_SUM_DECIMAL || f.function == TGPU_AGG_AVG_DECIMAL) {
                        TG_TRY(channel(f.input_channel + 1, &c));
                        outp.cols.push_back(*c);
                    }
                    if (f.function == TGPU_AGG_AVG_DECIMAL) {
                        TG_TRY(channel(f.input_channel + 2, &c));
                        outp.cols.push_back(*c);
                    }
                    continue;
                }
                if (spec.count >= SKIP_MAX_FNS) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "more than %d aggregates", SKIP_MAX_FNS);
                SkipFn& k = spec.f[spec.count++];
                k.function = f.function;
                k.in_ch = -1;
                k.mask_ch = -1;
                if (f.mask_channel >= 0) {
                    const DevColumn* m = nullptr;
                    TG_TRY(channel(f.mask_channel, &m));
                    k.mask_ch = f.mask_channel;
                }
                int in_type = TGPU_INT64;
                bool nullable = k.mask_ch >= 0;
                if (f.function != TGPU_AGG_COUNT_STAR) {
                    const DevColumn* c = nullptr;
                    TG_TRY(channel(f.input_channel, &c));
                    if (c->type == TGPU_UTF8) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "aggregates over variable-width inputs are not supported");
                    if (c->type == TGPU_FLOAT32) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "aggregate function %d over a REAL channel: keep the Java accumulator", f.function);
                    if (c->type == TGPU_INT128 && f.function != TGPU_AGG_SUM_DECIMAL && f.function != TGPU_AGG_AVG_DECIMAL && f.function != TGPU_AGG_COUNT)
                        return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "aggregate function %d over a 128-bit channel (only count and the decimal sum are built)", f.function);
                    k.in_ch = f.input_channel;
                    in_type = c->type;
                    nullable |= c->validity != nullptr;
                }
                k.in_is_double = in_type == TGPU_FLOAT64;
                switch (f.function) {
                    case TGPU_AGG_COUNT_STAR: case TGPU_AGG_COUNT:
                        TG_TRY(new_col(TGPU_INT64, &k.out0));
                        break;
                    case TGPU_AGG_AVG:
                        TG_TRY(new_col(TGPU_INT64, &k.out0));
                        TG_TRY(new_col(TGPU_FLOAT64, &k.out1));
                        break;
                    case TGPU_AGG_SUM_DECIMAL: case TGPU_AGG_AVG_DECIMAL: {
                        // LongDecimalWithOverflow[AndLong]State of one row: (the value in 128 bits, overflow 0[, 1 row])
                        if (in_type != TGPU_INT64 && in_type != TGPU_INT128)
                            return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "a decimal sum reads BIGINT (short decimal) or INT128 channels, not type %d", in_type);
                        TG_TRY(new_col(TGPU_INT128, &k.out0));
                        auto nm = std::make_shared<DevBuf>();
                        TG_TRY(nm->alloc(ctx, (size_t)n));
                        k.null0 = nm->as<unsigned char>();
                        if (nullable) nullmaps.emplace_back(outp.cols.size() - 1, nm);
                        else nullmaps.emplace_back((size_t)-1, nm);
                        TG_TRY(new_col(TGPU_INT64, &k.out1));
                        if (f.function == TGPU_AGG_AVG_DECIMAL) TG_TRY(new_col(TGPU_INT64, &k.out2));
                        break;
                    }
                    case TGPU_AGG_SUM: case TGPU_AGG_MIN: case TGPU_AGG_MAX: {
                        TG_TRY(new_col(k.in_is_double ? TGPU_FLOAT64 : TGPU_INT64, &k.out0));
                        auto nm = std::make_shared<DevBuf>();
                        TG_TRY(nm->alloc(ctx, (size_t)n));
                        k.null0 = nm->as<unsigned char>();
                        // (an input without NULLs and without a mask cannot produce a NULL state: no bitmap then)
                        if (nullable) nullmaps.emplace_back(outp.cols.size() - 1, nm);
                        else nullmaps.emplace_back((size_t)-1, nm);
                        break;
                    }
                    default: return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "aggregate function %d", f.function);
                }
            }
            if (spec.count > 0) {
                DColumns cols;
                TG_TRY(fill_cols(*in, &cols));
                TG_LAUNCH(ctx, agg_skip_kernel, tg_grid(ctx, n, 256, 8), 256, 0, cols, n, spec);
                for (auto& nm : nullmaps) {
                    if (nm.first == (size_t)-1) continue;
                    auto bm = std::make_shared<DevBuf>();
                    TG_TRY(bm->alloc(ctx, (size_t)((n + 7) / 8)));
                    TG_LAUNCH(ctx, nullmap_pack_kernel, tg_grid(ctx, (n + 7) / 8, 256, 8), 256, 0, nm.second->as<unsigned char>(), n, bm->as<unsigned char>(),
                              (unsigned int*)nullptr);
                    outp.cols[nm.first].own_validity = bm;
                    outp.cols[nm.first].validity = bm->as<uint8_t>();
                }
                // the byte maps are read by kernels queued on the stream: keep them until those ran
                TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
            }
            pending.push_back(tg_make_owned_page(std::move(outp)));
        }
        if (next_out >= pending.size()) close_builder(-1);       // (a filter that drops the whole page leaves nothing to hand out)
        return TGPU_OK;
    }

    // HashAggregationOperator.closeAggregationBuilder :512-523
    void close_builder(int64_t unique_rows)
    {
        if (!builder_open) return;
        if (controller) tgpu_partial_agg_controller_on_flush(controller, builder_bytes, builder_rows, skip_mode ? -1 : unique_rows);
        builder_open = false;
        skip_mode = false;
        builder_bytes = builder_rows = builder_unique = 0;
    }

    int add_via_filter_project(const tgpu_page* page)
    {
        TG_TRY(inner_fp->add_input(page));
        while (true) {
            OwnedPage* o = nullptr;
            TG_TRY(inner_fp->get_output(&o));
            if (!o) break;
            std::unique_ptr<OwnedPage> guard(o);
            TG_TRY(prepare_wide(&o->page));
            TG_TRY(encode_string_keys(&o->page));       // (has_pre is false by now: the keys are the projection's output channels)
            DColumns cols;
            TG_TRY(fill_cols(o->page, &cols));
            TG_TRY(run_general(o->page, cols));
        }
        return after_page();
    }

    int after_page()
    {
        // InMemoryHashAggregationBuilder.updateIsFull :193-200 -> HashAggregationOperator.needsInput :346-355
        if (step == TGPU_STEP_PARTIAL && max_partial_bytes > 0 && memory_bytes() > max_partial_bytes) flushing = true;
        return TGPU_OK;
    }

    int64_t memory_bytes() override
    {
        int64_t A = plan.num_accs > 0 ? plan.num_accs : 1;
        int64_t b = group_count * (8 + 8 * A + 9 * (int64_t)plan.num_keys);
        if (use_general) b += (int64_t)g_table.bytes + (int64_t)f_recs.bytes;
        for (auto& d : key_dicts)
            if (d) b += d->memory_bytes();
        return planned ? b : 0;
    }

    int build_output(OwnedPage** out)
    {
        *out = nullptr;
        if (planned && fused_general) TG_TRY(gf_finalize());
        if (!planned || group_count == 0) return TGPU_OK;
        int64_t G = group_count;
        DevPage outp;
        outp.rows = G;
        unsigned int* d_err = (unsigned int*)(ctx->d_scratch + 10);
        unsigned int* d_any = d_err + 2;    // two words of per-column null flags
        TG_CUDA(ctx, cudaMemsetAsync(d_err, 0, 16, ctx->stream));
        int grid = tg_grid(ctx, G, 256, 8);
        std::vector<std::shared_ptr<DevBuf>> nullmaps;
        // key columns
        for (int k = 0; k < plan.num_keys; k++) {
            DevColumn c;
            c.type = key_types[k];
            c.length = G;
            c.own_data = std::make_shared<DevBuf>();
            TG_TRY(c.own_data->alloc(ctx, (size_t)G * c.elem_size()));
            c.data = c.own_data->p;
            auto nm = std::make_shared<DevBuf>();
            TG_TRY(nm->alloc(ctx, (size_t)G));
            TG_LAUNCH(ctx, agg_key_output_kernel, grid, 256, 0, st_keyvals.as<long long>() + (size_t)k * st_cap, st_keynull.as<unsigned char>() + (size_t)k * st_cap,
                      G, c.elem_size(), c.own_data->p, nm->as<unsigned char>());
            if (k < (int)key_dicts.size() && key_dicts[k]) {
                // the key column holds dictionary ids: give the strings back (FlatHash.appendTo reads them from its variable-width data)
                DevColumn text;
                TG_TRY(key_dicts[k]->decode((const int32_t*)c.own_data->p, nm->as<unsigned char>(), G, &text));
                c = std::move(text);
            }
            if (k < (int)key_real.size() && key_real[k]) {
                DevColumn real;
                real.type = TGPU_FLOAT32;
                real.length = G;
                real.own_data = std::make_shared<DevBuf>();
                TG_TRY(real.own_data->alloc(ctx, (size_t)G * 4));
                real.data = real.own_data->p;
                TG_LAUNCH(ctx, agg_narrow_real_kernel, grid, 256, 0, (const unsigned long long*)c.own_data->p, G, real.own_data->as<unsigned int>());
                c = std::move(real);
            }
            if (k > 0 && k - 1 < (int)wide_key_high.size() && wide_key_high[k - 1]) {
                // the low word of an INT128 key: weld it to the high word emitted just before (both carry the same NULL flags)
                DevColumn& high = outp.cols.back();
                DevColumn wide;
                wide.type = TGPU_INT128;
                wide.length = G;
                wide.own_data = std::make_shared<DevBuf>();
                TG_TRY(wide.own_data->alloc(ctx, (size_t)G * 16));
                wide.data = wide.own_data->p;
                TG_LAUNCH(ctx, agg_join_int128_kernel, grid, 256, 0, (const long long*)high.data, (const long long*)c.data, G, wide.own_data->as<long long>());
                high = std::move(wide);
                continue;
            }
            nullmaps.push_back(nm);
            outp.cols.push_back(std::move(c));
        }
        // aggregate columns
        OutSpec spec;
        memset(&spec, 0, sizeof(spec));
        bool partial_out = step == TGPU_STEP_PARTIAL || step == TGPU_STEP_INTERMEDIATE;
        bool from_state = step == TGPU_STEP_FINAL || step == TGPU_STEP_INTERMEDIATE;
        auto add_col = [&](int type, int kind, int a0, int a1, int a2 = -1, int a3 = -1, int a4 = -1) -> int {
            if (spec.count >= 48) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "too many output columns");
            DevColumn c;
            c.type = type;
            c.length = G;
            c.own_data = std::make_shared<DevBuf>();
            TG_TRY(c.own_data->alloc(ctx, (size_t)G * (type == TGPU_INT128 ? 16 : 8)));
            c.data = c.own_data->p;
            auto nm = std::make_shared<DevBuf>();
            TG_TRY(nm->alloc(ctx, (size_t)G));
            int k = spec.count++;
            spec.kind[k] = kind;
            spec.a0[k] = a0;
            spec.a1[k] = a1;
            spec.a2[k] = a2;
            spec.a3[k] = a3;
            spec.a4[k] = a4;
            spec.a5[k] = -1;
            spec.data[k] = c.own_data->p;
            spec.nullmap[k] = nm->as<unsigned char>();
            nullmaps.push_back(nm);
            outp.cols.push_back(std::move(c));
            return TGPU_OK;
        };
        for (size_t i = 0; i < fns.size(); i++) {
            const AggFnPlan& fp = fnplans[i];
            bool dbl = fp.in_elem_is_double;
            bool count_is_i128 = from_state;   // counts combined from state columns are 128-bit sums
            switch (fp.function) {
                case TGPU_AGG_COUNT_STAR: case TGPU_AGG_COUNT:
                    TG_TRY(add_col(TGPU_INT64, count_is_i128 ? 3 : 0, fp.acc_main, -1));
                    break;
                case TGPU_AGG_SUM:
                    TG_TRY(add_col(dbl ? TGPU_FLOAT64 : TGPU_INT64, dbl ? 1 : 3, fp.acc_main, fp.acc_count));
                    break;
                case TGPU_AGG_AVG:
                    if (partial_out) {
                        TG_TRY(add_col(TGPU_INT64, count_is_i128 ? 3 : 0, fp.acc_count, -1));
                        TG_TRY(add_col(TGPU_FLOAT64, 6, fp.acc_main, -1));
                    }
                    else TG_TRY(add_col(TGPU_FLOAT64, 2, fp.acc_main, fp.acc_count));
                    break;
                case TGPU_AGG_MIN: case TGPU_AGG_MAX:
                    TG_TRY(add_col(dbl ? TGPU_FLOAT64 : TGPU_INT64, dbl ? 4 : 5, fp.acc_main, fp.acc_count));
                    break;
                case TGPU_AGG_SUM_DECIMAL:
                    if (partial_out) {
                        TG_TRY(add_col(TGPU_INT128, 7, fp.acc_main, fp.acc_count, fp.acc2, fp.acc3, fp.acc4));
                        TG_TRY(add_col(TGPU_INT64, 8, fp.acc_main, fp.acc_count, fp.acc2, fp.acc3, fp.acc4));
                    }
                    else TG_TRY(add_col(TGPU_INT128, 9, fp.acc_main, fp.acc_count, fp.acc2, fp.acc3, fp.acc4));
                    break;
                case TGPU_AGG_AVG_DECIMAL:
                    if (partial_out) {
                        TG_TRY(add_col(TGPU_INT128, 7, fp.acc_main, fp.acc_count, fp.acc2, fp.acc3, fp.acc4));
                        TG_TRY(add_col(TGPU_INT64, 8, fp.acc_main, fp.acc_count, fp.acc2, fp.acc3, fp.acc4));
                        // the row counter: non-NULL inputs of a raw step, the summed counters of a state step
                        if (fp.acc5 >= 0) TG_TRY(add_col(TGPU_INT64, 3, fp.acc5, -1));
                        else TG_TRY(add_col(TGPU_INT64, 0, fp.acc_count, -1));
                    }
                    else {
                        const bool narrow = fp.result_type == TGPU_INT64;
                        TG_TRY(add_col(narrow ? TGPU_INT64 : TGPU_INT128, narrow ? 11 : 10, fp.acc_main, fp.acc_count, fp.acc2, fp.acc3, fp.acc4));
                        spec.a5[spec.count - 1] = fp.acc5;
                    }
                    break;
                default: break;
            }
        }
        if (spec.count > 0) TG_LAUNCH(ctx, agg_output_kernel, grid, 256, 0, state(), G, spec, d_err, d_any);
        // validity bitmaps only for columns that actually hold a NULL
        DevBuf anyflags;
        TG_TRY(anyflags.alloc(ctx, outp.cols.size() * 4));
        TG_CUDA(ctx, cudaMemsetAsync(anyflags.p, 0, outp.cols.size() * 4, ctx->stream));
        std::vector<std::shared_ptr<DevBuf>> bitmaps(outp.cols.size());
        for (size_t c = 0; c < outp.cols.size(); c++) {
            bitmaps[c] = std::make_shared<DevBuf>();
            TG_TRY(bitmaps[c]->alloc(ctx, (size_t)((G + 7) / 8)));
            TG_LAUNCH(ctx, nullmap_pack_kernel, tg_grid(ctx, (G + 7) / 8, 256, 8), 256, 0, nullmaps[c]->as<unsigned char>(), G,
                      bitmaps[c]->as<unsigned char>(), anyflags.as<unsigned int>() + c);
        }
        std::vector<unsigned int> h_any(outp.cols.size());
        TG_CUDA(ctx, cudaMemcpyAsync(h_any.data(), anyflags.p, outp.cols.size() * 4, cudaMemcpyDeviceToHost, ctx->stream));
        int64_t errw = 0;
        TG_TRY(tg_read_i64(ctx, d_err, &errw));
        TG_TRY(raise((uint32_t)(errw & 0xFFFFFFFFLL)));
        for (size_t c = 0; c < outp.cols.size(); c++) {
            if (!h_any[c]) continue;
            outp.cols[c].own_validity = bitmaps[c];
            outp.cols[c].validity = bitmaps[c]->as<uint8_t>();
        }
        *out = tg_make_owned_page(std::move(outp));
        return TGPU_OK;
    }

    int reset_state()
    {
        // partial flush: the builder is rebuilt empty (HashAggregationOperator.getOutput :478-483)
        planned = true;
        g_slots = 0;
        g_table.release();
        fused_general = false;
        f_recs.release();
        f_cap = f_used = f_specials = rows_seen = 0;
        TG_TRY(init_state());
        // once the pre-stage was un-fused (inner_fp exists, the plan's sources point at projection OUTPUT channels) the
        // shared-memory path must never see a raw input page again: stay on the general path across flushes
        if (inner_fp) use_general = true;
        if (use_general) TG_TRY(switch_to_general());
        return TGPU_OK;
    }

    // HashAggregationOperator.getGlobalAggregationOutput :537-567: no input row reached the operator and the plan has global grouping
    // sets - one row per set: the $group_id key holds the set's id, the other keys are NULL, every aggregate evaluates over nothing
    // (count -> 0, everything else -> NULL)
    int build_default_output(OwnedPage** out)
    {
        *out = nullptr;
        const int64_t G = (int64_t)global_group_ids.size();
        if (G == 0) return TGPU_OK;
        auto type_of = [&](int ch) -> int { return ch >= 0 && ch < (int)input_types.size() ? input_types[ch] : 0; };
        DevPage outp;
        outp.rows = G;
        auto all_null = std::make_shared<DevBuf>();
        TG_TRY(all_null->alloc(ctx, (size_t)((G + 7) / 8)));
        TG_CUDA(ctx, cudaMemsetAsync(all_null->p, 0, (size_t)((G + 7) / 8), ctx->stream));
        auto null_column = [&](int type, DevColumn* c) -> int {
            if (!type) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "global aggregation default rows need tgpu_agg_spec.input_channel_types");
            c->type = type;
            c->length = G;
            c->own_data = std::make_shared<DevBuf>();
            size_t bytes = (size_t)G * (type == TGPU_UTF8 ? 1 : type == TGPU_INT128 ? 16 : 8);
            TG_TRY(c->own_data->alloc(ctx, bytes));
            TG_CUDA(ctx, cudaMemsetAsync(c->own_data->p, 0, bytes, ctx->stream));
            c->data = c->own_data->p;
            if (type == TGPU_UTF8) {
                c->own_offsets = std::make_shared<DevBuf>();
                TG_TRY(c->own_offsets->alloc(ctx, (size_t)(G + 1) * 4));
                TG_CUDA(ctx, cudaMemsetAsync(c->own_offsets->p, 0, (size_t)(G + 1) * 4, ctx->stream));
                c->offsets = c->own_offsets->as<int32_t>();
            }
            c->own_validity = all_null;
            c->validity = all_null->as<uint8_t>();
            return TGPU_OK;
        };
        for (int k = 0; k < (int)key_channels.size(); k++) {
            DevColumn c;
            if (k == group_id_key) {
                std::vector<long long> ids(global_group_ids.begin(), global_group_ids.end());
                c.type = TGPU_INT64;
                c.length = G;
                c.own_data = std::make_shared<DevBuf>();
                TG_TRY(c.own_data->alloc(ctx, (size_t)G * 8));
                TG_CUDA(ctx, cudaMemcpyAsync(c.own_data->p, ids.data(), (size_t)G * 8, cudaMemcpyHostToDevice, ctx->stream));
                TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
                c.data = c.own_data->p;
            }
            else {
                int ch = key_channels[k];
                int type = has_pre ? (ch >= 0 && ch < (int)projections.size() && projections[ch].kind == 0 ? type_of(projections[ch].index) : 0) : type_of(ch);
                TG_TRY(null_column(type, &c));
            }
            outp.cols.push_back(std::move(c));
        }
        const bool from_state = step == TGPU_STEP_FINAL || step == TGPU_STEP_INTERMEDIATE;
        for (auto& f : fns) {
            DevColumn c;
            if (f.function == TGPU_AGG_COUNT_STAR || f.function == TGPU_AGG_COUNT) {
                TG_TRY(null_column(TGPU_INT64, &c));
                c.own_validity.reset();
                c.validity = nullptr;                   // count over nothing is 0, not NULL
            }
            else if (f.function == TGPU_AGG_AVG) TG_TRY(null_column(TGPU_FLOAT64, &c));
            else if (f.function == TGPU_AGG_SUM_DECIMAL) TG_TRY(null_column(TGPU_INT128, &c));
            else if (f.function == TGPU_AGG_AVG_DECIMAL) TG_TRY(null_column(f.reserved == TGPU_INT64 ? TGPU_INT64 : TGPU_INT128, &c));
            else {
                int ch = f.input_channel;
                int type = has_pre ? (ch >= 0 && ch < (int)projections.size() ? (projections[ch].kind == 0 ? type_of(projections[ch].index)
                                      : projections[ch].vtype == TGPU_V_DOUBLE ? TGPU_FLOAT64 : TGPU_INT64) : 0) : type_of(ch);
                (void)from_state;                        // FINAL: the state column of sum / min / max has the value's type
                if (type == TGPU_INT32 || type == TGPU_INT16 || type == TGPU_INT8) type = TGPU_INT64;   // sum / min / max of narrow integers come out as BIGINT here
                TG_TRY(null_column(type, &c));
            }
            outp.cols.push_back(std::move(c));
        }
        TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        *out = tg_make_owned_page(std::move(outp));
        return TGPU_OK;
    }

    int get_output(OwnedPage** out) override
    {
        *out = nullptr;
        if (next_out < pending.size()) {
            *out = pending[next_out++];
            if (next_out >= pending.size()) {
                pending.clear();
                next_out = 0;
                if (skip_mode) close_builder(-1);
            }
            return TGPU_OK;
        }
        if (flushing) {
            TG_TRY(build_output(out));
            if (*out) saw_group = true;
            close_builder(*out ? (*out)->page.rows : 0);
            TG_TRY(reset_state());
            flushing = false;
            return TGPU_OK;
        }
        if (finishing && !finished) {
            TG_TRY(build_output(out));
            close_builder(*out ? (*out)->page.rows : 0);
            finished = true;
            const bool output_partial = step == TGPU_STEP_PARTIAL || step == TGPU_STEP_INTERMEDIATE;
            // (a group exists iff a row reached the aggregation: with a fused filter that is "a row passed the filter", which is what the
            //  reference's totalInputRowsProcessed counts behind its separate FilterAndProjectOperator)
            if (!*out && !saw_group && !output_partial && !global_group_ids.empty()) TG_TRY(build_default_output(out));
        }
        return TGPU_OK;
    }

    int finish() override { finishing = true; return TGPU_OK; }
    bool is_finished() override { return finished && next_out >= pending.size(); }
};

int build_agg_op(tgpu_ctx* ctx, const tgpu_agg_spec* spec, AggOp** out)
{
    if (spec->num_keys < 0 || spec->num_aggs < 0) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "negative counts in aggregation spec");
    if (spec->step < TGPU_STEP_SINGLE || spec->step > TGPU_STEP_INTERMEDIATE) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "bad aggregation step");
    std::unique_ptr<AggOp> op(new AggOp(ctx));
    op->key_channels.assign(spec->key_channels, spec->key_channels + spec->num_keys);
    op->spec_key_channels = op->key_channels;
    op->fns.assign(spec->aggs, spec->aggs + spec->num_aggs);
    op->step = spec->step;
    op->expected_groups = spec->expected_groups;
    op->max_partial_bytes = spec->max_partial_bytes;
    if (spec->partial_aggregation_controller) {
        if (spec->step != TGPU_STEP_PARTIAL && spec->step != TGPU_STEP_INTERMEDIATE)
            return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "partialAggregationController should be present only for partial aggregation");
        op->controller = spec->partial_aggregation_controller;
    }
    if (spec->num_global_group_ids > 0) {
        if (!spec->global_group_ids || spec->group_id_key < 0 || spec->group_id_key >= spec->num_keys)
            return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "global grouping sets need global_group_ids and a valid group_id_key");
        op->global_group_ids.assign(spec->global_group_ids, spec->global_group_ids + spec->num_global_group_ids);
        op->group_id_key = spec->group_id_key;
    }
    if (spec->num_input_channels > 0 && spec->input_channel_types)
        op->input_types.assign(spec->input_channel_types, spec->input_channel_types + spec->num_input_channels);
    if (spec->pre) {
        if (spec->step == TGPU_STEP_FINAL || spec->step == TGPU_STEP_INTERMEDIATE)
            return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "a fused pre-stage only makes sense on raw input");
        op->has_pre = true;
        TG_TRY(tg::expr_compile(ctx, spec->pre, &op->host_prog, &op->prog_max_channel));
        op->projections.assign(spec->pre->projections, spec->pre->projections + spec->pre->num_projections);
        op->pre_insns.assign(spec->pre->insns, spec->pre->insns + spec->pre->num_insns);
        for (int i = 0; i < spec->pre->num_in_lists; i++)
            op->pre_in_values.emplace_back(spec->pre->in_lists[i].values, spec->pre->in_lists[i].values + spec->pre->in_lists[i].count);
        op->pre_filter_temp = spec->pre->filter_temp;
        op->pre_num_filter_insns = spec->pre->num_filter_insns;
        TG_TRY(op->d_prog.alloc(ctx, sizeof(DProgram)));
        TG_CUDA(ctx, cudaMemcpyAsync(op->d_prog.p, &op->host_prog, sizeof(DProgram), cudaMemcpyHostToDevice, ctx->stream));
        TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    *out = op.release();
    return TGPU_OK;
}

}  // namespace

extern "C" int tgpu_agg_create(tgpu_ctx* ctx, const tgpu_agg_spec* spec, tgpu_op** out)
{
    if (!ctx || !spec || !out) return TGPU_ERR_INVALID_ARGUMENT;
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    AggOp* op = nullptr;
    TG_TRY(build_agg_op(ctx, spec, &op));
    *out = op;
    return TGPU_OK;
}

extern "C" int tgpu_partial_agg_controller_create(int64_t max_partial_memory_bytes, double unique_rows_ratio_threshold, tgpu_partial_agg_controller** out)
{
    if (!out || max_partial_memory_bytes < 0) return TGPU_ERR_INVALID_ARGUMENT;
    auto* c = new tgpu_partial_agg_controller();
    c->max_partial_bytes = max_partial_memory_bytes;
    c->threshold = unique_rows_ratio_threshold;
    *out = c;
    return TGPU_OK;
}

extern "C" void tgpu_partial_agg_controller_destroy(tgpu_partial_agg_controller* controller) { delete controller; }

extern "C" int tgpu_partial_agg_controller_is_disabled(const tgpu_partial_agg_controller* controller)
{
    return controller && controller->disabled.load(std::memory_order_acquire) ? 1 : 0;
}

// PartialAggregationController.onFlush :67-91, shouldDisablePartialAggregation :93-97
extern "C" void tgpu_partial_agg_controller_on_flush(tgpu_partial_agg_controller* c, int64_t bytes_processed, int64_t rows_processed, int64_t unique_rows_produced)
{
    if (!c) return;
    std::lock_guard<std::mutex> lock(c->mu);
    bool disabled = c->disabled.load(std::memory_order_relaxed);
    const bool has_unique = unique_rows_produced >= 0;
    if (!disabled && !has_unique) return;                 // when PA is re-enabled, stats from disabled flushes are ignored
    c->total_bytes += bytes_processed;
    c->total_rows += rows_processed;
    if (has_unique) c->total_unique += unique_rows_produced;
    const double disable_factor = 1.5, enable_factor = 1.5 * 200;
    if (!disabled && (double)c->total_bytes >= (double)c->max_partial_bytes * disable_factor
        && ((double)c->total_unique / (double)c->total_rows) > c->threshold)
        disabled = true;
    if (disabled && (double)c->total_bytes >= (double)c->max_partial_bytes * enable_factor) {
        c->total_bytes = c->total_rows = c->total_unique = 0;
        disabled = false;
    }
    c->disabled.store(disabled, std::memory_order_release);
}

extern "C" int tgpu_agg_rows_with_partial_aggregation_disabled(tgpu_op* op, int64_t* out)
{
    AggOp* a = dynamic_cast<AggOp*>(op);
    if (!a || !out) return TGPU_ERR_INVALID_ARGUMENT;
    *out = a->rows_skipped;
    return TGPU_OK;
}

extern "C" int tgpu_agg_group_count(tgpu_op* op, int64_t* out)
{
    AggOp* a = dynamic_cast<AggOp*>(op);
    if (!a || !out) return TGPU_ERR_INVALID_ARGUMENT;
    *out = a->group_count;
    return TGPU_OK;
}

extern "C" int tgpu_groupby_hash_create(tgpu_ctx* ctx, int32_t num_keys, const int32_t* key_channels, int64_t expected_groups, tgpu_op** out)
{
    if (!ctx || !key_channels || !out) return TGPU_ERR_INVALID_ARGUMENT;
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    tgpu_agg_spec spec;
    memset(&spec, 0, sizeof(spec));
    spec.num_keys = num_keys;
    spec.key_channels = key_channels;
    spec.step = TGPU_STEP_SINGLE;
    spec.expected_groups = expected_groups;
    AggOp* op = nullptr;
    TG_TRY(build_agg_op(ctx, &spec, &op));
    op->gids_only = true;
    *out = op;
    return TGPU_OK;
}

extern "C" int tgpu_groupby_hash_get_group_ids(tgpu_op* op, const tgpu_page* page, int32_t* out_group_ids)
{
    AggOp* a = dynamic_cast<AggOp*>(op);
    if (!a || !page || !out_group_ids) return TGPU_ERR_INVALID_ARGUMENT;
    tgpu_ctx* ctx = a->ctx;
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    if (page->num_rows == 0) return TGPU_OK;
    DevPage in;
    TG_TRY(tg_ingest_page(ctx, page, &in));
    TG_TRY(a->prepare_wide(&in));
    TG_TRY(a->encode_string_keys(&in));
    if (!a->planned) {
        TG_TRY(a->make_plan(in));
        TG_TRY(a->init_state());
        TG_TRY(a->switch_to_general());
    }
    DColumns cols;
    TG_TRY(a->fill_cols(in, &cols));
    bool device = (page->flags & TGPU_PAGE_DEVICE) != 0;
    if (device) return a->run_general_ids(in, cols, out_group_ids);
    DevBuf gids;
    TG_TRY(gids.alloc(ctx, (size_t)in.rows * 4));
    TG_TRY(a->run_general_ids(in, cols, gids.as<int>()));
    TG_CUDA(ctx, cudaMemcpyAsync(out_group_ids, gids.p, (size_t)in.rows * 4, cudaMemcpyDeviceToHost, ctx->stream));
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return TGPU_OK;
}

// test hook (no GPU needed): generate + NVRTC-compile the specialised small-group kernel for a spec whose input
// channels have the given tgpu_types; returns the cubin size in *cubin_bytes and the generated source length
extern "C" int tgpu_jit_selftest_agg(const tgpu_agg_spec* spec, const int32_t* channel_types, int32_t num_channels, uint32_t nullable_mask, int64_t* cubin_bytes, char* source_out, int64_t source_cap)
{
    if (!spec || !channel_types || !cubin_bytes) return TGPU_ERR_INVALID_ARGUMENT;
    tgpu_ctx fake;
    AggOp* op = nullptr;
    {
        // build_agg_op touches the device only when a pre-program has to be uploaded: mimic it on the host
        std::unique_ptr<AggOp> o(new AggOp(&fake));
        o->key_channels.assign(spec->key_channels, spec->key_channels + spec->num_keys);
        o->fns.assign(spec->aggs, spec->aggs + spec->num_aggs);
        o->step = spec->step;
        if (spec->pre) {
            o->has_pre = true;
            int st = tg::expr_compile(&fake, spec->pre, &o->host_prog, &o->prog_max_channel);
            if (st != TGPU_OK) return st;
            o->projections.assign(spec->pre->projections, spec->pre->projections + spec->pre->num_projections);
        }
        op = o.release();
    }
    std::unique_ptr<AggOp> guard(op);
    DevPage in;
    in.rows = 0;
    in.cols.resize(num_channels);
    int elems[TGPU_MAX_CHANNELS] = {0};
    for (int c = 0; c < num_channels && c < TGPU_MAX_CHANNELS; c++) in.cols[c].type = channel_types[c];
    op->key_dicts.resize(op->key_channels.size());
    for (size_t k = 0; k < op->key_channels.size(); k++) {
        int ch = op->key_input_channel((int)k);
        if (ch >= 0 && ch < num_channels && in.cols[ch].type == TGPU_UTF8) {     // variable-width key: the kernel sees its INT32 dictionary ids
            op->key_dicts[k] = std::make_shared<StringDict>(&fake);
            in.cols[ch].type = TGPU_INT32;
        }
    }
    for (int c = 0; c < num_channels && c < TGPU_MAX_CHANNELS; c++) elems[c] = in.cols[c].elem_size();
    int st = op->make_plan(in);
    if (st != TGPU_OK) return st;
    AccMap map;
    // (TGPU_JIT_SELFTEST_VEC: the variant with the four-consecutive-rows loader, as launched for 16-byte aligned columns)
    std::string src = gen_agg_small_source(op->plan, op->has_pre ? &op->host_prog : nullptr, elems, num_channels, 4, 2, nullable_mask, &map,
                                           getenv("TGPU_JIT_SELFTEST_VEC") != nullptr);
    if (source_out && source_cap > 0) { strncpy(source_out, src.c_str(), (size_t)source_cap - 1); source_out[source_cap - 1] = 0; }
    std::string cubin;
    st = tg::jit_compile_cubin(&fake, src, &cubin);
    if (st != TGPU_OK) { if (source_out && source_cap > 0) { strncpy(source_out, fake.err.c_str(), (size_t)source_cap - 1); source_out[source_cap - 1] = 0; } return st; }
    *cubin_bytes = (int64_t)cubin.size();
    return TGPU_OK;
}
