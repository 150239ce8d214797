// device_lib.cuh — device-side building blocks shared by the ahead-of-time kernels (nvcc) and the kernels
// specialised at run time with NVRTC (jit.cu embeds this file verbatim as the prelude of every generated
// translation unit).  It therefore includes NOTHING and defines its own fixed-width integer names under NVRTC.
//
// Contents: column refs, validity/loads, the reference's hash mixers, the per-operation semantics of the
// expression evaluator (one function, folded at compile time when op/type are constants), accumulator
// arithmetic, and the body of the small-group fused aggregation kernel as a template over a row program.
#ifndef TG_DEVICE_LIB_CUH
#define TG_DEVICE_LIB_CUH

#ifdef __CUDACC_RTC__
typedef signed char int8_t;
typedef short int16_t;
typedef int int32_t;
typedef long long int64_t;
typedef unsigned char uint8_t;
typedef unsigned short uint16_t;
typedef unsigned int uint32_t;
typedef unsigned long long uint64_t;
#define LLONG_MIN (-9223372036854775807LL - 1)
#endif

#define TGD_MAX_CHANNELS 32

// compact POD view of a fixed-width column
struct ColRef {
    const void* data;
    const uint8_t* validity;   // Arrow bitmap or null
    int32_t type;
    int32_t elem;
};

struct DColumns {
    ColRef cols[TGD_MAX_CHANNELS];
};

// expression opcodes / value types / operand kinds: numerically identical to include/trino_gpu.h
enum {
    TGD_EX_MOV = 0, TGD_EX_ADD = 1, TGD_EX_SUB = 2, TGD_EX_MUL = 3, TGD_EX_DIV = 4, TGD_EX_MOD = 5, TGD_EX_NEG = 6,
    TGD_EX_EQ = 10, TGD_EX_NE = 11, TGD_EX_LT = 12, TGD_EX_LE = 13, TGD_EX_GT = 14, TGD_EX_GE = 15,
    TGD_EX_AND = 20, TGD_EX_OR = 21, TGD_EX_NOT = 22, TGD_EX_IS_NULL = 23, TGD_EX_IS_NOT_NULL = 24, TGD_EX_BETWEEN = 25,
    TGD_EX_CAST_BIGINT_TO_DOUBLE = 30, TGD_EX_CAST_DOUBLE_TO_BIGINT = 31, TGD_EX_IN = 40
};
enum { TGD_V_BIGINT = 0, TGD_V_DOUBLE = 1, TGD_V_BOOLEAN = 2 };
enum { TG_ERR_BIT_OVERFLOW = 1, TG_ERR_BIT_DIV_ZERO = 2 };

enum AccKind {
    ACC_ROWS = 0, ACC_NONNULL = 1, ACC_SUM_F64 = 2, ACC_SUM_I64_LO = 3, ACC_SUM_I64_HI = 4,
    ACC_MIN_F64 = 5, ACC_MAX_F64 = 6, ACC_MIN_I64 = 7, ACC_MAX_I64 = 8, ACC_SUM_F64_FROM_I64 = 9
};

#define TGD_EMPTY_KEY 0x8000000000000000ULL
#define TGD_NO_ROW 0x7FFFFFFFFFFFFFFFLL
#define TGD_S_THREADS 256

// per-CTA partial results of the small-group aggregation kernel
struct SmallOut {
    unsigned long long* blk_keys;    // [grid][L]
    long long* blk_first;            // [grid][L+2]
    unsigned long long* blk_acc;     // [grid][L+2][A]
    int* overflow;
    unsigned int* err;
};

// computed projection outputs of the filter/project kernels
struct OutCols {
    int32_t count;
    int32_t temp[TGD_MAX_CHANNELS];
    int32_t vtype[TGD_MAX_CHANNELS];
    void* data[TGD_MAX_CHANNELS];
    uint8_t* nullmap[TGD_MAX_CHANNELS];   // 1 byte per row, 1 = NULL
    // pass-through projections copied by the fused (chunked) projection kernel; nullmap == nullptr: the input has no NULLs
    int32_t pass_count;
    void* pass_data[TGD_MAX_CHANNELS];
    uint8_t* pass_nullmap[TGD_MAX_CHANNELS];
};

#if defined(__CUDACC__)

__device__ __forceinline__ bool tg_valid(const uint8_t* validity, int64_t i)
{
    return validity == nullptr || ((validity[i >> 3] >> (i & 7)) & 1);
}

// sign-extending load of any fixed-width integer column element / raw bits of FLOAT64
__device__ __forceinline__ int64_t tg_load_i64(const ColRef& c, int64_t i)
{
    switch (c.elem) {
        case 8: return ((const int64_t*)c.data)[i];
        case 4: return ((const int32_t*)c.data)[i];
        case 2: return ((const int16_t*)c.data)[i];
        default: return ((const int8_t*)c.data)[i];
    }
}

template <int ELEM>
__device__ __forceinline__ int64_t tg_load_elem(const void* data, int64_t i)
{
    if (ELEM == 8) return ((const int64_t*)data)[i];
    if (ELEM == 4) return ((const int32_t*)data)[i];
    if (ELEM == 2) return ((const int16_t*)data)[i];
    return ((const int8_t*)data)[i];
}

__device__ __forceinline__ uint64_t tgd_murmur3_mix(uint64_t x)
{
    x ^= x >> 33; x *= 0xff51afd7ed558ccdULL; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ULL; x ^= x >> 33;
    return x;
}

// ---- expression semantics ---------------------------------------------------------------------------
struct Value {
    int64_t bits;
    bool is_null;
};

__device__ __forceinline__ bool vm_cmp(int op, int vtype, int64_t a, int64_t b)
{
    if (vtype == TGD_V_DOUBLE) {
        double x = __longlong_as_double(a), y = __longlong_as_double(b);
        switch (op) {
            case TGD_EX_EQ: return x == y;
            case TGD_EX_NE: return !(x == y);
            case TGD_EX_LT: return x < y;
            case TGD_EX_LE: return x <= y;
            case TGD_EX_GT: return x > y;
            default: return x >= y;
        }
    }
    switch (op) {
        case TGD_EX_EQ: return a == b;
        case TGD_EX_NE: return a != b;
        case TGD_EX_LT: return a < b;
        case TGD_EX_LE: return a <= b;
        case TGD_EX_GT: return a > b;
        default: return a >= b;
    }
}

// One operation of the evaluator (everything except IN, whose constant list lives with the caller).
// SQL three-valued logic; checked BIGINT arithmetic (Math.*Exact); IEEE DOUBLE arithmetic through the
// *_rn intrinsics, which are never contracted into FMAs.
__device__ __forceinline__ Value vm_apply(int op, int vtype, Value a, Value b, Value c, uint32_t* err)
{
    Value res;
    int64_t r = 0;
    bool rn = false;
    const bool dbl = vtype == TGD_V_DOUBLE;
    switch (op) {
        case TGD_EX_MOV: r = a.bits; rn = a.is_null; break;
        case TGD_EX_ADD: case TGD_EX_SUB: case TGD_EX_MUL: case TGD_EX_DIV: case TGD_EX_MOD: {
            rn = a.is_null || b.is_null;
            if (rn) break;
            if (dbl) {
                double x = __longlong_as_double(a.bits), y = __longlong_as_double(b.bits), z;
                if (op == TGD_EX_ADD) z = __dadd_rn(x, y);
                else if (op == TGD_EX_SUB) z = __dsub_rn(x, y);
                else if (op == TGD_EX_MUL) z = __dmul_rn(x, y);
                else if (op == TGD_EX_DIV) z = __ddiv_rn(x, y);
                else z = fmod(x, y);
                r = __double_as_longlong(z);
            }
            else {
                long long x = a.bits, y = b.bits, z = 0;
                if (op == TGD_EX_ADD) {
                    z = (long long)((unsigned long long)x + (unsigned long long)y);
                    if (((x ^ z) & (y ^ z)) < 0) *err |= TG_ERR_BIT_OVERFLOW;
                }
                else if (op == TGD_EX_SUB) {
                    z = (long long)((unsigned long long)x - (unsigned long long)y);
                    if (((x ^ y) & (x ^ z)) < 0) *err |= TG_ERR_BIT_OVERFLOW;
                }
                else if (op == TGD_EX_MUL) {
                    z = (long long)((unsigned long long)x * (unsigned long long)y);
                    long long hi = __mul64hi(x, y);
                    if (hi != (z >> 63)) *err |= TG_ERR_BIT_OVERFLOW;
                }
                else {
                    if (y == 0) { *err |= TG_ERR_BIT_DIV_ZERO; }
                    else if (y == -1) {
                        if (op == TGD_EX_DIV) {
                            if (x == LLONG_MIN) *err |= TG_ERR_BIT_OVERFLOW;
                            else z = -x;
                        }
                        else z = 0;
                    }
                    else z = op == TGD_EX_DIV ? x / y : x % y;
                }
                r = z;
            }
            break;
        }
        case TGD_EX_NEG:
            rn = a.is_null;
            if (rn) break;
            if (dbl) r = a.bits ^ (long long)0x8000000000000000ULL;
            else {
                if (a.bits == LLONG_MIN) *err |= TG_ERR_BIT_OVERFLOW;
                r = (long long)(0ULL - (unsigned long long)a.bits);
            }
            break;
        case TGD_EX_EQ: case TGD_EX_NE: case TGD_EX_LT: case TGD_EX_LE: case TGD_EX_GT: case TGD_EX_GE:
            rn = a.is_null || b.is_null;
            if (!rn) r = vm_cmp(op, vtype, a.bits, b.bits) ? 1 : 0;
            break;
        case TGD_EX_AND: {
            bool af = !a.is_null && a.bits == 0, bf = !b.is_null && b.bits == 0;
            if (af || bf) { r = 0; rn = false; }
            else if (a.is_null || b.is_null) rn = true;
            else r = 1;
            break;
        }
        case TGD_EX_OR: {
            bool at = !a.is_null && a.bits != 0, bt = !b.is_null && b.bits != 0;
            if (at || bt) { r = 1; rn = false; }
            else if (a.is_null || b.is_null) rn = true;
            else r = 0;
            break;
        }
        case TGD_EX_NOT: rn = a.is_null; r = a.bits == 0 ? 1 : 0; break;
        case TGD_EX_IS_NULL: r = a.is_null ? 1 : 0; break;
        case TGD_EX_IS_NOT_NULL: r = a.is_null ? 0 : 1; break;
        case TGD_EX_BETWEEN: {
            // value BETWEEN min AND max  ==  value >= min AND value <= max (Kleene AND)
            bool n1 = a.is_null || b.is_null, n2 = a.is_null || c.is_null;
            bool v1 = !n1 && vm_cmp(TGD_EX_GE, vtype, a.bits, b.bits);
            bool v2 = !n2 && vm_cmp(TGD_EX_LE, vtype, a.bits, c.bits);
            bool f1 = !n1 && !v1, f2 = !n2 && !v2;
            if (f1 || f2) r = 0;
            else if (n1 || n2) rn = true;
            else r = 1;
            break;
        }
        case TGD_EX_CAST_BIGINT_TO_DOUBLE:
            rn = a.is_null;
            r = __double_as_longlong((double)a.bits);
            break;
        case TGD_EX_CAST_DOUBLE_TO_BIGINT: {
            rn = a.is_null;
            if (rn) break;
            double x = __longlong_as_double(a.bits);
            // DoubleMath.roundToLong(x, HALF_UP): NaN / out of range is an error
            if (!(x >= -9.2233720368547758e18 && x < 9.2233720368547758e18)) *err |= TG_ERR_BIT_OVERFLOW;
            else r = llround(x);
            break;
        }
        default: break;
    }
    res.bits = r;
    res.is_null = rn;
    return res;
}

// ---- accumulators -------------------------------------------------------------------------------------
// order-preserving encodings so MIN/MAX are plain integer min/max.  min(DOUBLE) compares with COMPARISON_UNORDERED_LAST
// (NaN is the largest value, S/type/DoubleType.java:231-235), max(DOUBLE) with COMPARISON_UNORDERED_FIRST (NaN is the
// smallest, :237-252; M/operator/aggregation/MaxAggregationFunction.java:49): max({1.0, NaN}) = 1.0, max({NaN}) = NaN.
__host__ __device__ __forceinline__ unsigned long long f64_order_key(long long bits)
{
    unsigned long long u = (unsigned long long)bits;
    if ((u & 0x7FFFFFFFFFFFFFFFULL) > 0x7FF0000000000000ULL) u = 0x7FF8000000000000ULL;
    return (u >> 63) ? ~u : (u | 0x8000000000000000ULL);
}
// key for MAX: NaN ranks below every other value (key 1: above the "no row yet" initial 0, below -Infinity's key)
__host__ __device__ __forceinline__ unsigned long long f64_order_key_max(long long bits)
{
    unsigned long long u = (unsigned long long)bits;
    if ((u & 0x7FFFFFFFFFFFFFFFULL) > 0x7FF0000000000000ULL) return 1ULL;
    return (u >> 63) ? ~u : (u | 0x8000000000000000ULL);
}
__host__ __device__ __forceinline__ long long f64_from_order_key(unsigned long long k)
{
    if (k == 1ULL) return 0x7FF8000000000000LL;      // MAX's NaN (never produced by f64_order_key)
    return (long long)((k >> 63) ? (k & 0x7FFFFFFFFFFFFFFFULL) : ~k);
}
__host__ __device__ __forceinline__ unsigned long long i64_order_key(long long v) { return (unsigned long long)v ^ 0x8000000000000000ULL; }

__host__ __device__ __forceinline__ unsigned long long acc_init(int kind)
{
    return (kind == ACC_MIN_F64 || kind == ACC_MIN_I64) ? 0xFFFFFFFFFFFFFFFFULL : 0ULL;
}

__device__ __forceinline__ unsigned long long acc_combine(int kind, unsigned long long a, unsigned long long b)
{
    switch (kind) {
        case ACC_SUM_F64: case ACC_SUM_F64_FROM_I64:
            return (unsigned long long)__double_as_longlong(__dadd_rn(__longlong_as_double((long long)a), __longlong_as_double((long long)b)));
        case ACC_MIN_F64: case ACC_MIN_I64: return a < b ? a : b;
        case ACC_MAX_F64: case ACC_MAX_I64: return a > b ? a : b;
        default: return a + b;   // counts and the two halves of the 128-bit integer sum (carry handled by caller)
    }
}

// one accumulator update by one row on a thread-private accumulator word; `hi_off` = distance to the HI half
__device__ __forceinline__ void acc_update_private(int kind, unsigned long long* p, long long hi_off, long long bits)
{
    switch (kind) {
        case ACC_ROWS: case ACC_NONNULL: *p += 1; break;
        case ACC_SUM_F64: *p = (unsigned long long)__double_as_longlong(__dadd_rn(__longlong_as_double((long long)*p), __longlong_as_double(bits))); break;
        case ACC_SUM_F64_FROM_I64: *p = (unsigned long long)__double_as_longlong(__dadd_rn(__longlong_as_double((long long)*p), (double)bits)); break;
        case ACC_SUM_I64_LO: {
            unsigned long long old = *p, add = (unsigned long long)bits, nw = old + add;
            *p = nw;
            p[hi_off] += (unsigned long long)((bits < 0 ? -1LL : 0LL) + (nw < old ? 1LL : 0LL));
            break;
        }
        case ACC_MIN_F64: { unsigned long long k = f64_order_key(bits); if (k < *p) *p = k; break; }
        case ACC_MAX_F64: { unsigned long long k = f64_order_key_max(bits); if (k > *p) *p = k; break; }
        case ACC_MIN_I64: { unsigned long long k = i64_order_key(bits); if (k < *p) *p = k; break; }
        case ACC_MAX_I64: { unsigned long long k = i64_order_key(bits); if (k > *p) *p = k; break; }
        default: break;
    }
}

// ---- small-group fused aggregation: kernel body as a template over a row program ------------------------
// A row program P provides
//   static constexpr int L (key slots per CTA, power of two), A (accumulator words per group), R (rows per thread
//   in flight per loop trip)
//   struct P::Regs                      raw column values of one row
//   __device__ static int acc_kind(int a)
//   __device__ void load(cols, row, Regs&)                 all global loads of a row, nothing else
//   __device__ bool row(const Regs&, &key, &special, &err) filter + projections + key packing; false = row rejected;
//        `special` = 0 (NULL key) / 1 (key equal to the EMPTY sentinel) / -1
//   __device__ void accumulate(acc_ptr /* &acc[(slot*A)*T + tid] */, T)   applies every accumulator for that row
// The loads of R rows are issued back to back before the first row is consumed (memory-level parallelism), then the
// rows are folded one by one into the thread-private accumulators.
// Shared memory: tkeys[L] | lfirst[L+2] | acc[(L+2)*A*T].
template <class P>
__device__ __forceinline__ void agg_small_body(P& prog, const DColumns& cols, int64_t n, SmallOut out, unsigned long long* smem_u64)
{
    constexpr int L = P::L, A = P::A, T = TGD_S_THREADS;
    unsigned long long* tkeys = smem_u64;
    long long* lfirst = (long long*)(tkeys + L);
    unsigned long long* acc = (unsigned long long*)(lfirst + L + 2);
    const int tid = threadIdx.x;

    for (int i = tid; i < L; i += T) tkeys[i] = TGD_EMPTY_KEY;
    for (int i = tid; i < L + 2; i += T) lfirst[i] = TGD_NO_ROW;
    // the two special groups (NULL key, sentinel-valued key) exist for single-key plans only: a packed multi-column key never takes them,
    // and without their accumulator sets a CTA needs a third less shared memory (Q1: 73.8 -> 49.2 KB, 4 CTAs per SM instead of 3)
    constexpr int SETS = P::SPECIALS ? L + 2 : L;
    for (int s = 0; s < SETS; s++)
        for (int a = 0; a < A; a++) acc[((size_t)s * A + a) * T + tid] = acc_init(P::acc_kind(a));
    __shared__ int s_overflow;
    if (tid == 0) s_overflow = 0;
    __syncthreads();

    unsigned long long seen = 0;
    uint32_t err = 0;
    constexpr int R = P::R;
    const int64_t stride = (int64_t)gridDim.x * T;
    bool stop = false;
    // VEC: a thread owns R = 4 CONSECUTIVE rows per trip (16-byte loads, a warp reads 128 consecutive rows of every column);
    // otherwise its R rows are a grid stride apart.  Either way the rows of one thread ascend.
    static_assert(!P::VEC || R == 4, "the vector loader handles four rows");
    const int64_t first = P::VEC ? ((int64_t)blockIdx.x * T + tid) * R : (int64_t)blockIdx.x * T + tid;
    const int64_t row_step = P::VEC ? 1 : stride;
    for (int64_t base = first; base < n && !stop; base += stride * R) {
        if (*((volatile int*)&s_overflow)) break;   // some thread of this CTA ran out of key slots: the pass is void
        typename P::Regs regs[R];
        if (P::VEC && base + R <= n) prog.load4(cols, base, regs);
        else {
#pragma unroll
            for (int j = 0; j < R; j++) {
                int64_t row = base + (int64_t)j * row_step;
                if (row < n) prog.load(cols, row, regs[j]);
            }
        }
#pragma unroll
        for (int j = 0; j < R; j++) {
            int64_t row = base + (int64_t)j * row_step;
            if (row >= n || stop) continue;
            unsigned long long pk = 0;
            int special = -1;
            if (!prog.row(regs[j], &pk, &special, &err)) continue;
            int slot;
            if (special >= 0) slot = L + special;
            else {
                int h = (int)(tgd_murmur3_mix(pk) & (unsigned long long)(L - 1));
                slot = -1;
                for (int probe = 0; probe < L; probe++) {
                    unsigned long long cur = tkeys[h];
                    if (cur == TGD_EMPTY_KEY) cur = atomicCAS(&tkeys[h], TGD_EMPTY_KEY, pk);
                    if (cur == TGD_EMPTY_KEY || cur == pk) { slot = h; break; }
                    h = (h + 1) & (L - 1);
                }
                if (slot < 0) { s_overflow = 1; stop = true; continue; }   // more distinct keys in this CTA than L: host switches to path G
            }
            if (!((seen >> slot) & 1)) {
                seen |= 1ULL << slot;
                atomicMin(&lfirst[slot], (long long)row);   // rows of one thread ascend: its first hit is its minimum
            }
            prog.accumulate(&acc[((size_t)slot * A) * T + tid], T);
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
        int kind = P::acc_kind(a);
        if (kind == ACC_SUM_I64_HI) continue;   // reduced together with its LO half
        if (lfirst[s] == TGD_NO_ROW) continue;
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

// ---- general group-by, fused single pass (path G): kernel body as a template over the same row program ---------------------
// One AoS record per table slot: {key, first-row stamp, accumulator words ...} (W 8-byte words).  A row finds or claims its key's
// record, lowers the stamp and applies its accumulators with fire-and-forget reductions.  R rows are in flight per thread: all column
// loads of the R rows first, then the R record heads (independent random reads), then the resolves.  Claims are budgeted through
// TGD_TICKET_WAYS counters (tickets[way]; a way is picked by the lane) so that a page of mostly new keys does not serialise on one
// L2 address; a row that finds its way's budget exhausted goes to the deferred list and is replayed after the table has grown.
// tickets layout: [0, WAYS) claims per way, [WAYS] deferred rows, [WAYS + 1] special groups born.
// P supplies, besides load() / row(): accumulate_global(unsigned long long* acc) - reductions on the record's accumulator words.
#define TGD_TICKET_WAYS 64
#define TGD_G_ROWS 2      // rows in flight per thread with __launch_bounds__(256, 4)

// {a, b} = the two 64-bit words at p (16-byte aligned) in one L2 transaction, never served from the L1
__device__ __forceinline__ void tgd_ld_pair(const unsigned long long* p, unsigned long long& a, unsigned long long& b)
{
    asm volatile("ld.volatile.global.v2.u64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "l"(p) : "memory");
}

template <class P>
__device__ __forceinline__ void agg_general_body(P& prog, const DColumns& cols, long long n, const int* __restrict__ rows, long long first,
                                                 const int* __restrict__ stamp_rows, long long page_base, unsigned long long* __restrict__ recs, long long cap, int W,
                                                 int* __restrict__ tickets, int budget_per_way, int* __restrict__ deferred, unsigned int* __restrict__ err_out)
{
    constexpr int R = P::GR;          // rows in flight per thread (TGD_G_ROWS unless the generator says otherwise)
    const unsigned long long mask = (unsigned long long)cap - 1;
    const int way = ((threadIdx.x >> 5) + blockIdx.x * 8) & (TGD_TICKET_WAYS - 1);      // one ticket word per warp at a time
    const int lane = threadIdx.x & 31;
    unsigned int err = 0;
    int have = 0;                                                     // tickets in hand (the same number in every lane)
    const int batch = budget_per_way >= (32 << 8) ? 32 : (budget_per_way >> 8) > 0 ? (budget_per_way >> 8) : 1;
    const long long stride = (long long)gridDim.x * blockDim.x;
    // the loop is uniform per warp (every lane makes the same trips) so that the warp can re-converge explicitly between the phases:
    // measured on the first version, the divergent tail of the probe loop ran the stamp + accumulator code with ~7 of 32 lanes active
    for (long long wbase = (long long)blockIdx.x * blockDim.x + (threadIdx.x & ~31); wbase < n; wbase += stride * R) {
        typename P::Regs regs[R];
        long long row[R];
#pragma unroll
        for (int j = 0; j < R; j++) {
            long long i = wbase + lane + (long long)j * stride;
            row[j] = i < n ? (rows ? (long long)rows[i] : first + i) : -1;
            if (row[j] >= 0) prog.load(cols, row[j], regs[j]);
        }
        unsigned long long pk[R], pos[R], cur[R], nxt[R];
        long long slot[R];
        bool open[R];        // still looking for its slot
#pragma unroll
        for (int j = 0; j < R; j++) {
            pk[j] = 0;
            int sp = -1;
            if (row[j] >= 0 && !prog.row(regs[j], &pk[j], &sp, &err)) row[j] = -1;      // rejected by the fused filter
            pos[j] = tgd_murmur3_mix(pk[j]) & mask;
            slot[j] = (row[j] >= 0 && sp >= 0) ? cap + sp : -1;
            open[j] = row[j] >= 0 && sp < 0;
        }
        // one 16-byte load brings the home slot's key AND its first-row stamp; the successor's key is requested with it: a row that
        // has to move on finds the next key already on its way, and a row that stays (most do) never reads its stamp separately
        unsigned long long st0[R];
#pragma unroll
        for (int j = 0; j < R; j++) {
            cur[j] = 0; st0[j] = 0; nxt[j] = 0;
            if (open[j]) {
                tgd_ld_pair(recs + (size_t)pos[j] * W, cur[j], st0[j]);
                nxt[j] = *((volatile unsigned long long*)(recs + (size_t)((pos[j] + 1) & mask) * W));
            }
        }
        bool moved[R];
#pragma unroll
        for (int j = 0; j < R; j++) moved[j] = false;
        // lock-step probing: one step of every open row per trip, the warp stays converged.  Insertions need a ticket (the fill limit
        // of the table is a budget of tickets per way); a warp draws them in batches and keeps the remainder (`have`, warp-uniform), so
        // the returning atomicAdd sits on the critical path of one insertion in `batch`, not of every trip that inserts.
        while (true) {
            bool any = false;
#pragma unroll
            for (int j = 0; j < R; j++) {
                bool active = open[j];
                unsigned long long c = cur[j];
                const bool want = active && c == TGD_EMPTY_KEY;
                const unsigned int wmask = __ballot_sync(0xffffffffu, want);
                if (wmask) {
                    const int cnt = __popc(wmask), leader = __ffs(wmask) - 1;
                    if (cnt > have) {
                        int got = 0;
                        if (lane == leader) {
                            const int ask = cnt - have > batch ? cnt - have : batch;
                            const int base = atomicAdd(tickets + way, ask);
                            got = budget_per_way - base;
                            got = got < 0 ? 0 : (got > ask ? ask : got);
                            if (got < ask) atomicSub(tickets + way, ask - got);          // drawn beyond the budget: handed back at once
                        }
                        have += __shfl_sync(0xffffffffu, got, leader);
                    }
                    const bool granted = want && __popc(wmask & ((1u << lane) - 1)) < have;
                    have -= cnt < have ? cnt : have;
                    bool won = false;
                    if (granted) {
                        c = atomicCAS(recs + (size_t)pos[j] * W, TGD_EMPTY_KEY, pk[j]);
                        won = c == TGD_EMPTY_KEY;
                    }
                    have += __popc(__ballot_sync(0xffffffffu, granted && !won));          // lost the race for the slot: the ticket stays in hand
                    if (want && !granted) { open[j] = false; active = false; }              // no room: deferred below
                    if (won) { slot[j] = (long long)pos[j]; open[j] = false; active = false; }
                }
                if (active) {
                    if (c == pk[j]) { slot[j] = (long long)pos[j]; open[j] = false; }
                    else {
                        pos[j] = (pos[j] + 1) & mask;
                        cur[j] = nxt[j];
                        nxt[j] = *((volatile unsigned long long*)(recs + (size_t)((pos[j] + 1) & mask) * W));
                        moved[j] = true;
                        any = true;
                    }
                }
            }
            if (!__any_sync(0xffffffffu, any)) break;
        }
        __syncwarp();
        // stamps: read the R stamps first, lower the ones that need it
        long long stamp[R], seen[R];
#pragma unroll
        for (int j = 0; j < R; j++) {
            stamp[j] = 0;
            seen[j] = 0;
            if (row[j] >= 0 && slot[j] >= 0) {
                stamp[j] = page_base + (stamp_rows ? (long long)stamp_rows[row[j]] : row[j]);
                // (a stamp read together with the key may be stale, i.e. too high: stamps only ever go down, so the worst case is one
                //  atomicMin that changes nothing)
                seen[j] = (!moved[j] && slot[j] < cap) ? (long long)st0[j] : *((volatile long long*)(recs + (size_t)slot[j] * W + 1));
            }
        }
#pragma unroll
        for (int j = 0; j < R; j++) {
            if (row[j] < 0) continue;
            if (slot[j] < 0) { deferred[atomicAdd(tickets + TGD_TICKET_WAYS, 1)] = (int)row[j]; continue; }
            if (seen[j] > stamp[j]) {
                long long old = atomicMin((long long*)(recs + (size_t)slot[j] * W + 1), stamp[j]);
                if (old == TGD_NO_ROW && slot[j] >= cap) atomicAdd(tickets + TGD_TICKET_WAYS + 1, 1);   // a special (NULL / sentinel key) group came to life
            }
        }
        __syncwarp();
#pragma unroll
        for (int j = 0; j < R; j++) {
            if (row[j] < 0 || slot[j] < 0) continue;
            unsigned long long pk2;
            int sp2;
            prog.row(regs[j], &pk2, &sp2, &err);          // re-establish this row's values (registers only) for the accumulators
            prog.accumulate_global(recs + (size_t)slot[j] * W + 2);
        }
    }
    if (lane == 0 && have > 0) atomicSub(tickets + way, have);        // tickets drawn and not used
    if (err) atomicOr(err_out, err);
}

// ---- FilterAndProject in two passes without a selection vector -------------------------------------------------------------
// Every CTA owns a contiguous chunk of rows.  Pass 1 evaluates the filter (flags, 1 byte per row) and counts the selected rows
// of the chunk; a scan of the chunk counts gives every chunk its first output row.  Pass 2 ranks the selected rows of a tile
// (ballot + a scan over the tile's (iteration, warp) cells), evaluates the projections and copies the pass-through channels
// straight to output row chunk_off + rank: output order = input order (PageProcessor.java:302-336).
// P supplies: static bool filter(cols, row, err*), static void row(cols, row, j, out, err*, nulls_seen*).
constexpr int FPC_R = 4;          // tile = FPC_R x 256 rows
constexpr int FPC_T = 256;

template <class P>
__device__ __forceinline__ void fp_filter_chunks_body(const DColumns& cols, long long n, long long chunk, unsigned char* __restrict__ flags,
                                                      unsigned int* __restrict__ chunk_counts, unsigned int* __restrict__ err_out)
{
    __shared__ unsigned int warp_sel[FPC_T / 32];
    const long long begin = (long long)blockIdx.x * chunk, end = begin + chunk < n ? begin + chunk : n;
    unsigned int err = 0, mine = 0;
    for (long long row = begin + threadIdx.x; row < end; row += FPC_T) {
        bool s = P::filter(cols, row, &err);
        flags[row] = s ? 1 : 0;
        mine += s ? 1u : 0u;
    }
    for (int off = 16; off > 0; off >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, off);
    if ((threadIdx.x & 31) == 0) warp_sel[threadIdx.x >> 5] = mine;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned int total = 0;
        for (int w = 0; w < FPC_T / 32; w++) total += warp_sel[w];
        chunk_counts[blockIdx.x] = total;
    }
    if (err) atomicOr(err_out, err);
}

template <class P>
__device__ __forceinline__ void fp_project_chunks_body(const DColumns& cols, const unsigned char* __restrict__ flags, long long n, long long chunk,
                                                       const long long* __restrict__ chunk_off, const OutCols& out, unsigned int* __restrict__ err_out,
                                                       unsigned int* __restrict__ any_null)
{
    constexpr int NW = FPC_T / 32;
    __shared__ unsigned int cells[FPC_R * NW];     // selected rows per (iteration, warp), then their exclusive prefix
    __shared__ unsigned int tile_total;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long begin = (long long)blockIdx.x * chunk, end = begin + chunk < n ? begin + chunk : n;
    long long running = chunk_off[blockIdx.x];
    unsigned int err = 0, nulls_seen = 0;
    for (long long tile = begin; tile < end; tile += (long long)FPC_R * FPC_T) {
        bool sel[FPC_R];
        unsigned int rank[FPC_R];
#pragma unroll
        for (int i = 0; i < FPC_R; i++) {
            long long row = tile + (long long)i * FPC_T + threadIdx.x;
            sel[i] = row < end && flags[row] != 0;
            unsigned int b = __ballot_sync(0xffffffffu, sel[i]);
            rank[i] = __popc(b & ((1u << lane) - 1));
            if (lane == 0) cells[i * NW + warp] = __popc(b);
        }
        __syncthreads();
        if (warp == 0) {
            static_assert(FPC_R * NW == 32, "one cell per lane");
            unsigned int v = cells[lane], incl = v;
            for (int off = 1; off < 32; off <<= 1) {
                unsigned int u = __shfl_up_sync(0xffffffffu, incl, off);
                if (lane >= off) incl += u;
            }
            cells[lane] = incl - v;
            if (lane == 31) tile_total = incl;
        }
        __syncthreads();
#pragma unroll
        for (int i = 0; i < FPC_R; i++) {
            if (!sel[i]) continue;
            long long row = tile + (long long)i * FPC_T + threadIdx.x;
            P::row(cols, row, running + cells[i * NW + warp] + rank[i], out, &err, &nulls_seen);
        }
        running += tile_total;
        __syncthreads();
    }
    if (err) atomicOr(err_out, err);
    if (nulls_seen) atomicOr(any_null, nulls_seen);
}

#endif  // __CUDACC__
#endif  // TG_DEVICE_LIB_CUH
