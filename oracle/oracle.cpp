// oracle.cpp — CPU restatement of the reference algorithms.  TEST INFRASTRUCTURE ONLY (see oracle.h).
// Every function cites the reference file:line it follows; nothing here is shipped in libtrino_gpu.so.
// Compile: g++ -O3 -march=native -ffp-contract=off -std=c++17 -shared -fPIC -pthread
// (-ffp-contract=off: Java never fuses a*b+c; M/type/DoubleOperators.java:66-86)
#include <sys/syscall.h>
#include <unistd.h>
#include "oracle.h"

#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <functional>
#include <mutex>
#include <chrono>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <string>
#include <unordered_set>
#include <thread>
#include <vector>

namespace {

// ------------------------------------------------------------------------------------------------
// hashes
// ------------------------------------------------------------------------------------------------
constexpr uint64_t P1 = 0x9E3779B185EBCA87ULL, P2 = 0xC2B2AE3D27D4EB4FULL, P3 = 0x165667B19E3779F9ULL,
                   P4 = 0x85EBCA77C2B2AE63ULL, P5 = 0x27D4EB2F165667C5ULL;

inline uint64_t rotl(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }

// S/type/AbstractLongType.java:121-125
inline uint64_t hash_long(int64_t v) { return rotl((uint64_t)v * P2, 31) * P1; }

// Java Double.doubleToLongBits: every NaN collapses to 0x7ff8000000000000
inline int64_t double_to_long_bits(double d)
{
    if (d != d) return 0x7ff8000000000000LL;
    int64_t b;
    memcpy(&b, &d, 8);
    return b;
}

// S/type/DoubleType.java:199-206
inline uint64_t hash_double(double d)
{
    if (d == 0) d = 0;  // collapses -0.0 to +0.0
    return hash_long(double_to_long_bits(d));
}

// S/type/RealType.java:151-159: AbstractLongType.hash(floatToIntBits(v)) with -0.0 collapsed to +0.0; Float.floatToIntBits collapses every
// NaN to 0x7fc00000 and the int widens to long with its sign
inline uint64_t hash_real(float f)
{
    if (f == 0) f = 0;
    int32_t bits;
    if (f != f) bits = 0x7fc00000;
    else memcpy(&bits, &f, 4);
    return hash_long((int64_t)bits);
}

inline uint64_t rd64(const uint8_t* p) { uint64_t v; memcpy(&v, p, 8); return v; }
inline uint32_t rd32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }

// public XXH64 algorithm (io.airlift.slice.XxHash64; not vendored under trinodb/trino)
uint64_t xxh64(const uint8_t* p, int64_t len, uint64_t seed)
{
    const uint8_t* end = p + len;
    uint64_t h;
    if (len >= 32) {
        uint64_t v1 = seed + P1 + P2, v2 = seed + P2, v3 = seed, v4 = seed - P1;
        const uint8_t* limit = end - 32;
        do {
            v1 = rotl(v1 + rd64(p) * P2, 31) * P1;
            v2 = rotl(v2 + rd64(p + 8) * P2, 31) * P1;
            v3 = rotl(v3 + rd64(p + 16) * P2, 31) * P1;
            v4 = rotl(v4 + rd64(p + 24) * P2, 31) * P1;
            p += 32;
        } while (p <= limit);
        h = rotl(v1, 1) + rotl(v2, 7) + rotl(v3, 12) + rotl(v4, 18);
        auto merge = [&](uint64_t v) { h ^= rotl(v * P2, 31) * P1; h = h * P1 + P4; };
        merge(v1); merge(v2); merge(v3); merge(v4);
    }
    else {
        h = seed + P5;
    }
    h += (uint64_t)len;
    while (p + 8 <= end) { h ^= rotl(rd64(p) * P2, 31) * P1; h = rotl(h, 27) * P1 + P4; p += 8; }
    if (p + 4 <= end) { h ^= (uint64_t)rd32(p) * P1; h = rotl(h, 23) * P2 + P3; p += 4; }
    while (p < end) { h ^= (uint64_t)(*p) * P5; h = rotl(h, 11) * P1; p++; }
    h ^= h >> 33; h *= P2; h ^= h >> 29; h *= P3; h ^= h >> 32;
    return h;
}

inline uint64_t xxh64_long(int64_t v)
{
    uint8_t b[8];
    memcpy(b, &v, 8);
    return xxh64(b, 8, 0);
}

// M/operator/join/PagesHash.java:44-50 (== fastutil HashCommon.murmurHash3)
inline uint64_t murmur3(uint64_t x)
{
    x ^= x >> 33; x *= 0xff51afd7ed558ccdULL; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ULL; x ^= x >> 33;
    return x;
}

inline uint64_t bitreverse64(uint64_t x)
{
    x = ((x >> 1) & 0x5555555555555555ULL) | ((x & 0x5555555555555555ULL) << 1);
    x = ((x >> 2) & 0x3333333333333333ULL) | ((x & 0x3333333333333333ULL) << 2);
    x = ((x >> 4) & 0x0F0F0F0F0F0F0F0FULL) | ((x & 0x0F0F0F0F0F0F0F0FULL) << 4);
    return __builtin_bswap64(x);
}

// fastutil 8.5.18 HashCommon.arraySize(expected, f) = max(2, nextPowerOfTwo(ceil(expected / f)))
int32_t array_size(int64_t expected, double f)
{
    // fastutil takes f as float; ceil(expected / f) evaluated in double after float->double widening
    double fd = (double)(float)f;
    int64_t need = (int64_t)std::ceil((double)expected / fd);
    int64_t s = 1;
    while (s < need) s <<= 1;
    if (s < 2) s = 2;
    if (s > (1LL << 30)) return -1;
    return (int32_t)s;
}

// M/operator/HashGenerator.java:41-46: Long.hashCode then scale to [0, partitionCount)
inline int32_t process_raw_hash(int64_t raw, int32_t count)
{
    uint32_t x = (uint32_t)((uint64_t)raw ^ ((uint64_t)raw >> 32));
    return (int32_t)(((uint64_t)x * (uint64_t)(uint32_t)count) >> 32);
}

// ------------------------------------------------------------------------------------------------
// column access
// ------------------------------------------------------------------------------------------------
struct ColView {
    const tgpu_column* col;     // the value column (after unwrapping DICT/RLE)
    const int32_t* ids;         // DICT32 ids or null
    bool rle;
    bool bytemap;
    int type;

    explicit ColView(const tgpu_column* c) : ids(nullptr), rle(false)
    {
        if (c->type == TGPU_DICT32) { ids = (const int32_t*)c->data; c = c->dictionary; }
        else if (c->type == TGPU_RLE) { rle = true; c = c->dictionary; }
        col = c;
        type = c->type;
        bytemap = (c->flags & TGPU_COL_NULLS_BYTEMAP) != 0;
    }
    inline int64_t pos(int64_t i) const { return rle ? 0 : (ids ? ids[i] : i); }
    inline bool is_null(int64_t i) const
    {
        if (!col->validity) return false;
        int64_t p = pos(i);
        if (bytemap) return col->validity[p] != 0;
        return ((col->validity[p >> 3] >> (p & 7)) & 1) == 0;
    }
    inline int64_t i64(int64_t i) const
    {
        int64_t p = pos(i);
        switch (type) {
            case TGPU_INT64: return ((const int64_t*)col->data)[p];
            case TGPU_INT32: return ((const int32_t*)col->data)[p];
            case TGPU_INT16: return ((const int16_t*)col->data)[p];
            case TGPU_INT8: return ((const int8_t*)col->data)[p];
            case TGPU_FLOAT64: return ((const int64_t*)col->data)[p];
            case TGPU_FLOAT32: return ((const int32_t*)col->data)[p];     // REAL: the float's raw bits in an IntArrayBlock (S/type/RealType.java:104-121)
            default: return 0;
        }
    }
    // Int128ArrayBlock: long[2 * positions], the high word first (S/block/Int128ArrayBlock.java:123-133)
    inline int64_t i128_high(int64_t i) const { return ((const int64_t*)col->data)[2 * pos(i)]; }
    inline int64_t i128_low(int64_t i) const { return ((const int64_t*)col->data)[2 * pos(i) + 1]; }
    inline double f64(int64_t i) const { return ((const double*)col->data)[pos(i)]; }
    inline float f32(int64_t i) const { return ((const float*)col->data)[pos(i)]; }
    inline const uint8_t* bytes(int64_t i, int32_t* len) const
    {
        int64_t p = pos(i);
        int32_t a = col->offsets[p], b = col->offsets[p + 1];
        *len = b - a;
        return (const uint8_t*)col->data + a;
    }
    // per-type hash code, null -> 0 (NULL_HASH_CODE, S/type/TypeUtils.java:34)
    inline uint64_t hash(int64_t i) const
    {
        if (is_null(i)) return 0;
        switch (type) {
            case TGPU_FLOAT64: return hash_double(f64(i));
            case TGPU_FLOAT32: return hash_real(f32(i));
            case TGPU_UTF8: { int32_t len; const uint8_t* b = bytes(i, &len); return xxh64(b, len, 0); }
            case TGPU_INT128: return xxh64_long(i128_high(i)) ^ xxh64_long(i128_low(i));   // S/type/LongDecimalType.java:203-229
            default: return hash_long(i64(i));  // integer widths sign-extend first (AbstractIntType.java:183-187)
        }
    }
    // IDENTICAL semantics on the non-null values of two positions (group-by keys)
    inline bool identical(int64_t i, const ColView& o, int64_t j) const
    {
        switch (type) {
            case TGPU_FLOAT64: {
                double a = f64(i), b = o.f64(j);
                if (a != a && b != b) return true;
                return a == b;
            }
            case TGPU_FLOAT32: {      // S/type/RealType.java:172-185
                float a = f32(i), b = o.f32(j);
                if (a != a && b != b) return true;
                return a == b;
            }
            case TGPU_UTF8: {
                int32_t la, lb;
                const uint8_t* a = bytes(i, &la);
                const uint8_t* b = o.bytes(j, &lb);
                return la == lb && memcmp(a, b, la) == 0;
            }
            case TGPU_INT128: return i128_high(i) == o.i128_high(j) && i128_low(i) == o.i128_low(j);   // LongDecimalType.java:190-201
            default: return i64(i) == o.i64(j);
        }
    }
    // EQUAL semantics (join keys): NaN never equals
    inline bool equal(int64_t i, const ColView& o, int64_t j) const
    {
        if (type == TGPU_FLOAT64) return f64(i) == o.f64(j);
        if (type == TGPU_FLOAT32) return f32(i) == o.f32(j);       // S/type/RealType.java:145-149
        return identical(i, o, j);
    }
};

inline uint64_t row_hash(const std::vector<ColView>& cols, int64_t i)
{
    uint64_t h = 0;  // INITIAL_HASH_VALUE, M/operator/HashGenerator.java:20
    for (const ColView& c : cols) h = 31 * h + c.hash(i);
    return h;
}

std::vector<ColView> views(const tgpu_page* page, const int32_t* channels, int32_t n)
{
    std::vector<ColView> v;
    for (int32_t k = 0; k < n; k++) v.emplace_back(&page->columns[channels ? channels[k] : k]);
    return v;
}

inline bool valid_bit(const uint8_t* validity, int64_t i) { return !validity || ((validity[i >> 3] >> (i & 7)) & 1); }

// a stored copy of one key tuple (FlatHash record; M/operator/FlatHash.java:90-96)
struct KeyCell {
    uint8_t is_null;
    int64_t fixed;           // raw 64-bit value for fixed-width types (INT128: the high word)
    int64_t fixed_low;       // INT128: the low word
    std::string bytes;       // UTF8
};

}  // namespace

// ================================================================================================
extern "C" {

uint64_t orc_hash_long(int64_t v) { return hash_long(v); }
uint64_t orc_hash_double(double d) { return hash_double(d); }
uint64_t orc_hash_real(float f) { return hash_real(f); }
uint64_t orc_xxh64(const void* data, int64_t len, uint64_t seed) { return xxh64((const uint8_t*)data, len, seed); }
uint64_t orc_xxh64_long(int64_t v) { return xxh64_long(v); }
uint64_t orc_murmur3(uint64_t x) { return murmur3(x); }
uint64_t orc_combine_hash(uint64_t prev, uint64_t v) { return 31 * prev + v; }
int32_t orc_array_size(int64_t expected, double f) { return array_size(expected, f); }

int32_t orc_join_hash_array_size(int64_t n)
{
    if (n <= (1 << 16)) return array_size(n, 0.25);
    if (n <= (1 << 20)) return array_size(n, 0.5);
    return array_size(n, 0.75);
}

int32_t orc_process_raw_hash(int64_t raw, int32_t count) { return process_raw_hash(raw, count); }

int32_t orc_local_partition(int64_t raw, int32_t p)
{
    return (int32_t)xxh64_long((int64_t)bitreverse64((uint64_t)raw)) & (p - 1);
}

void orc_row_hashes(const tgpu_page* page, const int32_t* channels, int32_t n, int64_t* out)
{
    auto cols = views(page, channels, n);
    for (int64_t i = 0; i < page->num_rows; i++) out[i] = (int64_t)row_hash(cols, i);
}

// ------------------------------------------------------------------------------------------------
// GroupByHash
// ------------------------------------------------------------------------------------------------
struct orc_groupby {
    int kind;           // 0 auto, 1 bigint, 2 flat
    int resolved = 0;
    int expected;
    // --- BigintGroupByHash state (M/operator/BigintGroupByHash.java:49-66)
    int32_t capacity = 0, max_fill = 0, mask = 0;
    std::vector<int64_t> values;
    std::vector<int32_t> group_ids;
    int32_t null_group = -1;
    int32_t next_group = 0;
    // --- FlatHash state (M/operator/FlatHash.java:64-78)
    std::vector<uint8_t> control;          // capacity + 8 (mirror of the first vector)
    std::vector<int32_t> ids_by_hash;
    std::vector<uint64_t> group_hash;      // cached hash per group (cacheHashValue records)
    std::vector<std::vector<KeyCell>> group_keys;
};

static int32_t bigint_max_fill(int32_t cap)
{   // BigintGroupByHash.calculateMaxFill :302-311
    int32_t mf = (int32_t)std::ceil(cap * 0.75f);
    if (mf == cap) mf--;
    return mf;
}

static void bigint_init(orc_groupby* g)
{
    g->capacity = array_size(g->expected, 0.75);
    g->max_fill = bigint_max_fill(g->capacity);
    g->mask = g->capacity - 1;
    g->values.assign(g->capacity, 0);
    g->group_ids.assign(g->capacity, -1);
}

// BigintGroupByHash.tryRehash :239-290
static int bigint_rehash(orc_groupby* g)
{
    int64_t ncap = (int64_t)g->capacity * 2;
    if (ncap > INT32_MAX) return -3;
    int32_t nmask = (int32_t)ncap - 1;
    std::vector<int64_t> nv(ncap, 0);
    std::vector<int32_t> ng(ncap, -1);
    for (int32_t i = 0; i < g->capacity; i++) {
        int32_t gid = g->group_ids[i];
        if (gid == -1) continue;
        int64_t v = g->values[i];
        int32_t pos = (int32_t)(murmur3((uint64_t)v) & (uint64_t)nmask);
        while (ng[pos] != -1) pos = (pos + 1) & nmask;
        nv[pos] = v;
        ng[pos] = gid;
    }
    g->capacity = (int32_t)ncap;
    g->mask = nmask;
    g->max_fill = bigint_max_fill(g->capacity);
    g->values.swap(nv);
    g->group_ids.swap(ng);
    return 0;
}

// BigintGroupByHash.putIfAbsent :191-221 + addNewGroup :223-237
static int32_t bigint_put(orc_groupby* g, bool is_null, int64_t value, int* err)
{
    if (is_null) {
        if (g->null_group < 0) g->null_group = g->next_group++;
        return g->null_group;
    }
    int32_t pos = (int32_t)(murmur3((uint64_t)value) & (uint64_t)g->mask);
    while (true) {
        int32_t gid = g->group_ids[pos];
        if (gid == -1) break;
        if (value == g->values[pos]) return gid;
        pos = (pos + 1) & g->mask;
    }
    int32_t gid = g->next_group++;
    g->values[pos] = value;
    g->group_ids[pos] = gid;
    if (g->next_group >= g->max_fill) {
        int e = bigint_rehash(g);
        if (e) *err = e;
    }
    return gid;
}

// FlatHash.computeCapacity :44-48 / calculateMaxFill :50-53
static int32_t flat_capacity(int32_t max_size)
{
    int32_t cap = (int32_t)(max_size / (15.0 / 16));
    int64_t p = 1;
    while (p < cap) p <<= 1;   // 1L << (64 - nlz(cap - 1))
    return (int32_t)std::max<int64_t>(p, 16);
}

static inline uint64_t swar_match(uint64_t vec, uint64_t repeated)
{   // FlatHash.match :489-494
    uint64_t c = vec ^ repeated;
    return (c - 0x0101010101010101ULL) & ~c & 0x8080808080808080ULL;
}

static void flat_init(orc_groupby* g, int32_t cap)
{
    g->capacity = cap;
    g->mask = cap - 1;
    g->max_fill = (int32_t)((int64_t)cap * 15 / 16);
    g->control.assign(cap + 8, 0);
    g->ids_by_hash.assign(cap, -1);
}

static inline void flat_set_control(orc_groupby* g, int32_t index, uint8_t prefix)
{   // FlatHash.setControl :350-356: mirror the first vector after the end
    g->control[index] = prefix;
    if (index < 8) g->control[index + g->capacity] = prefix;
}

// FlatHash.rehash :381-423
static int flat_rehash(orc_groupby* g)
{
    int64_t ncap = (int64_t)g->capacity * 2;
    if (ncap > (1LL << 30)) return -3;
    flat_init(g, (int32_t)ncap);
    for (int32_t gid = 0; gid < g->next_group; gid++) {
        uint64_t hash = g->group_hash[gid];
        uint8_t prefix = (uint8_t)((hash & 0x7F) | 0x80);
        int32_t bucket = (int32_t)((int64_t)hash >> 7) & g->mask;
        int32_t step = 1;
        while (true) {
            uint64_t vec = rd64(&g->control[bucket]);
            uint64_t empties = swar_match(vec, 0);
            if (empties) {
                int32_t idx = (bucket + (__builtin_ctzll(empties) >> 3)) & g->mask;
                flat_set_control(g, idx, prefix);
                g->ids_by_hash[idx] = gid;
                break;
            }
            bucket = (bucket + step) & g->mask;
            step += 8;
        }
    }
    return 0;
}

// FlatHash.putIfAbsent :238-255, getIndex :257-282, matchInVector :284-297, addNewGroup :309-348
static int32_t flat_put(orc_groupby* g, const std::vector<ColView>& cols, int64_t row, uint64_t hash, int* err)
{
    uint8_t prefix = (uint8_t)((hash & 0x7F) | 0x80);
    int32_t bucket = (int32_t)((int64_t)hash >> 7) & g->mask;
    int32_t step = 1;
    uint64_t repeated = (uint64_t)prefix * 0x0101010101010101ULL;
    int32_t insert_at = -1;
    while (true) {
        uint64_t vec = rd64(&g->control[bucket]);
        uint64_t m = swar_match(vec, repeated);
        while (m) {
            int32_t idx = (bucket + (__builtin_ctzll(m) >> 3)) & g->mask;
            int32_t gid = g->ids_by_hash[idx];
            // valueIdentical :445-469: cached hash first, then per-column IDENTICAL incl. null flags
            if (g->group_hash[gid] == hash) {
                bool same = true;
                const std::vector<KeyCell>& k = g->group_keys[gid];
                for (size_t c = 0; c < cols.size() && same; c++) {
                    bool n = cols[c].is_null(row);
                    if (n != (bool)k[c].is_null) { same = false; break; }
                    if (n) continue;
                    switch (cols[c].type) {
                        case TGPU_UTF8: {
                            int32_t len; const uint8_t* b = cols[c].bytes(row, &len);
                            same = (size_t)len == k[c].bytes.size() && memcmp(b, k[c].bytes.data(), len) == 0;
                            break;
                        }
                        case TGPU_FLOAT64: {
                            double a = cols[c].f64(row), b; memcpy(&b, &k[c].fixed, 8);
                            same = (a != a && b != b) || a == b;
                            break;
                        }
                        case TGPU_FLOAT32: {
                            float a = cols[c].f32(row), b; int32_t bits = (int32_t)k[c].fixed; memcpy(&b, &bits, 4);
                            same = (a != a && b != b) || a == b;
                            break;
                        }
                        case TGPU_INT128: same = cols[c].i128_high(row) == k[c].fixed && cols[c].i128_low(row) == k[c].fixed_low; break;
                        default: same = cols[c].i64(row) == k[c].fixed;
                    }
                }
                if (same) return gid;
            }
            m &= m - 1;
        }
        uint64_t empties = swar_match(vec, 0);
        if (empties) { insert_at = (bucket + (__builtin_ctzll(empties) >> 3)) & g->mask; break; }
        bucket = (bucket + step) & g->mask;
        step += 8;
    }
    flat_set_control(g, insert_at, prefix);
    int32_t gid = g->next_group++;
    g->ids_by_hash[insert_at] = gid;
    g->group_hash.push_back(hash);
    std::vector<KeyCell> k(cols.size());
    for (size_t c = 0; c < cols.size(); c++) {
        k[c].is_null = cols[c].is_null(row);
        k[c].fixed = 0;
        k[c].fixed_low = 0;
        if (k[c].is_null) continue;
        if (cols[c].type == TGPU_INT128) { k[c].fixed = cols[c].i128_high(row); k[c].fixed_low = cols[c].i128_low(row); continue; }
        if (cols[c].type == TGPU_UTF8) { int32_t len; const uint8_t* b = cols[c].bytes(row, &len); k[c].bytes.assign((const char*)b, len); }
        else if (cols[c].type == TGPU_FLOAT64) { double d = cols[c].f64(row); memcpy(&k[c].fixed, &d, 8); }
        else k[c].fixed = cols[c].i64(row);
    }
    g->group_keys.push_back(std::move(k));
    if (g->next_group >= g->max_fill) {
        int e = flat_rehash(g);
        if (e) *err = e;
    }
    return gid;
}

orc_groupby* orc_groupby_create(int32_t kind, int32_t expected)
{
    orc_groupby* g = new orc_groupby();
    g->kind = kind;
    g->expected = expected < 1 ? 1 : expected;
    return g;
}

void orc_groupby_destroy(orc_groupby* g) { delete g; }

int32_t orc_groupby_get_group_ids(orc_groupby* g, const tgpu_page* page, const int32_t* key_channels, int32_t num_keys, int32_t* out)
{
    auto cols = views(page, key_channels, num_keys);
    if (!g->resolved) {
        // GroupByHash.createGroupByHash :82-100
        bool single_bigint = num_keys == 1 && cols[0].type == TGPU_INT64;
        g->resolved = g->kind ? g->kind : (single_bigint ? 1 : 2);
        if (g->resolved == 1) bigint_init(g);
        else flat_init(g, std::max(8, flat_capacity(g->expected)));
    }
    int err = 0;
    if (g->resolved == 1) {
        for (int64_t i = 0; i < page->num_rows; i++) out[i] = bigint_put(g, cols[0].is_null(i), cols[0].i64(i), &err);
    }
    else {
        // FlatGroupByHash.GetNonDictionaryGroupIdsWork :515-540 (hashBlocksBatched then putIfAbsent per row)
        for (int64_t i = 0; i < page->num_rows; i++) out[i] = flat_put(g, cols, i, row_hash(cols, i), &err);
    }
    return err;
}

int32_t orc_groupby_group_count(const orc_groupby* g) { return g->next_group; }
int32_t orc_groupby_capacity(const orc_groupby* g) { return g->capacity; }

// ------------------------------------------------------------------------------------------------
// accumulators (left fold in row order)
// ------------------------------------------------------------------------------------------------
static inline bool selected(const uint8_t* mask_sel, int64_t i) { return !mask_sel || mask_sel[i]; }

void orc_agg_sum_double(const int32_t* gids, int64_t n, const double* v, const uint8_t* validity, const uint8_t* mask_sel, double* sum, uint8_t* nonnull)
{   // DoubleSumAggregation.sum :37-41
    for (int64_t i = 0; i < n; i++) {
        if (!selected(mask_sel, i) || !valid_bit(validity, i)) continue;
        nonnull[gids[i]] = 1;
        sum[gids[i]] = sum[gids[i]] + v[i];
    }
}

void orc_agg_avg_double(const int32_t* gids, int64_t n, const double* v, const uint8_t* validity, const uint8_t* mask_sel, double* sum, int64_t* count)
{   // DoubleAverageAggregations.input :37-41
    for (int64_t i = 0; i < n; i++) {
        if (!selected(mask_sel, i) || !valid_bit(validity, i)) continue;
        count[gids[i]] += 1;
        sum[gids[i]] = sum[gids[i]] + v[i];
    }
}

void orc_agg_count(const int32_t* gids, int64_t n, const uint8_t* validity, const uint8_t* mask_sel, int64_t* count)
{   // CountAggregation.input :36-39 (validity == NULL) / CountColumn (non-null inputs only)
    for (int64_t i = 0; i < n; i++) {
        if (!selected(mask_sel, i) || !valid_bit(validity, i)) continue;
        count[gids[i]] += 1;
    }
}

int32_t orc_agg_sum_bigint(const int32_t* gids, int64_t n, const int64_t* v, const uint8_t* validity, const uint8_t* mask_sel, int64_t* sum, uint8_t* nonnull)
{   // BigintSumAggregation.sum :38-42 with BigintOperators.add = Math.addExact
    for (int64_t i = 0; i < n; i++) {
        if (!selected(mask_sel, i) || !valid_bit(validity, i)) continue;
        nonnull[gids[i]] = 1;
        int64_t r;
        if (__builtin_add_overflow(sum[gids[i]], v[i], &r)) return -4;
        sum[gids[i]] = r;
    }
    return 0;
}

// DecimalSumAggregation (M/operator/aggregation/DecimalSumAggregation.java:44-146) over LongDecimalWithOverflowState: per group
// decimal[2] = (high, low), overflow, notNull.  `values` holds n x (high, low) pairs (long decimal input, :67-90) or, with is_short,
// n BIGINT values sign-extended to 128 bits (:44-65).  Int128Math.addWithOverflow :192-210 word for word.
static int64_t add_with_overflow(int64_t left_high, int64_t left_low, int64_t right_high, int64_t right_low, int64_t* out)
{
    int64_t low = (int64_t)((uint64_t)left_low + (uint64_t)right_low);
    int64_t low_carry = ((uint64_t)low < (uint64_t)left_low) ? 1 : 0;              // unsignedCarry
    int64_t high = (int64_t)((uint64_t)left_high + (uint64_t)right_high + (uint64_t)low_carry);
    int64_t overflow = 0;
    if (left_high >= 0 && right_high >= 0 && high < 0) overflow = 1;
    else if (left_high < 0 && right_high < 0 && high >= 0) overflow = -1;
    out[0] = high;
    out[1] = low;
    return overflow;
}

void orc_agg_sum_decimal(const int32_t* gids, int64_t n, const int64_t* values, int32_t is_short, const uint8_t* validity, const uint8_t* mask_sel,
                         int64_t* decimal /* [groups][2] */, int64_t* overflow, uint8_t* nonnull)
{
    for (int64_t i = 0; i < n; i++) {
        if (!selected(mask_sel, i) || !valid_bit(validity, i)) continue;
        const int32_t g = gids[i];
        nonnull[g] = 1;
        const int64_t right_low = is_short ? values[i] : values[2 * i + 1];
        const int64_t right_high = is_short ? (values[i] >> 63) : values[2 * i];
        overflow[g] += add_with_overflow(decimal[2 * g], decimal[2 * g + 1], right_high, right_low, decimal + 2 * g);
    }
}

// combine :92-120 of one other state into a group's state
void orc_agg_sum_decimal_combine(int64_t* decimal, int64_t* overflow, uint8_t* nonnull, const int64_t* other_decimal, int64_t other_overflow)
{
    if (*nonnull) {
        int64_t o = add_with_overflow(decimal[0], decimal[1], other_decimal[0], other_decimal[1], decimal);
        *overflow += o + other_overflow;
    }
    else {
        *nonnull = 1;
        decimal[0] = other_decimal[0];
        decimal[1] = other_decimal[1];
        *overflow = other_overflow;
    }
}

// outputDecimal :122-146: 0 = value ok, -4 = "Decimal overflow" (Decimals.overflows: outside +-(10^38 - 1), S/type/Decimals.java:319-323)
int32_t orc_decimal_sum_overflows(int64_t high, int64_t low, int64_t overflow)
{
    if (overflow != 0) return -4;
    const unsigned __int128 max = ((unsigned __int128)0x4B3B4CA85A86C47AULL << 64) | 0x098A224000000000ULL;    // 10^38
    __int128 v = ((__int128)high << 64) | (unsigned __int128)(uint64_t)low;
    unsigned __int128 a = v < 0 ? (unsigned __int128)(-v) : (unsigned __int128)v;
    return a >= max ? -4 : 0;
}

void orc_agg_minmax_double(const int32_t* gids, int64_t n, const double* v, const uint8_t* validity, int32_t is_max, double* acc, uint8_t* nonnull)
{   // min(DOUBLE): COMPARISON_UNORDERED_LAST, NaN is the largest value (M/operator/aggregation/MinAggregationFunction.java:49,
    // S/type/DoubleType.java:231-235); max(DOUBLE): COMPARISON_UNORDERED_FIRST, NaN is the smallest value
    // (MaxAggregationFunction.java:49, DoubleType.java:237-252): the state is replaced when compare(value, state) > 0 (max)
    // or < 0 (min)
    for (int64_t i = 0; i < n; i++) {
        if (!valid_bit(validity, i)) continue;
        int32_t g = gids[i];
        double x = v[i];
        if (!nonnull[g]) { nonnull[g] = 1; acc[g] = x; continue; }
        double a = acc[g];
        bool xnan = x != x, anan = a != a;
        bool x_greater = is_max ? (anan ? !xnan : (!xnan && x > a))      // unordered first: any number beats NaN
                                : (xnan ? !anan : (!anan && x > a));
        bool x_less = anan ? !xnan : (!xnan && x < a);                   // unordered last (only read for min)
        if (is_max ? x_greater : x_less) acc[g] = x;
    }
}

void orc_agg_minmax_bigint(const int32_t* gids, int64_t n, const int64_t* v, const uint8_t* validity, int32_t is_max, int64_t* acc, uint8_t* nonnull)
{
    for (int64_t i = 0; i < n; i++) {
        if (!valid_bit(validity, i)) continue;
        int32_t g = gids[i];
        if (!nonnull[g]) { nonnull[g] = 1; acc[g] = v[i]; continue; }
        if (is_max ? v[i] > acc[g] : v[i] < acc[g]) acc[g] = v[i];
    }
}

// ------------------------------------------------------------------------------------------------
// hash join
// ------------------------------------------------------------------------------------------------
struct orc_join {
    bool bigint;
    int32_t mask;
    int64_t n;
    std::vector<int32_t> keys;        // slot -> address index, -1 empty
    std::vector<int64_t> values;      // BigintPagesHash: address index -> key
    std::vector<uint8_t> tags;        // DefaultPagesHash.positionToHashes
    std::vector<int32_t> links;       // ArrayPositionLinks.positionLinks
    int64_t link_count = 0;
    // DefaultPagesHash compares against the retained build blocks: we keep views into the caller's page
    tgpu_page build_page;
    std::vector<tgpu_column> build_cols;
    std::vector<int32_t> key_channels;
};

orc_join* orc_join_build(const tgpu_page* build, const int32_t* key_channels, int32_t num_keys, int32_t force_default)
{
    orc_join* j = new orc_join();
    j->n = build->num_rows;
    j->key_channels.assign(key_channels, key_channels + num_keys);
    j->build_cols.assign(build->columns, build->columns + build->num_columns);
    j->build_page = *build;
    j->build_page.columns = j->build_cols.data();
    auto cols = views(&j->build_page, key_channels, num_keys);
    // JoinHashSupplier.getPagesHashType :162-168
    j->bigint = num_keys == 1 && cols[0].type == TGPU_INT64 && ((j->n <= (1 << 20) && !force_default) || force_default == 2);
    int32_t hash_size = orc_join_hash_array_size(j->n);
    j->mask = hash_size - 1;
    j->keys.assign(hash_size, -1);
    j->links.assign(j->n, -1);
    if (j->bigint) {
        // BigintPagesHash ctor :62-100, indexPages :102-120, insertValue :122-141
        j->values.assign(j->n, 0);
        for (int64_t r = 0; r < j->n; r++) {
            if (cols[0].is_null(r)) continue;
            int64_t value = cols[0].i64(r);
            int32_t pos = (int32_t)(murmur3((uint64_t)value) & (uint64_t)j->mask);
            int32_t address = (int32_t)r;
            while (j->keys[pos] != -1) {
                int32_t cur = j->keys[pos];
                if (value == j->values[cur]) {
                    j->links[address] = cur;   // ArrayPositionLinks.link :45-50
                    j->link_count++;
                    break;
                }
                pos = (pos + 1) & j->mask;
            }
            j->keys[pos] = address;
            j->values[address] = value;
        }
    }
    else {
        // DefaultPagesHash ctor :61-99, extractHashes :101-109, indexPages :111-124, insertValue :126-144
        j->tags.assign(j->n, 0);
        for (int64_t r = 0; r < j->n; r++) j->tags[r] = (uint8_t)row_hash(cols, r);
        for (int64_t r = 0; r < j->n; r++) {
            bool any_null = false;
            for (auto& c : cols) any_null |= c.is_null(r);
            if (any_null) continue;
            uint64_t h = row_hash(cols, r);
            int32_t pos = (int32_t)(murmur3(h) & (uint64_t)j->mask);
            int32_t address = (int32_t)r;
            while (j->keys[pos] != -1) {
                int32_t cur = j->keys[pos];
                bool eq = j->tags[cur] == (uint8_t)h;
                for (size_t c = 0; c < cols.size() && eq; c++) eq = cols[c].equal(cur, cols[c], r);
                if (eq) {
                    j->links[address] = cur;
                    j->link_count++;
                    break;
                }
                pos = (pos + 1) & j->mask;
            }
            j->keys[pos] = address;
        }
    }
    return j;
}

void orc_join_destroy(orc_join* j) { delete j; }
int32_t orc_join_hash_size(const orc_join* j) { return j->mask + 1; }
int32_t orc_join_has_links(const orc_join* j) { return j->link_count > 0; }
void orc_join_copy_links(const orc_join* j, int32_t* out) { memcpy(out, j->links.data(), j->n * sizeof(int32_t)); }

void orc_join_positions(const orc_join* j, const tgpu_page* probe, const int32_t* key_channels, int32_t* out)
{
    int32_t nk = (int32_t)j->key_channels.size();
    auto pcols = views(probe, key_channels, nk);
    auto bcols = views(&j->build_page, j->key_channels.data(), nk);
    for (int64_t i = 0; i < probe->num_rows; i++) {
        bool any_null = false;
        for (auto& c : pcols) any_null |= c.is_null(i);
        if (any_null) { out[i] = -1; continue; }   // JoinProbe.fillCache :154-171
        int32_t res = -1;
        if (j->bigint) {
            // BigintPagesHash.getAddressIndex :162-175 (the batched :184-220 form returns the same values)
            int64_t value = pcols[0].i64(i);
            int32_t pos = (int32_t)(murmur3((uint64_t)value) & (uint64_t)j->mask);
            while (j->keys[pos] != -1) {
                if (value == j->values[j->keys[pos]]) { res = j->keys[pos]; break; }
                pos = (pos + 1) & j->mask;
            }
        }
        else {
            // DefaultPagesHash.getAddressIndex :193-282
            uint64_t h = row_hash(pcols, i);
            int32_t pos = (int32_t)(murmur3(h) & (uint64_t)j->mask);
            while (j->keys[pos] != -1) {
                int32_t cur = j->keys[pos];
                bool eq = j->tags[cur] == (uint8_t)h;
                for (int32_t c = 0; c < nk && eq; c++) eq = bcols[c].equal(cur, pcols[c], i);
                if (eq) { res = cur; break; }
                pos = (pos + 1) & j->mask;
            }
        }
        out[i] = res;
    }
}

int64_t orc_join_expand(const orc_join* j, const int32_t* jp, int64_t n, int32_t join_type, int32_t single_match,
                        int32_t* out_probe, int32_t* out_build, int64_t capacity)
{
    // PageJoiner.processProbe :138-163, joinCurrentPosition :203-227, outerJoinCurrentPosition :234-242
    int64_t count = 0;
    // lookupOuterJoin probes like INNER, fullOuterJoin like PROBE_OUTER (M/operator/JoinOperatorType.java); the build rows they
    // emit are the "visited" positions of OuterLookupSource.java:168-196
    bool outer = join_type == TGPU_JOIN_PROBE_OUTER || join_type == TGPU_JOIN_FULL_OUTER;
    for (int64_t i = 0; i < n; i++) {
        int32_t pos = jp[i];
        bool produced = false;
        while (pos >= 0) {
            produced = true;
            if (count < capacity) { out_probe[count] = (int32_t)i; out_build[count] = pos; }
            count++;
            if (single_match) pos = -1;
            else pos = j->link_count ? j->links[pos] : -1;   // JoinHash.getNextJoinPosition :145-151
        }
        if (outer && !produced) {
            if (count < capacity) { out_probe[count] = (int32_t)i; out_build[count] = -1; }
            count++;
        }
    }
    return count;
}

double orc_join_probe_timed(const orc_join* j, const int64_t* probe_keys, int64_t n, int32_t threads, int32_t* out,
                            const int32_t* build_payload, int32_t* out_payload)
{
    // T probe drivers over 8192-row pages sharing one table; 3-phase batched probe of
    // BigintPagesHash.getAddressIndex(int[], Page) :184-268 (also the shape of DefaultPagesHash :204-282)
    const int64_t PAGE = 8192;
    int64_t pages = (n + PAGE - 1) / PAGE;
    auto t0 = std::chrono::steady_clock::now();
    std::vector<std::thread> pool;
    for (int32_t t = 0; t < threads; t++) {
        pool.emplace_back([=]() {
            std::vector<int32_t> hash_pos(PAGE), found_keys(PAGE), found(PAGE);
            for (int64_t p = t; p < pages; p += threads) {
                int64_t base = p * PAGE;
                int32_t cnt = (int32_t)std::min(PAGE, n - base);
                const int64_t* in = probe_keys + base;
                int32_t* res = out + base;
                for (int32_t i = 0; i < cnt; i++) hash_pos[i] = (int32_t)(murmur3((uint64_t)in[i]) & (uint64_t)j->mask);
                for (int32_t i = 0; i < cnt; i++) found_keys[i] = j->keys[hash_pos[i]];
                int32_t fc = 0;
                for (int32_t i = 0; i < cnt; i++) { res[i] = -1; if (found_keys[i] != -1) found[fc++] = i; }
                int32_t rc = 0;
                for (int32_t k = 0; k < fc; k++) {
                    int32_t idx = found[k];
                    if (j->values[found_keys[idx]] == in[idx]) res[idx] = found_keys[idx];
                    else found[rc++] = idx;
                }
                for (int32_t k = 0; k < rc; k++) {
                    int32_t idx = found[k];
                    int32_t pos = (hash_pos[idx] + 1) & j->mask;
                    while (j->keys[pos] != -1) {
                        if (j->values[j->keys[pos]] == in[idx]) { res[idx] = j->keys[pos]; break; }
                        pos = (pos + 1) & j->mask;
                    }
                }
                // PageJoiner.joinCurrentPosition :203-227 + LookupJoinPageBuilder.appendRow :89-97: one output row per
                // match, build-side column copied row by row (probe-side columns are views: :131-151)
                if (build_payload) {
                    int32_t* po = out_payload + base;
                    for (int32_t i = 0; i < cnt; i++) po[i] = res[i] >= 0 ? build_payload[res[i]] : 0;
                }
            }
        });
    }
    for (auto& th : pool) th.join();
    return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

// ------------------------------------------------------------------------------------------------
// Partitioned lookup source + persistent probe drivers: the stable CPU timing arm.
// Structure of a Trino task: the build side goes through a local hash exchange into P HashBuilderOperators
// (P = task.concurrency; partition = LocalPartitionGenerator.getPartition(rawHash),
// M/operator/exchange/LocalPartitionGenerator.java:76-80), each builds its own PagesHash over its own PagesIndex;
// T probe drivers share the PartitionedLookupSource (M/operator/join/unspilled/PartitionedLookupSource.java:149-186).
// ------------------------------------------------------------------------------------------------
namespace {

// a fixed set of worker threads; run(fn) executes fn(worker) on every worker and returns when all are done
// Memory placement of the CPU timing arm: pages are interleaved over the online NUMA nodes (set_mempolicy(MPOL_INTERLEAVE), a raw
// syscall: no libnuma in the image), for the calling thread - every pool worker and the thread that allocates the probe buffers call
// it - so that two runs of the arm do not land on different node mixes (run-to-run differences of 15 % were measured without it).
// Best effort: a kernel or cpuset that refuses leaves the default first-touch policy.
static void numa_interleave_this_thread()
{
#ifdef SYS_set_mempolicy
    unsigned long mask[16] = {0};
    int max_node = -1;
    if (FILE* f = fopen("/sys/devices/system/node/online", "r")) {
        char buf[256] = {0};
        if (fgets(buf, sizeof(buf), f)) {
            // "0-3" or "0,2-3"
            for (char* p = buf; *p;) {
                int a = (int)strtol(p, &p, 10), b = a;
                if (*p == '-') b = (int)strtol(p + 1, &p, 10);
                for (int n = a; n <= b && n < 1024; n++) { mask[n / 64] |= 1UL << (n % 64); if (n > max_node) max_node = n; }
                while (*p && (*p < '0' || *p > '9')) p++;
            }
        }
        fclose(f);
    }
    if (max_node >= 1) syscall(SYS_set_mempolicy, 3 /* MPOL_INTERLEAVE */, mask, (unsigned long)(max_node + 2));
#endif
}

struct WorkerPool {
    std::vector<std::thread> threads;
    std::mutex m;
    std::condition_variable cv_start, cv_done;
    std::function<void(int)> job;
    int64_t generation = 0;
    int pending = 0;
    bool stop = false;

    explicit WorkerPool(int n)
    {
        for (int t = 0; t < n; t++) threads.emplace_back([this, t]() { loop(t); });
    }
    ~WorkerPool()
    {
        { std::lock_guard<std::mutex> g(m); stop = true; generation++; }
        cv_start.notify_all();
        for (auto& th : threads) th.join();
    }
    void loop(int t)
    {
        numa_interleave_this_thread();
        int64_t seen = 0;
        while (true) {
            std::function<void(int)> fn;
            {
                std::unique_lock<std::mutex> g(m);
                cv_start.wait(g, [&]() { return generation != seen; });
                seen = generation;
                if (stop) return;
                fn = job;
            }
            fn(t);
            {
                std::lock_guard<std::mutex> g(m);
                if (--pending == 0) cv_done.notify_all();
            }
        }
    }
    void run(const std::function<void(int)>& fn)
    {
        std::unique_lock<std::mutex> g(m);
        job = fn;
        pending = (int)threads.size();
        generation++;
        cv_start.notify_all();
        cv_done.wait(g, [&]() { return pending == 0; });
    }
    int size() const { return (int)threads.size(); }
};

struct PJoinPart {
    bool bigint = true;                 // JoinHashSupplier.getPagesHashType :162-168: BigintPagesHash up to 2^20 positions, else DefaultPagesHash
    int32_t mask = 0;
    int64_t n = 0;
    std::vector<int32_t> keys;          // slot -> address index inside the partition, -1 empty
    std::vector<int64_t> values;        // address index -> key (BigintPagesHash.values / the key block of the partition's PagesIndex)
    std::vector<uint8_t> tags;          // DefaultPagesHash.positionToHashes
    std::vector<int32_t> payload;       // the partition's build output channel
    std::vector<int32_t> global_row;    // address index -> row of the unpartitioned build side (verification only)
};

}  // namespace

struct orc_pjoin {
    int32_t P = 1, shift = 1;
    std::vector<PJoinPart> parts;
    WorkerPool* pool = nullptr;
    ~orc_pjoin() { delete pool; }
};

orc_pjoin* orc_pjoin_build(const int64_t* build_keys, const int32_t* build_payload, int64_t n, int32_t partitions, int32_t threads, double* seconds_out)
{
    // partitions must be a power of two (LocalPartitionGenerator.java:43-47)
    orc_pjoin* j = new orc_pjoin();
    int32_t P = 1;
    while (P < partitions) P <<= 1;
    j->P = P;
    j->shift = __builtin_ctz((unsigned)P) + 1;            // PartitionedLookupSource.java:105-106
    j->parts.resize(P);
    j->pool = new WorkerPool(threads);
    const int T = threads;
    auto t0 = std::chrono::steady_clock::now();
    // local exchange: rows to partitions, stable (PartitioningExchanger.accept :58-103 appends positions in page order)
    std::vector<uint8_t> part_of((size_t)n);
    std::vector<std::vector<int64_t>> counts(T, std::vector<int64_t>(P, 0));
    const int64_t slice = (n + T - 1) / T;
    j->pool->run([&](int t) {
        int64_t lo = std::min<int64_t>(n, t * slice), hi = std::min<int64_t>(n, lo + slice);
        for (int64_t r = lo; r < hi; r++) {
            int32_t p = (int32_t)xxh64_long((int64_t)bitreverse64(hash_long(build_keys[r]))) & (P - 1);
            part_of[r] = (uint8_t)p;
            counts[t][p]++;
        }
    });
    std::vector<std::vector<int64_t>> start(T, std::vector<int64_t>(P, 0));
    for (int p = 0; p < P; p++) {
        int64_t run = 0;
        for (int t = 0; t < T; t++) { start[t][p] = run; run += counts[t][p]; }
        j->parts[p].n = run;
    }
    // every partition is allocated, first-touched and built by its own builder thread (one HashBuilderOperator per partition)
    std::vector<std::vector<int32_t>> rows(P);
    j->pool->run([&](int t) {
        for (int p = t; p < P; p += T) rows[p].assign((size_t)j->parts[p].n, 0);
    });
    j->pool->run([&](int t) {
        int64_t lo = std::min<int64_t>(n, t * slice), hi = std::min<int64_t>(n, lo + slice);
        std::vector<int64_t> at = start[t];
        for (int64_t r = lo; r < hi; r++) rows[part_of[r]][at[part_of[r]]++] = (int32_t)r;
    });
    j->pool->run([&](int t) {
        for (int p = t; p < P; p += T) {
            PJoinPart& part = j->parts[p];
            const int64_t m = part.n;
            part.bigint = m <= (1 << 20);
            int32_t hash_size = orc_join_hash_array_size(m);      // IncrementalLoadFactorHashArraySizeSupplier, multiplier 1
            part.mask = hash_size - 1;
            part.keys.assign((size_t)hash_size, -1);
            part.values.resize((size_t)m);
            part.payload.resize((size_t)m);
            part.global_row.resize((size_t)m);
            if (!part.bigint) part.tags.resize((size_t)m);
            for (int64_t a = 0; a < m; a++) {
                int64_t r = rows[p][a];
                int64_t value = build_keys[r];
                part.values[a] = value;
                part.payload[a] = build_payload ? build_payload[r] : 0;
                part.global_row[a] = (int32_t)r;
                uint64_t raw = hash_long(value);
                if (!part.bigint) part.tags[a] = (uint8_t)raw;
                // BigintPagesHash.insertValue :122-141 (slot = mix(key)) / DefaultPagesHash.insertValue :126-144 (slot = mix(rawHash)).
                // The timing workload has unique keys; a repeated key replaces the slot's address like the reference (links are
                // kept by the single-table oracle, orc_join_build, which is the one the parity tests check chains against).
                int32_t pos = (int32_t)(murmur3(part.bigint ? (uint64_t)value : raw) & (uint64_t)part.mask);
                while (part.keys[pos] != -1) {
                    if (part.values[part.keys[pos]] == value) break;
                    pos = (pos + 1) & part.mask;
                }
                part.keys[pos] = (int32_t)a;
            }
            std::vector<int32_t>().swap(rows[p]);
        }
    });
    if (seconds_out) *seconds_out = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    return j;
}

void orc_pjoin_destroy(orc_pjoin* j) { delete j; }
int32_t orc_pjoin_partitions(const orc_pjoin* j) { return j->P; }
int32_t orc_pjoin_threads(const orc_pjoin* j) { return j->pool->size(); }

// first touch of caller-allocated probe-side arrays by the worker that will use them: page p (8192 rows) belongs to worker
// p % T in orc_pjoin_probe, so its memory lands on that worker's NUMA node
void orc_pjoin_touch(orc_pjoin* j, void* base, int64_t bytes_per_row, int64_t n)
{
    const int64_t PAGE = 8192;
    const int64_t pages = (n + PAGE - 1) / PAGE;
    const int T = j->pool->size();
    j->pool->run([&](int t) {
        for (int64_t p = t; p < pages; p += T) {
            int64_t lo = p * PAGE, hi = std::min(n, lo + PAGE);
            memset((char*)base + lo * bytes_per_row, 0, (size_t)((hi - lo) * bytes_per_row));
        }
    });
}

double orc_pjoin_probe(orc_pjoin* j, const int64_t* probe_keys, int64_t n, int64_t* out_positions, int32_t* out_payload)
{
    const int64_t PAGE = 8192;
    const int64_t pages = (n + PAGE - 1) / PAGE;
    const int T = j->pool->size();
    const int P = j->P;
    const int shift = j->shift;
    auto t0 = std::chrono::steady_clock::now();
    j->pool->run([&](int t) {
        std::vector<int64_t> raw(PAGE);
        std::vector<int32_t> part(PAGE), hash_pos(PAGE), found_keys(PAGE), found(PAGE), list(PAGE), res(PAGE);
        std::vector<int32_t> pcount(P), pstart(P + 1);
        for (int64_t pg = t; pg < pages; pg += T) {
            const int64_t base = pg * PAGE;
            const int32_t cnt = (int32_t)std::min(PAGE, n - base);
            const int64_t* in = probe_keys + base;
            // PartitionedLookupSource.getJoinPosition(int[], Page, Page, long[]) :187-199 raw hashes, then :149-186
            for (int32_t i = 0; i < cnt; i++) raw[i] = (int64_t)hash_long(in[i]);
            std::fill(pcount.begin(), pcount.end(), 0);
            for (int32_t i = 0; i < cnt; i++) {
                int32_t p = (int32_t)xxh64_long((int64_t)bitreverse64((uint64_t)raw[i])) & (P - 1);
                part[i] = p;
                pcount[p]++;
            }
            pstart[0] = 0;
            for (int p = 0; p < P; p++) pstart[p + 1] = pstart[p] + pcount[p];
            std::fill(pcount.begin(), pcount.end(), 0);
            for (int32_t i = 0; i < cnt; i++) list[pstart[part[i]] + pcount[part[i]]++] = i;
            for (int p = 0; p < P; p++) {
                const PJoinPart& ps = j->parts[p];
                const int32_t* pos_list = list.data() + pstart[p];
                const int32_t m = pstart[p + 1] - pstart[p];
                if (m == 0) continue;
                // the partition's 3-phase batched getAddressIndex: BigintPagesHash.java:184-268 / DefaultPagesHash.java:193-282
                for (int32_t k = 0; k < m; k++) {
                    int32_t i = pos_list[k];
                    hash_pos[k] = (int32_t)(murmur3(ps.bigint ? (uint64_t)in[i] : (uint64_t)raw[i]) & (uint64_t)ps.mask);
                }
                for (int32_t k = 0; k < m; k++) found_keys[k] = ps.keys[hash_pos[k]];
                int32_t fc = 0;
                for (int32_t k = 0; k < m; k++) { res[pos_list[k]] = -1; if (found_keys[k] != -1) found[fc++] = k; }
                int32_t rc = 0;
                for (int32_t f = 0; f < fc; f++) {
                    int32_t k = found[f], i = pos_list[k], a = found_keys[k];
                    bool eq = (ps.bigint || ps.tags[a] == (uint8_t)raw[i]) && ps.values[a] == in[i];
                    if (eq) res[i] = a;
                    else found[rc++] = k;
                }
                for (int32_t f = 0; f < rc; f++) {
                    int32_t k = found[f], i = pos_list[k];
                    int32_t pos = (hash_pos[k] + 1) & ps.mask;
                    while (ps.keys[pos] != -1) {
                        int32_t a = ps.keys[pos];
                        if ((ps.bigint || ps.tags[a] == (uint8_t)raw[i]) && ps.values[a] == in[i]) { res[i] = a; break; }
                        pos = (pos + 1) & ps.mask;
                    }
                }
            }
            // encodePartitionedJoinPosition :259-262, then PageJoiner.joinCurrentPosition :203-227 -> PartitionedLookupSource.appendTo
            // :226-233 -> the partition's PagesIndex: one build output value copied per match
            int64_t* out = out_positions + base;
            for (int32_t i = 0; i < cnt; i++) out[i] = res[i] < 0 ? -1 : (((int64_t)res[i] << shift) | part[i]);
            if (out_payload) {
                int32_t* po = out_payload + base;
                for (int32_t i = 0; i < cnt; i++) po[i] = res[i] >= 0 ? j->parts[part[i]].payload[res[i]] : 0;
            }
        }
    });
    return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

// decodePartition / decodeJoinPosition :264-275, mapped back to rows of the unpartitioned build side
void orc_pjoin_decode(const orc_pjoin* j, const int64_t* positions, int64_t n, int32_t* out_rows)
{
    for (int64_t i = 0; i < n; i++) {
        if (positions[i] < 0) { out_rows[i] = -1; continue; }
        int32_t p = (int32_t)(positions[i] & (j->P - 1));
        out_rows[i] = j->parts[p].global_row[(size_t)(positions[i] >> j->shift)];
    }
}

// ------------------------------------------------------------------------------------------------
// PagePartitioner
// ------------------------------------------------------------------------------------------------
void orc_partition_ids(const tgpu_page* page, const int32_t* key_channels, int32_t num_keys, int32_t bucket_count,
                       const int32_t* b2p, int32_t* out)
{
    auto cols = views(page, key_channels, num_keys);
    for (int64_t i = 0; i < page->num_rows; i++) {
        int32_t bucket = process_raw_hash((int64_t)row_hash(cols, i), bucket_count);
        out[i] = b2p ? b2p[bucket] : bucket;
    }
}

void orc_partition_positions(const tgpu_page* page, const int32_t* key_channels, int32_t num_keys, int32_t bucket_count,
                             const int32_t* b2p, int32_t partition_count, int32_t null_channel,
                             int32_t replicates_any_row, int32_t* any_row_replicated,
                             int64_t* out_offsets, int32_t* out_positions)
{
    // PagePartitioner.partitionPage :133-162.  Row-wise (:229-271) and column-wise (:273-314) strategies append
    // rows to a partition in different orders only when nulls are replicated; we follow the strategy the reference picks.
    int64_t n = page->num_rows;
    std::vector<std::vector<int32_t>> lists(partition_count);
    if (n == 0) { for (int32_t p = 0; p <= partition_count; p++) out_offsets[p] = 0; return; }
    auto cols = views(page, key_channels, num_keys);
    auto part_of = [&](int64_t i) {
        int32_t bucket = process_raw_hash((int64_t)row_hash(cols, i), bucket_count);
        return b2p ? b2p[bucket] : bucket;
    };
    int64_t start = 0;
    if (partition_count == 1) {
        if (replicates_any_row && !*any_row_replicated) *any_row_replicated = 1;
        for (int64_t i = 0; i < n; i++) lists[0].push_back((int32_t)i);
    }
    else {
        if (replicates_any_row && !*any_row_replicated) {
            for (auto& l : lists) l.push_back(0);
            *any_row_replicated = 1;
            start = 1;
        }
        bool nullable = null_channel >= 0 && ColView(&page->columns[null_channel]).col->validity != nullptr;
        bool row_wise = n < (int64_t)partition_count * 2;   // COLUMNAR_STRATEGY_COEFFICIENT = 2 (:57)
        if (nullable) {
            ColView nc(&page->columns[null_channel]);
            if (row_wise) {
                for (int64_t i = start; i < n; i++) {
                    if (nc.is_null(i)) for (auto& l : lists) l.push_back((int32_t)i);
                    else lists[part_of(i)].push_back((int32_t)i);
                }
            }
            else {
                // partitionNullablePositions :401-422: null positions first (inserted at index startPosition), then the rest
                std::vector<int32_t> nulls, nonnull;
                for (int64_t i = start; i < n; i++) (nc.is_null(i) ? nulls : nonnull).push_back((int32_t)i);
                for (auto& l : lists) l.insert(l.begin() + std::min<size_t>(start, l.size()), nulls.begin(), nulls.end());
                for (int32_t i : nonnull) lists[part_of(i)].push_back(i);
            }
        }
        else {
            for (int64_t i = start; i < n; i++) lists[part_of(i)].push_back((int32_t)i);
        }
    }
    int64_t off = 0;
    for (int32_t p = 0; p < partition_count; p++) {
        out_offsets[p] = off;
        for (int32_t v : lists[p]) out_positions[off++] = v;
    }
    out_offsets[partition_count] = off;
}

// ------------------------------------------------------------------------------------------------
// Q1 pipeline
// ------------------------------------------------------------------------------------------------
namespace {
struct Q1Partial {
    orc_groupby* gbh;
    std::vector<int8_t> rf, ls;
    std::vector<double> s_qty, s_price, s_disc_price, s_charge, a_qty, a_price, a_disc;
    std::vector<int64_t> c_qty, c_price, c_disc, c_star;
    std::vector<uint8_t> nn;
    void ensure(int32_t groups)
    {
        size_t g = groups;
        if (s_qty.size() >= g) return;
        for (auto* v : {&s_qty, &s_price, &s_disc_price, &s_charge, &a_qty, &a_price, &a_disc}) v->resize(g, 0.0);
        for (auto* v : {&c_qty, &c_price, &c_disc, &c_star}) v->resize(g, 0);
        nn.resize(g * 4, 0);
        rf.resize(g); ls.resize(g);
    }
};
}  // namespace

double orc_q1_run(int64_t n, const int32_t* shipdate, const int8_t* returnflag, const int8_t* linestatus,
                  const double* quantity, const double* extendedprice, const double* discount, const double* tax,
                  int32_t cutoff, int32_t threads, orc_q1_result* out)
{
    const int64_t PAGE = 8192;     // PageProcessor.MAX_BATCH_SIZE, M/operator/project/PageProcessor.java:58
    int64_t pages = (n + PAGE - 1) / PAGE;
    std::vector<Q1Partial> partials(threads);
    auto t0 = std::chrono::steady_clock::now();
    std::vector<std::thread> pool;
    for (int32_t t = 0; t < threads; t++) {
        pool.emplace_back([&, t]() {
            Q1Partial& st = partials[t];
            st.gbh = orc_groupby_create(2, 16);
            std::vector<int32_t> sel(PAGE), gids(PAGE), offs(PAGE + 1);
            std::vector<int8_t> p_rf(PAGE), p_ls(PAGE);
            std::vector<double> p_qty(PAGE), p_price(PAGE), p_disc(PAGE), p_disc_price(PAGE), p_charge(PAGE);
            for (int32_t i = 0; i <= PAGE; i++) offs[i] = i;
            // contiguous slice per driver (a split), pages in order
            int64_t p_begin = pages * t / threads, p_end = pages * (t + 1) / threads;
            for (int64_t p = p_begin; p < p_end; p++) {
                int64_t base = p * PAGE;
                int32_t cnt = (int32_t)std::min(PAGE, n - base);
                // filter: ColumnarFilter.filterPositionsRange -> selected positions list
                int32_t m = 0;
                for (int32_t i = 0; i < cnt; i++) { sel[m] = i; m += shipdate[base + i] <= cutoff; }
                if (m == 0) continue;
                // projections, one loop each (PageProcessor.processBatch :302-336); unfused FP64
                for (int32_t k = 0; k < m; k++) p_rf[k] = returnflag[base + sel[k]];
                for (int32_t k = 0; k < m; k++) p_ls[k] = linestatus[base + sel[k]];
                for (int32_t k = 0; k < m; k++) p_qty[k] = quantity[base + sel[k]];
                for (int32_t k = 0; k < m; k++) p_price[k] = extendedprice[base + sel[k]];
                for (int32_t k = 0; k < m; k++) p_disc[k] = discount[base + sel[k]];
                for (int32_t k = 0; k < m; k++) p_disc_price[k] = extendedprice[base + sel[k]] * (1.0 - discount[base + sel[k]]);
                for (int32_t k = 0; k < m; k++) p_charge[k] = extendedprice[base + sel[k]] * (1.0 - discount[base + sel[k]]) * (1.0 + tax[base + sel[k]]);
                // GroupByHash over two VARCHAR(1) keys -> FlatGroupByHash
                tgpu_column kc[2] = {};
                kc[0].type = TGPU_UTF8; kc[0].length = m; kc[0].data = p_rf.data(); kc[0].offsets = offs.data();
                kc[1].type = TGPU_UTF8; kc[1].length = m; kc[1].data = p_ls.data(); kc[1].offsets = offs.data();
                tgpu_page kp = {2, 0, m, kc};
                int32_t ch[2] = {0, 1};
                int32_t before = orc_groupby_group_count(st.gbh);
                orc_groupby_get_group_ids(st.gbh, &kp, ch, 2, gids.data());
                int32_t groups = orc_groupby_group_count(st.gbh);
                st.ensure(groups);
                if (groups > before)
                    for (int32_t k = 0; k < m; k++) { st.rf[gids[k]] = p_rf[k]; st.ls[gids[k]] = p_ls[k]; }
                // one pass per aggregate (GroupedAggregator.processPage :77-101)
                orc_agg_sum_double(gids.data(), m, p_qty.data(), nullptr, nullptr, st.s_qty.data(), st.nn.data());
                orc_agg_sum_double(gids.data(), m, p_price.data(), nullptr, nullptr, st.s_price.data(), st.nn.data() + groups);
                orc_agg_sum_double(gids.data(), m, p_disc_price.data(), nullptr, nullptr, st.s_disc_price.data(), st.nn.data() + 2 * groups);
                orc_agg_sum_double(gids.data(), m, p_charge.data(), nullptr, nullptr, st.s_charge.data(), st.nn.data() + 3 * groups);
                orc_agg_avg_double(gids.data(), m, p_qty.data(), nullptr, nullptr, st.a_qty.data(), st.c_qty.data());
                orc_agg_avg_double(gids.data(), m, p_price.data(), nullptr, nullptr, st.a_price.data(), st.c_price.data());
                orc_agg_avg_double(gids.data(), m, p_disc.data(), nullptr, nullptr, st.a_disc.data(), st.c_disc.data());
                orc_agg_count(gids.data(), m, nullptr, nullptr, st.c_star.data());
            }
        });
    }
    for (auto& th : pool) th.join();
    // FINAL step: merge partial states in driver order (combine functions)
    orc_q1_result r;
    memset(&r, 0, sizeof(r));
    int64_t c_qty[16] = {0}, c_price[16] = {0}, c_disc[16] = {0};
    for (int32_t t = 0; t < threads; t++) {
        Q1Partial& st = partials[t];
        int32_t groups = orc_groupby_group_count(st.gbh);
        for (int32_t g = 0; g < groups; g++) {
            int32_t f = -1;
            for (int32_t k = 0; k < r.num_groups; k++) if (r.returnflag[k] == st.rf[g] && r.linestatus[k] == st.ls[g]) f = k;
            if (f < 0) {
                if (r.num_groups >= 16) continue;
                f = r.num_groups++;
                r.returnflag[f] = st.rf[g];
                r.linestatus[f] = st.ls[g];
            }
            r.sum_qty[f] += st.s_qty[g];
            r.sum_base_price[f] += st.s_price[g];
            r.sum_disc_price[f] += st.s_disc_price[g];
            r.sum_charge[f] += st.s_charge[g];
            r.avg_qty[f] += st.a_qty[g]; c_qty[f] += st.c_qty[g];
            r.avg_price[f] += st.a_price[g]; c_price[f] += st.c_price[g];
            r.avg_disc[f] += st.a_disc[g]; c_disc[f] += st.c_disc[g];
            r.count_order[f] += st.c_star[g];
        }
        orc_groupby_destroy(st.gbh);
    }
    for (int32_t k = 0; k < r.num_groups; k++) {
        r.avg_qty[k] = r.avg_qty[k] / (double)c_qty[k];
        r.avg_price[k] = r.avg_price[k] / (double)c_price[k];
        r.avg_disc[k] = r.avg_disc[k] / (double)c_disc[k];
    }
    double secs = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    *out = r;
    return secs;
}

// ------------------------------------------------------------------------------------------------
// synthetic generators — MUST stay identical to trino_b200/csrc/synth.cuh
// ------------------------------------------------------------------------------------------------
uint64_t orc_splitmix64(uint64_t x)
{
    x += 0x9E3779B97F4A7C15ULL;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ULL;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBULL;
    return x ^ (x >> 31);
}

// seeded permutation of [0, n): 4-round Feistel over 2*hb bits with cycle walking
static inline uint64_t feistel_perm(uint64_t i, uint64_t n, uint64_t seed)
{
    int bits = 1;
    while ((1ULL << bits) < n) bits++;
    int hb = (bits + 1) / 2;
    uint64_t hm = (1ULL << hb) - 1;
    uint64_t x = i;
    do {
        uint64_t l = x >> hb, r = x & hm;
        for (int round = 0; round < 4; round++) {
            uint64_t f = orc_splitmix64(r ^ (seed + 0x1000003ULL * (uint64_t)round)) & hm;
            uint64_t nl = r, nr = l ^ f;
            l = nl; r = nr;
        }
        x = (l << hb) | r;
    } while (x >= n);
    return x;
}

static inline int64_t order_key(int64_t i) { return (i / 8) * 32 + (i % 8) + 1; }   // TPC-H sparse order keys

void orc_synth_orders_keys(int64_t n_total, int64_t first, int64_t count, uint64_t seed, int32_t shuffle, int64_t* out)
{
    // rows [first, first+count) of the n_total-row orders table; row j holds order_key(perm(j))
    for (int64_t j = 0; j < count; j++) {
        int64_t i = shuffle ? (int64_t)feistel_perm((uint64_t)(first + j), (uint64_t)n_total, seed) : first + j;
        out[j] = order_key(i);
    }
}

// lineitems per order i: 1 + ((i + i/7) % 7): every block of 7 orders has exactly 28 lineitems
static inline int64_t lineitem_order_index(int64_t r)
{
    int64_t b = r / 28, w = r % 28;
    int64_t acc = 0;
    for (int64_t jj = 0; jj < 7; jj++) {
        int64_t c = 1 + ((jj + b) % 7);
        if (w < acc + c) return b * 7 + jj;
        acc += c;
    }
    return b * 7 + 6;
}

int64_t orc_synth_lineitem_rows(int64_t n_orders)
{
    int64_t full = n_orders / 7, rem = n_orders % 7;
    int64_t rows = full * 28;
    for (int64_t jj = 0; jj < rem; jj++) rows += 1 + ((jj + full) % 7);
    return rows;
}

void orc_synth_lineitem_keys(int64_t n_orders, int64_t first, int64_t count, uint64_t seed, int32_t shuffle, int64_t* out)
{
    // rows [first, first+count) of lineitem in order-key order (TPC-H clustering); shuffle != 0 permutes the rows
    int64_t rows = orc_synth_lineitem_rows(n_orders);
    for (int64_t k = 0; k < count; k++) {
        int64_t r = shuffle ? (int64_t)feistel_perm((uint64_t)(first + k), (uint64_t)rows, seed) : first + k;
        out[k] = order_key(lineitem_order_index(r));
    }
}

void orc_synth_lineitem_q1(int64_t n, int64_t first, uint64_t seed, int32_t* shipdate, int8_t* returnflag, int8_t* linestatus,
                           double* quantity, double* extendedprice, double* discount, double* tax)
{
    for (int64_t k = 0; k < n; k++) {
        uint64_t x = orc_splitmix64(seed ^ (uint64_t)(first + k));
        uint64_t y = orc_splitmix64(x);
        int32_t sd = 8036 + (int32_t)(x % 2556);                 // 1992-01-02 .. 1998-12-01
        int32_t receipt = sd + 1 + (int32_t)((y >> 40) % 30);
        int64_t qty = 1 + (int64_t)((x >> 12) % 50);
        int64_t retail_cents = 90000 + (int64_t)(y % 20001);
        shipdate[k] = sd;
        linestatus[k] = sd > 9298 ? 'O' : 'F';                    // 1995-06-17
        returnflag[k] = receipt <= 9298 ? (((y >> 50) & 1) ? 'R' : 'A') : 'N';
        quantity[k] = (double)qty;
        extendedprice[k] = (double)(qty * retail_cents) / 100.0;
        discount[k] = (double)((y >> 20) % 11) / 100.0;
        tax[k] = (double)((y >> 30) % 9) / 100.0;
    }
}

// o_custkey of order index i (same formula as the device generator, synth.cu)
static inline int64_t order_custkey(int64_t i, int64_t n_customers, uint64_t seed)
{
    uint64_t with_orders = (uint64_t)(n_customers - n_customers / 3);
    uint64_t j = orc_splitmix64(seed ^ (0x9E3779B97F4A7C15ULL * (uint64_t)(i + 1))) % with_orders;
    return (int64_t)((j / 2) * 3 + (j % 2) + 1);
}

void orc_synth_orders_custkeys(int64_t n_total, int64_t first, int64_t count, uint64_t seed, int32_t shuffle, int64_t n_customers, uint64_t cust_seed, int64_t* out)
{
    for (int64_t j = 0; j < count; j++) {
        int64_t i = shuffle ? (int64_t)feistel_perm((uint64_t)(first + j), (uint64_t)n_total, seed) : first + j;
        out[j] = order_custkey(i, n_customers, cust_seed);
    }
}

int64_t orc_synth_store_sales(int64_t n, int64_t first, uint64_t seed, int64_t* date_sk, int64_t* item_sk, int64_t* customer_sk, uint8_t* customer_valid,
                              int64_t* store_sk, uint8_t* store_valid, double* net_paid)
{
    int64_t both = 0;
    memset(customer_valid, 0, (size_t)((n + 7) / 8));
    memset(store_valid, 0, (size_t)((n + 7) / 8));
    for (int64_t j = 0; j < n; j++) {
        uint64_t x = orc_splitmix64(seed ^ (uint64_t)(first + j));
        uint64_t y = orc_splitmix64(x);
        bool cn = ((x >> 40) % 1000) < 45, sn = ((y >> 48) % 1000) < 45;
        date_sk[j] = 2450816 + (int64_t)(x % 1823);
        item_sk[j] = 1 + (int64_t)((x >> 16) % 300000);
        customer_sk[j] = cn ? 0 : 1 + (int64_t)(y % 12000000);
        store_sk[j] = sn ? 0 : 1 + (int64_t)((y >> 32) % 1002);
        net_paid[j] = (double)((x >> 8) % 2000000) / 100.0;
        if (!cn) customer_valid[j >> 3] |= (uint8_t)(1u << (j & 7));
        if (!sn) store_valid[j >> 3] |= (uint8_t)(1u << (j & 7));
        both += (!cn && !sn) ? 1 : 0;
    }
    return both;
}

int32_t orc_hardware_threads(void)
{
    unsigned n = std::thread::hardware_concurrency();
    return n ? (int32_t)n : 1;
}

}  // extern "C"


// ---- HashSemiJoinOperator -------------------------------------------------------------------------------------------------
// M/operator/HashSemiJoinOperator.java:181-199; the set is SetBuilderOperator's ChannelSet (FlatSet.java:120-153)
extern "C" void orc_semi_join_bigint(const int64_t* set_values, const uint8_t* set_validity, int64_t set_rows, const int64_t* probe, const uint8_t* probe_validity,
                                     int64_t probe_rows, int8_t* out_value, uint8_t* out_null)
{
    std::unordered_set<int64_t> set;
    bool has_null = false;
    for (int64_t i = 0; i < set_rows; i++) {
        bool valid = !set_validity || ((set_validity[i >> 3] >> (i & 7)) & 1);
        if (!valid) has_null = true;          // FlatSet.add :146-153
        else set.insert(set_values[i]);
    }
    const bool empty = set.empty() && !has_null;   // FlatSet.size :120-123 counts the NULL
    for (int64_t i = 0; i < probe_rows; i++) {
        bool valid = !probe_validity || ((probe_validity[i >> 3] >> (i & 7)) & 1);
        if (!valid) {
            out_value[i] = 0;
            out_null[i] = empty ? 0 : 1;      // :184-190
            continue;
        }
        bool contains = set.count(probe[i]) != 0;
        if (!contains && has_null) { out_value[i] = 0; out_null[i] = 1; }   // :193-195
        else { out_value[i] = contains ? 1 : 0; out_null[i] = 0; }
    }
}

// the same operator over a DOUBLE (kind 1: 8-byte raw bits) or REAL (kind 2: 4-byte raw bits) channel: the ChannelSet's FlatSet compares with
// IDENTICAL (M/operator/FlatSet.java:54,374; S/type/DoubleType.java:218-229, S/type/RealType.java:172-185): every NaN is one member, -0.0 and +0.0 are one
extern "C" void orc_semi_join_float(int32_t kind, const void* set_values, const uint8_t* set_validity, int64_t set_rows, const void* probe, const uint8_t* probe_validity,
                                    int64_t probe_rows, int8_t* out_value, uint8_t* out_null)
{
    auto canonical = [kind](const void* base, int64_t i) -> uint64_t {
        if (kind == 1) {
            uint64_t u = ((const uint64_t*)base)[i];
            if ((u << 1) == 0) return 0;
            if ((u & 0x7FFFFFFFFFFFFFFFULL) > 0x7FF0000000000000ULL) return 0x7FF8000000000000ULL;
            return u;
        }
        uint32_t u = ((const uint32_t*)base)[i];
        if ((u << 1) == 0) return 0;
        if ((u & 0x7FFFFFFFu) > 0x7F800000u) return 0x7FC00000u;
        return u;
    };
    std::unordered_set<uint64_t> set;
    bool has_null = false;
    for (int64_t i = 0; i < set_rows; i++) {
        bool valid = !set_validity || ((set_validity[i >> 3] >> (i & 7)) & 1);
        if (!valid) has_null = true;
        else set.insert(canonical(set_values, i));
    }
    const bool empty = set.empty() && !has_null;
    for (int64_t i = 0; i < probe_rows; i++) {
        bool valid = !probe_validity || ((probe_validity[i >> 3] >> (i & 7)) & 1);
        if (!valid) {
            out_value[i] = 0;
            out_null[i] = empty ? 0 : 1;
            continue;
        }
        bool contains = set.count(canonical(probe, i)) != 0;
        if (!contains && has_null) { out_value[i] = 0; out_null[i] = 1; }
        else { out_value[i] = contains ? 1 : 0; out_null[i] = 0; }
    }
}
