// partition.cu — PagePartitioner / PartitionedOutputOperator for sm_90a, and the NCCL all-to-all exchange.
//
// Reference semantics reproduced:
//   - partition id = bucketToPartition[ processRawHash(rowHash, bucketCount) ] with rowHash folded as
//     h = 31*h + typeHash(col) and NULL -> 0 (M/operator/HashGenerator.java:25-46,
//     M/operator/InterpretedHashGenerator.java:102-110, M/operator/BucketPartitionFunction.java:45-64)
//   - per-partition row order of PagePartitioner.partitionPage (M/operator/output/PagePartitioner.java:133-162):
//       column-wise strategy (:273-314, positions >= 2 x partitions): [row 0 once when replicatesAnyRow],
//       then every NULL-channel row (replicated to all partitions, :401-416), then the partition's own rows,
//       each list ascending; row-wise strategy (:229-271): plain ascending row order with replicated rows
//       interleaved.  A single partition takes the whole page.
//   - output buffers are flushed per input page here (the reference flushes at 1 MB / 32768 rows,
//     PositionsAppenderPageBuilder.java:34,132-142); values per partition and their order are identical.
//
// Device paths.  The common one is the multi-split (multisplit.cuh, DESIGN.md §3.6): a histogram pass, an offsets pass and one
// stable scatter move every fixed-width column of up to 8 bytes straight to its partition-contiguous place, which in the exchanges
// is the send buffer or the destination's arena.  Replicated rows (nullChannel, replicatesAnyRow), variable-width and 16-byte
// columns, more than 64 partitions or too many columns take the sort + compose path: one kernel computes row hash -> partition id,
// a stable radix sort of (partition, row) pairs yields the per-partition position lists, and one gather per column writes the
// partition's page.
#include <dlfcn.h>

#include <algorithm>
#include <chrono>

#include "multisplit.cuh"

namespace {

using namespace tg;

// partition id per row; rows whose null_channel is NULL get id == partition_count (replicated later)
__global__ void __launch_bounds__(256) partition_ids_kernel(KeyCols keys, int64_t n, int32_t bucket_count, const int32_t* __restrict__ bucket_to_partition,
                                                           ColRef null_col, int32_t has_null_col, int32_t partition_count, int32_t* __restrict__ out)
{
    int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; row < n; row += stride) {
        if (has_null_col && !tg_valid(null_col.validity, row)) { out[row] = partition_count; continue; }
        uint64_t h = 0;
        for (int c = 0; c < keys.count; c++) h = combine_hash(h, type_hash(keys, c, row));
        int32_t bucket = process_raw_hash(h, bucket_count);
        out[row] = bucket_to_partition ? bucket_to_partition[bucket] : bucket;
    }
}

// first index of every partition id in the sorted id array (P+2 boundaries)
__global__ void partition_bounds_kernel(const int32_t* __restrict__ sorted_ids, int64_t n, int32_t nbounds, long long* __restrict__ bounds)
{
    int32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= nbounds) return;
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        int64_t mid = (lo + hi) >> 1;
        if (sorted_ids[mid] < p) lo = mid + 1;
        else hi = mid;
    }
    bounds[p] = lo;
}

// final gather index of the column-wise strategy: per partition [any-row] + nulls + own rows
__global__ void partition_compose_kernel(const int32_t* __restrict__ sorted_rows, const long long* __restrict__ bounds, int32_t partition_count,
                                         int32_t prepend_row0, const long long* __restrict__ out_offsets, int32_t* __restrict__ out)
{
    int32_t p = blockIdx.y;
    long long nulls_begin = bounds[partition_count], nulls_end = bounds[partition_count + 1];
    long long own_begin = bounds[p], own_end = bounds[p + 1];
    long long n_nulls = nulls_end - nulls_begin, n_own = own_end - own_begin;
    long long total = prepend_row0 + n_nulls + n_own;
    long long base = out_offsets[p];
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < total; i += stride) {
        int32_t v;
        if (i < prepend_row0) v = 0;
        else if (i < prepend_row0 + n_nulls) v = sorted_rows[nulls_begin + (i - prepend_row0)];
        else v = sorted_rows[own_begin + (i - prepend_row0 - n_nulls)];
        out[base + i] = v;
    }
}

// row-wise strategy (tiny pages): one thread per partition walks the rows in order
__global__ void partition_rowwise_kernel(const int32_t* __restrict__ ids, int64_t n, int32_t partition_count, int32_t start_row, int32_t prepend_row0,
                                         long long* __restrict__ counts, int32_t* __restrict__ out, int64_t out_stride)
{
    int32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= partition_count) return;
    long long c = 0;
    int32_t* o = out + (int64_t)p * out_stride;
    if (prepend_row0) o[c++] = 0;
    for (int64_t i = start_row; i < n; i++) {
        int32_t id = ids[i];
        if (id == partition_count || id == p) o[c++] = (int32_t)i;
    }
    counts[p] = c;
}

// type hash of the single position of a HOST column (the value of a partition constant); same functions as the device's type_hash
int host_type_hash(tgpu_ctx* ctx, const tgpu_column& c, uint64_t* out)
{
    if (c.length != 1) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "a partition constant holds one position, not %lld", (long long)c.length);
    if (c.validity) {
        bool is_null = (c.flags & TGPU_COL_NULLS_BYTEMAP) ? c.validity[0] != 0 : (c.validity[0] & 1) == 0;
        if (is_null) { *out = 0; return TGPU_OK; }
    }
    if (!c.data && c.type != TGPU_UTF8) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "partition constant without a value");
    switch (c.type) {
        case TGPU_INT64: *out = hash_long(*(const int64_t*)c.data); return TGPU_OK;
        case TGPU_INT32: *out = hash_long(*(const int32_t*)c.data); return TGPU_OK;
        case TGPU_INT16: *out = hash_long(*(const int16_t*)c.data); return TGPU_OK;
        case TGPU_INT8: *out = hash_long(*(const int8_t*)c.data); return TGPU_OK;
        case TGPU_FLOAT64: *out = hash_double_bits(*(const int64_t*)c.data); return TGPU_OK;
        case TGPU_FLOAT32: *out = hash_real_bits(*(const int32_t*)c.data); return TGPU_OK;
        case TGPU_INT128: *out = hash_int128(((const int64_t*)c.data)[0], ((const int64_t*)c.data)[1]); return TGPU_OK;
        case TGPU_UTF8:
            if (!c.offsets) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "variable-width partition constant without offsets");
            *out = xxh64_bytes((const uint8_t*)c.data + c.offsets[0], c.offsets[1] - c.offsets[0]);
            return TGPU_OK;
        default: return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "partition constant of type %d", c.type);
    }
}

// One lane of a multi-split: the values of column `col`, or (`nulls`) its NULL bytes, 1 = NULL.  `elem` is the scatter's
// XchgCols.elem: the value width, 0 for a NULL-byte lane.  A NULL-byte lane without `src` (the page has no validity buffer) writes
// all zeros: an exchange carries it when another rank's page of the same column has NULLs.
struct XchgLane {
    int col;
    int32_t type;
    int elem;
    bool nulls;
    const void* src;
};

size_t lane_bytes(const XchgLane& lane) { return lane.elem ? (size_t)lane.elem : 1; }

// a value lane per column, followed by a NULL-byte lane where null_lane[c]
std::vector<XchgLane> xchg_lanes(const DevPage& in, const std::vector<bool>& null_lane)
{
    std::vector<XchgLane> lanes;
    for (int c = 0; c < (int)in.cols.size(); c++) {
        lanes.push_back(XchgLane{c, in.cols[c].type, in.cols[c].elem_size(), false, in.cols[c].data});
        if (null_lane[c]) lanes.push_back(XchgLane{c, in.cols[c].type, 0, true, in.cols[c].validity});
    }
    return lanes;
}

// the scatter's lane table; h_dst[lane * P + partition] is where the lane's rows of that partition start (uploaded to *d_dst)
int xchg_cols(tgpu_ctx* ctx, const std::vector<XchgLane>& lanes, const std::vector<char*>& h_dst, DevBuf* d_dst, XchgCols* xc)
{
    TG_TRY(d_dst->alloc(ctx, h_dst.size() * sizeof(char*)));
    TG_CUDA(ctx, cudaMemcpyAsync(d_dst->p, h_dst.data(), h_dst.size() * sizeof(char*), cudaMemcpyHostToDevice, ctx->stream));
    memset(xc, 0, sizeof(*xc));
    xc->count = (int32_t)lanes.size();
    for (size_t l = 0; l < lanes.size(); l++) { xc->elem[l] = lanes[l].elem; xc->src[l] = lanes[l].src; }
    xc->dst = d_dst->as<char*>();
    return TGPU_OK;
}

// The page of `rows` rows whose lane l starts at base[l]: value lanes become its columns, owning owner[l] when `owner` is given and
// aliasing memory they do not own otherwise; NULL-byte lanes are packed into validity bitmaps.  A page of 0 rows has no validity.
int xchg_page(tgpu_ctx* ctx, const std::vector<XchgLane>& lanes, const std::vector<char*>& base, int64_t rows,
              const std::vector<std::shared_ptr<DevBuf>>* owner, DevPage* out)
{
    out->rows = rows;
    out->cols.resize((size_t)std::count_if(lanes.begin(), lanes.end(), [](const XchgLane& l) { return !l.nulls; }));
    for (size_t l = 0; l < lanes.size(); l++) {
        DevColumn& dst = out->cols[lanes[l].col];
        if (!lanes[l].nulls) {
            dst.type = lanes[l].type;
            dst.length = rows;
            dst.data = base[l];
            if (owner) dst.own_data = (*owner)[l];
        }
        else if (rows > 0) {
            tgpu_column bytemap_col;
            memset(&bytemap_col, 0, sizeof(bytemap_col));
            bytemap_col.type = TGPU_INT8;
            bytemap_col.flags = TGPU_COL_NULLS_BYTEMAP;
            bytemap_col.length = rows;
            bytemap_col.data = base[l];
            bytemap_col.validity = (const uint8_t*)base[l];
            DevColumn packed;
            TG_TRY(tg_ingest_column(ctx, &bytemap_col, true, &packed));
            dst.own_validity = packed.own_validity;
            dst.validity = packed.validity;
        }
    }
    return TGPU_OK;
}

// TGPU_TRACE=1: mark() synchronises and prints the wall time since the previous mark (diagnostics only)
struct PhaseTrace {
    tgpu_ctx* ctx;
    std::string who;
    bool on = getenv("TGPU_TRACE") != nullptr;
    std::chrono::steady_clock::time_point last = std::chrono::steady_clock::now();

    void mark(const char* what)
    {
        if (!on) return;
        cudaStreamSynchronize(ctx->stream);
        auto now = std::chrono::steady_clock::now();
        fprintf(stderr, "[tgpu %s] %-22s %8.3f ms\n", who.c_str(), what, std::chrono::duration<double, std::milli>(now - last).count());
        last = now;
    }
};

struct PartitionOp : tgpu_op {
    std::vector<int32_t> key_channels;
    std::vector<uint64_t> constant_hash;    // per partition channel; read where key_channels[c] < 0
    int32_t bucket_count = 1, partition_count = 1;
    std::vector<int32_t> bucket_to_partition;
    DevBuf d_b2p;
    int32_t null_channel = -1;
    bool replicates_any_row = false, any_row_replicated = false;
    std::vector<OwnedPage*> pending;
    size_t next_out = 0;
    int32_t last_partition = -1;
    bool finishing = false;

    explicit PartitionOp(tgpu_ctx* c) : tgpu_op(c) {}
    ~PartitionOp() override { for (size_t i = next_out; i < pending.size(); i++) delete pending[i]; }

    bool needs_input() override { return !finishing && next_out >= pending.size(); }

    int key_cols(const DevPage& in, KeyCols* k)
    {
        memset(k, 0, sizeof(*k));
        if (key_channels.size() > 8) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "more than 8 partition channels");
        k->count = (int32_t)key_channels.size();
        for (int c = 0; c < k->count; c++) {
            int ch = key_channels[c];
            if (ch < 0) { k->is_const[c] = 1; k->const_hash[c] = constant_hash[c]; continue; }
            if (ch >= (int)in.cols.size()) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "partition channel %d out of range", ch);
            key_cols_set(k, c, in.cols[ch]);
        }
        return TGPU_OK;
    }

    // partition id per row into d_ids (int32[n]); NULL-channel rows get partition_count
    int compute_ids(const DevPage& in, int32_t* d_ids, bool use_null_channel)
    {
        KeyCols k;
        TG_TRY(key_cols(in, &k));
        ColRef nullcol;
        memset(&nullcol, 0, sizeof(nullcol));
        int has_null = 0;
        if (use_null_channel && null_channel >= 0) {
            if (null_channel >= (int)in.cols.size()) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "null channel out of range");
            if (in.cols[null_channel].validity) { nullcol = tg_colref(in.cols[null_channel]); has_null = 1; }
        }
        TG_LAUNCH(ctx, partition_ids_kernel, tg_grid(ctx, in.rows, 256, 8), 256, 0, k, in.rows, bucket_count,
                  bucket_to_partition.empty() ? nullptr : d_b2p.as<int32_t>(), nullcol, has_null, partition_count, d_ids);
        return TGPU_OK;
    }

    // stable sort of rows by partition id: sorted row list + P+2 boundaries (bounds[P]..bounds[P+1] = NULL-channel rows)
    int sort_rows(const int32_t* d_ids, int64_t n, DevBuf* sorted_rows, DevBuf* bounds)
    {
        DevBuf rows_in, ids_out;
        TG_TRY(rows_in.alloc(ctx, (size_t)n * 4));
        TG_TRY(ids_out.alloc(ctx, (size_t)n * 4));
        TG_TRY(sorted_rows->alloc(ctx, (size_t)n * 4));
        TG_TRY(bounds->alloc(ctx, (size_t)(partition_count + 2) * 8));
        TG_TRY(tg_iota(ctx, rows_in.as<int32_t>(), n));
        int bits = 1;
        while ((1 << bits) <= partition_count) bits++;
        TG_TRY(tg_sort_pairs(ctx, d_ids, ids_out.as<int32_t>(), rows_in.as<int32_t>(), sorted_rows->as<int32_t>(), (int)n, 0, bits));
        int nb = partition_count + 2;
        TG_LAUNCH(ctx, partition_bounds_kernel, (nb + 127) / 128, 128, 0, ids_out.as<int32_t>(), n, nb, bounds->as<long long>());
        return TGPU_OK;
    }

    int add_input(const tgpu_page* page) override
    {
        for (size_t i = next_out; i < pending.size(); i++) delete pending[i];   // pages the caller never took
        pending.clear();
        next_out = 0;
        int64_t n = page->num_rows;
        if (n == 0) return TGPU_OK;   // PagePartitioner.partitionPage :135-137
        if (n > (int64_t)INT32_MAX) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "page has more than 2^31-1 positions");
        DevPage in;
        TG_TRY(tg_ingest_page(ctx, page, &in));
        const int P = partition_count;
        if (P == 1) {
            // single output partition: the whole page (:141-148)
            if (replicates_any_row && !any_row_replicated) any_row_replicated = true;
            OwnedPage* o = tg_make_owned_page(std::move(in));
            o->partition = 0;
            pending.push_back(o);
            return TGPU_OK;
        }
        int prepend = 0, start_row = 0;
        if (replicates_any_row && !any_row_replicated) { prepend = 1; start_row = 1; any_row_replicated = true; }
        bool row_wise = n < (int64_t)P * 2;   // COLUMNAR_STRATEGY_COEFFICIENT (:57,149)
        if (!row_wise && prepend == 0 && multisplit_applies(in)) return add_input_multisplit(in);
        DevBuf ids;
        TG_TRY(ids.alloc(ctx, (size_t)n * 4));
        TG_TRY(compute_ids(in, ids.as<int32_t>(), true));
        std::vector<long long> h_off(P + 1, 0);
        DevBuf gather_idx;
        int64_t idx_stride = 0;
        if (row_wise) {
            DevBuf counts;
            TG_TRY(counts.alloc(ctx, (size_t)P * 8));
            idx_stride = n + 1;
            TG_TRY(gather_idx.alloc(ctx, (size_t)P * idx_stride * 4));
            TG_LAUNCH(ctx, partition_rowwise_kernel, (P + 63) / 64, 64, 0, ids.as<int32_t>(), n, P, start_row, prepend, counts.as<long long>(),
                      gather_idx.as<int32_t>(), idx_stride);
            std::vector<long long> h_counts(P);
            TG_CUDA(ctx, cudaMemcpyAsync(h_counts.data(), counts.p, (size_t)P * 8, cudaMemcpyDeviceToHost, ctx->stream));
            TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
            for (int p = 0; p < P; p++) {
                if (h_counts[p] == 0) continue;
                TG_TRY(emit(in, gather_idx.as<int32_t>() + (int64_t)p * idx_stride, h_counts[p], p));
            }
            return TGPU_OK;
        }
        // column-wise: rows [start_row, n) sorted by partition, NULL-channel rows in bucket P
        DevBuf sorted_rows, bounds;
        TG_TRY(sort_rows(ids.as<int32_t>() + start_row, n - start_row, &sorted_rows, &bounds));
        std::vector<long long> h_bounds(P + 2);
        TG_CUDA(ctx, cudaMemcpyAsync(h_bounds.data(), bounds.p, (size_t)(P + 2) * 8, cudaMemcpyDeviceToHost, ctx->stream));
        TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        long long n_nulls = h_bounds[P + 1] - h_bounds[P];
        if (start_row == 0 && n_nulls == 0) {
            // common case: the sorted row list already is the per-partition gather index
            for (int p = 0; p < P; p++) {
                long long cnt = h_bounds[p + 1] - h_bounds[p];
                if (cnt == 0) continue;
                TG_TRY(emit(in, sorted_rows.as<int32_t>() + h_bounds[p], cnt, p));
            }
            return TGPU_OK;
        }
        // sorted rows are relative to start_row: shift back while composing
        long long total = 0;
        for (int p = 0; p < P; p++) { h_off[p] = total; total += prepend + n_nulls + (h_bounds[p + 1] - h_bounds[p]); }
        h_off[P] = total;
        DevBuf d_off, shifted;
        TG_TRY(d_off.alloc(ctx, (size_t)(P + 1) * 8));
        TG_CUDA(ctx, cudaMemcpyAsync(d_off.p, h_off.data(), (size_t)(P + 1) * 8, cudaMemcpyHostToDevice, ctx->stream));
        TG_TRY(gather_idx.alloc(ctx, (size_t)total * 4));
        const int32_t* rows_ptr = sorted_rows.as<int32_t>();
        if (start_row) {
            TG_TRY(shifted.alloc(ctx, (size_t)(n - start_row) * 4));
            TG_TRY(tg_add_i32(ctx, sorted_rows.as<int32_t>(), n - start_row, start_row, shifted.as<int32_t>()));
            rows_ptr = shifted.as<int32_t>();
        }
        dim3 grid((unsigned)std::max<int64_t>(1, std::min<int64_t>(tg_div_up(total / P + 1, 256), ctx->sm_count)), (unsigned)P);
        TG_LAUNCH(ctx, partition_compose_kernel, grid, 256, 0, rows_ptr, bounds.as<long long>(), P, prepend, d_off.as<long long>(), gather_idx.as<int32_t>());
        TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));   // h_off staging buffer must outlive the copy
        for (int p = 0; p < P; p++) {
            long long cnt = h_off[p + 1] - h_off[p];
            if (cnt == 0) continue;
            TG_TRY(emit(in, gather_idx.as<int32_t>() + h_off[p], cnt, p));
        }
        return TGPU_OK;
    }

    // Common case (no replicated rows, fixed-width columns, <= 64 partitions): one stable multi-split pass moves every
    // column straight to its partition-contiguous place; no sort, no gather index.  Same row order as the column-wise
    // strategy of the reference (ascending position inside a partition, PagePartitioner.java:242-276).
    bool multisplit_applies(const DevPage& in) const
    {
        if (partition_count > XMAXP || 2 * (int)in.cols.size() > XMAXC || getenv("TGPU_PARTITION_SORT")) return false;
        if (null_channel >= 0 && null_channel < (int)in.cols.size() && in.cols[null_channel].validity) return false;
        for (auto& c : in.cols)
            if (c.type == TGPU_UTF8 || c.type == TGPU_INT128) return false;     // (the multi-split lanes are at most 8 bytes wide)
        return true;
    }

    int add_input_multisplit(const DevPage& in)
    {
        const int P = partition_count, C = (int)in.cols.size();
        const int64_t n = in.rows;
        PhaseTrace trace{ctx, "partition"};
        const XchgGeom geom = xchg_geom(ctx, n, P, false);
        const int grid = geom.nchunks;
        DevBuf pids, hist, block_off, d_totals;
        TG_TRY(hist.alloc(ctx, (size_t)grid * P * 4));
        TG_TRY(block_off.alloc(ctx, (size_t)grid * P * 8));
        TG_TRY(d_totals.alloc(ctx, (size_t)P * 8));
        KeyCols k;
        TG_TRY(key_cols(in, &k));
        const int32_t* b2p = bucket_to_partition.empty() ? nullptr : d_b2p.as<int32_t>();
        const bool ids_from_key = xchg_ids_from_key(geom, k);      // plain BIGINT key: no 1-byte id array between the two passes
        if (!ids_from_key) TG_TRY(pids.alloc(ctx, (size_t)n));
        TG_TRY(xchg_launch_hist(ctx, geom, k, n, bucket_count, b2p, P, ids_from_key ? nullptr : pids.as<uint8_t>(), hist.as<unsigned int>()));
        TG_LAUNCH(ctx, xchg_offsets_kernel, P, 256, 0, hist.as<unsigned int>(), grid, P, block_off.as<long long>(), d_totals.as<long long>());
        std::vector<long long> counts(P), off(P + 1, 0);
        TG_CUDA(ctx, cudaMemcpyAsync(counts.data(), d_totals.p, (size_t)P * 8, cudaMemcpyDeviceToHost, ctx->stream));
        TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        for (int q = 0; q < P; q++) off[q + 1] = off[q] + counts[q];
        trace.mark("hist+offsets");
        std::vector<bool> has_nulls(C);
        for (int c = 0; c < C; c++) has_nulls[c] = in.cols[c].validity != nullptr;
        const std::vector<XchgLane> lanes = xchg_lanes(in, has_nulls);
        std::vector<std::shared_ptr<DevBuf>> out(lanes.size());
        std::vector<char*> h_dst(lanes.size() * P);
        for (size_t l = 0; l < lanes.size(); l++) {
            out[l] = std::make_shared<DevBuf>();
            TG_TRY(out[l]->alloc(ctx, (size_t)n * lane_bytes(lanes[l])));
            for (int q = 0; q < P; q++) h_dst[l * P + q] = (char*)out[l]->p + off[q] * lane_bytes(lanes[l]);
        }
        DevBuf d_dst;
        XchgCols xc;
        TG_TRY(xchg_cols(ctx, lanes, h_dst, &d_dst, &xc));
        TG_TRY(xchg_launch_scatter(ctx, geom, ids_from_key ? nullptr : pids.as<uint8_t>(), n, P, block_off.as<long long>(), xc, &k, bucket_count, b2p));
        trace.mark("scatter");
        std::vector<char*> base(lanes.size());
        for (int q = 0; q < P; q++) {
            if (counts[q] == 0) continue;
            for (size_t l = 0; l < lanes.size(); l++) base[l] = h_dst[l * P + q];
            DevPage outp;
            TG_TRY(xchg_page(ctx, lanes, base, counts[q], &out, &outp));     // all partitions alias slices of one buffer per lane
            OwnedPage* o = tg_make_owned_page(std::move(outp));
            o->partition = q;
            pending.push_back(o);
        }
        TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));   // h_dst staging must outlive its copy; NULL byte lanes are released here
        return TGPU_OK;
    }

    int emit(const DevPage& in, const int32_t* d_idx, int64_t count, int32_t partition)
    {
        DevPage outp;
        outp.rows = count;
        outp.cols.resize(in.cols.size());
        for (size_t c = 0; c < in.cols.size(); c++) TG_TRY(tg_gather_column(ctx, in.cols[c], d_idx, count, false, &outp.cols[c]));
        OwnedPage* o = tg_make_owned_page(std::move(outp));
        o->partition = partition;
        pending.push_back(o);
        return TGPU_OK;
    }

    int get_output(OwnedPage** out) override
    {
        *out = nullptr;
        if (next_out < pending.size()) {
            *out = pending[next_out++];
            last_partition = (*out)->partition;
        }
        return TGPU_OK;
    }
    int finish() override { finishing = true; return TGPU_OK; }
    bool is_finished() override { return finishing && next_out >= pending.size(); }
};

// ------------------------------------------------------------------------------------------------
// NCCL, resolved at run time so that libtrino_gpu.so has no link-time dependency on a particular libnccl
// ------------------------------------------------------------------------------------------------
typedef struct { char internal[128]; } ncclUniqueIdT;
typedef int (*nccl_get_unique_id_t)(ncclUniqueIdT*);
typedef int (*nccl_comm_init_rank_t)(ncclComm**, int, ncclUniqueIdT, int);
typedef int (*nccl_comm_destroy_t)(ncclComm*);
typedef int (*nccl_send_t)(const void*, size_t, int, int, ncclComm*, cudaStream_t);
typedef int (*nccl_recv_t)(void*, size_t, int, int, ncclComm*, cudaStream_t);
typedef int (*nccl_group_t)(void);
typedef int (*nccl_all_gather_t)(const void*, void*, size_t, int, ncclComm*, cudaStream_t);
typedef int (*nccl_all_reduce_t)(const void*, void*, size_t, int, int, ncclComm*, cudaStream_t);
typedef const char* (*nccl_get_error_string_t)(int);
typedef int (*nccl_comm_split_t)(ncclComm*, int, int, ncclComm**, void*);

struct NcclApi {
    void* handle = nullptr;
    nccl_get_unique_id_t get_unique_id = nullptr;
    nccl_comm_init_rank_t comm_init_rank = nullptr;
    nccl_comm_destroy_t comm_destroy = nullptr;
    nccl_send_t send = nullptr;
    nccl_recv_t recv = nullptr;
    nccl_group_t group_start = nullptr, group_end = nullptr;
    nccl_all_gather_t all_gather = nullptr;
    nccl_all_reduce_t all_reduce = nullptr;
    nccl_get_error_string_t error_string = nullptr;
    nccl_comm_split_t comm_split = nullptr;
};

NcclApi g_nccl;

int load_nccl(tgpu_ctx* ctx)
{
    if (g_nccl.handle) return TGPU_OK;
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "libnccl.so.2 not found: %s", dlerror());
    g_nccl.get_unique_id = (nccl_get_unique_id_t)dlsym(h, "ncclGetUniqueId");
    g_nccl.comm_init_rank = (nccl_comm_init_rank_t)dlsym(h, "ncclCommInitRank");
    g_nccl.comm_destroy = (nccl_comm_destroy_t)dlsym(h, "ncclCommDestroy");
    g_nccl.send = (nccl_send_t)dlsym(h, "ncclSend");
    g_nccl.recv = (nccl_recv_t)dlsym(h, "ncclRecv");
    g_nccl.group_start = (nccl_group_t)dlsym(h, "ncclGroupStart");
    g_nccl.group_end = (nccl_group_t)dlsym(h, "ncclGroupEnd");
    g_nccl.all_gather = (nccl_all_gather_t)dlsym(h, "ncclAllGather");
    g_nccl.all_reduce = (nccl_all_reduce_t)dlsym(h, "ncclAllReduce");
    g_nccl.error_string = (nccl_get_error_string_t)dlsym(h, "ncclGetErrorString");
    g_nccl.comm_split = (nccl_comm_split_t)dlsym(h, "ncclCommSplit");   // optional (NCCL >= 2.18): split-phase exchange only
    if (!g_nccl.get_unique_id || !g_nccl.comm_init_rank || !g_nccl.send || !g_nccl.recv || !g_nccl.group_start || !g_nccl.group_end || !g_nccl.all_gather)
        return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "libnccl is missing required symbols");
    g_nccl.handle = h;
    return TGPU_OK;
}

#define TG_NCCL(ctx, call)                                                                                               \
    do {                                                                                                                 \
        int _r = (call);                                                                                                 \
        if (_r != 0)                                                                                                     \
            return tg_fail((ctx), TGPU_ERR_CUDA, "%s failed: %s", #call, g_nccl.error_string ? g_nccl.error_string(_r) : "nccl error"); \
    } while (0)

constexpr int NCCL_INT8 = 0;    // ncclInt8 / ncclChar
constexpr int NCCL_INT64 = 4;   // ncclInt64

}  // namespace

int tg_comm_destroy_internal(tgpu_ctx* ctx)
{
    if (ctx->comm2 && g_nccl.comm_destroy) g_nccl.comm_destroy(ctx->comm2);
    if (ctx->comm && g_nccl.comm_destroy) g_nccl.comm_destroy(ctx->comm);
    ctx->comm = ctx->comm2 = nullptr;
    if (ctx->copy_stream) { cudaStreamDestroy(ctx->copy_stream); ctx->copy_stream = nullptr; }
    // receive arenas: unmap the peers', free this rank's (the caller synchronises the ranks before tearing a communicator down)
    for (int k = 0; k < TGPU_NUM_ARENAS; k++) {
        for (size_t r = 0; r < ctx->arena_peer[k].size(); r++)
            if ((int)r != ctx->rank && ctx->arena_peer[k][r]) cudaIpcCloseMemHandle(ctx->arena_peer[k][r]);
        ctx->arena_peer[k].clear();
        if (ctx->arena_local[k]) { cudaFree(ctx->arena_local[k]); ctx->arena_local[k] = nullptr; }
    }
    ctx->arena_bytes = 0;
    ctx->arena_epoch = 0;
    ctx->exchanges_in_flight = 0;
    ctx->rank = 0;
    ctx->world = 1;
    return TGPU_OK;
}

// ------------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------------
extern "C" int tgpu_partition_create(tgpu_ctx* ctx, const tgpu_partition_spec* spec, tgpu_op** out)
{
    if (!ctx || !spec || !out) return TGPU_ERR_INVALID_ARGUMENT;
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    if (spec->bucket_count < 1) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "partitionCount must be at least 1");   // HashBucketFunction.java:30
    std::unique_ptr<PartitionOp> op(new PartitionOp(ctx));
    op->key_channels.assign(spec->key_channels, spec->key_channels + spec->num_key_channels);
    op->constant_hash.assign((size_t)spec->num_key_channels, 0);
    for (int32_t c = 0; c < spec->num_key_channels; c++) {
        if (spec->key_channels[c] >= 0) continue;
        if (!spec->key_constants) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "partition channel %d is a constant but key_constants is NULL", c);   // PagePartitioner.java:111
        TG_TRY(host_type_hash(ctx, spec->key_constants[c], &op->constant_hash[c]));
    }
    op->bucket_count = spec->bucket_count;
    op->partition_count = spec->bucket_count;
    if (spec->partition_function == TGPU_PARTITION_LOCAL) {
        if (spec->bucket_count & (spec->bucket_count - 1)) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "partitionCount must be a power of 2");   // LocalPartitionGenerator.java:33
        if (spec->bucket_to_partition) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "the local partition function has no bucket-to-partition map");
        op->bucket_count = -spec->bucket_count;      // process_raw_hash (hash.cuh) reads a negative count as the local function
    }
    else if (spec->partition_function != TGPU_PARTITION_HASH_BUCKET)
        return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "unknown partition function %d", spec->partition_function);
    if (spec->bucket_to_partition) {
        op->bucket_to_partition.assign(spec->bucket_to_partition, spec->bucket_to_partition + spec->bucket_count);
        int mx = 0;
        for (int v : op->bucket_to_partition) {
            if (v < 0) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "negative partition in bucket_to_partition");
            mx = std::max(mx, v);
        }
        op->partition_count = mx + 1;   // BucketPartitionFunction.java:35
        TG_TRY(op->d_b2p.alloc(ctx, (size_t)spec->bucket_count * 4));
        TG_CUDA(ctx, cudaMemcpyAsync(op->d_b2p.p, op->bucket_to_partition.data(), (size_t)spec->bucket_count * 4, cudaMemcpyHostToDevice, ctx->stream));
        TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    op->null_channel = spec->null_channel;
    op->replicates_any_row = spec->replicates_any_row != 0;
    *out = op.release();
    return TGPU_OK;
}

extern "C" int tgpu_partition_last_output_partition(tgpu_op* op, int32_t* out)
{
    PartitionOp* p = dynamic_cast<PartitionOp*>(op);
    if (!p || !out) return TGPU_ERR_INVALID_ARGUMENT;
    *out = p->last_partition;
    return TGPU_OK;
}

extern "C" int tgpu_partition_get_partitions(tgpu_op* op, const tgpu_page* page, int32_t* out_partitions)
{
    PartitionOp* p = dynamic_cast<PartitionOp*>(op);
    if (!p || !page || !out_partitions) return TGPU_ERR_INVALID_ARGUMENT;
    tgpu_ctx* ctx = p->ctx;
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    if (page->num_rows == 0) return TGPU_OK;
    DevPage in;
    TG_TRY(tg_ingest_page(ctx, page, &in));
    bool device = (page->flags & TGPU_PAGE_DEVICE) != 0;
    if (device) return p->compute_ids(in, out_partitions, false);
    DevBuf ids;
    TG_TRY(ids.alloc(ctx, (size_t)in.rows * 4));
    TG_TRY(p->compute_ids(in, ids.as<int32_t>(), false));
    TG_CUDA(ctx, cudaMemcpyAsync(out_partitions, ids.p, (size_t)in.rows * 4, cudaMemcpyDeviceToHost, ctx->stream));
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return TGPU_OK;
}

extern "C" int tgpu_comm_get_unique_id(uint8_t id[TGPU_COMM_ID_BYTES])
{
    TG_TRY(load_nccl(nullptr));
    ncclUniqueIdT uid;
    int r = g_nccl.get_unique_id(&uid);
    if (r != 0) return tg_fail(nullptr, TGPU_ERR_CUDA, "ncclGetUniqueId failed");
    memcpy(id, uid.internal, TGPU_COMM_ID_BYTES);
    return TGPU_OK;
}

extern "C" int tgpu_comm_init(tgpu_ctx* ctx, const uint8_t id[TGPU_COMM_ID_BYTES], int rank, int world)
{
    if (!ctx || !id) return TGPU_ERR_INVALID_ARGUMENT;
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    TG_TRY(load_nccl(ctx));
    ncclUniqueIdT uid;
    memcpy(uid.internal, id, TGPU_COMM_ID_BYTES);
    TG_NCCL(ctx, g_nccl.comm_init_rank(&ctx->comm, world, uid, rank));
    ctx->rank = rank;
    ctx->world = world;
    // a second communicator and a side stream for the split-phase exchange: its barrier must not be ordered behind (or ahead
    // of) the count all-gather of the next exchange, which NCCL would do for two operations on one communicator
    if (g_nccl.comm_split && !getenv("TGPU_NO_COMM_SPLIT")) TG_NCCL(ctx, g_nccl.comm_split(ctx->comm, 0, rank, &ctx->comm2, nullptr));
    TG_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking));
    return TGPU_OK;
}

extern "C" int tgpu_comm_destroy(tgpu_ctx* ctx)
{
    if (!ctx) return TGPU_ERR_INVALID_ARGUMENT;
    return tg_comm_destroy_internal(ctx);
}

extern "C" int tgpu_comm_arena_create(tgpu_ctx* ctx, size_t bytes, uint8_t handles_out[TGPU_NUM_ARENAS * TGPU_IPC_HANDLE_BYTES])
{
    if (!ctx || !handles_out || bytes == 0) return TGPU_ERR_INVALID_ARGUMENT;
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    static_assert(sizeof(cudaIpcMemHandle_t) == TGPU_IPC_HANDLE_BYTES, "IPC handle size");
    for (int k = 0; k < TGPU_NUM_ARENAS; k++) {
        if (ctx->arena_local[k]) return tg_fail(ctx, TGPU_ERR_ILLEGAL_STATE, "arenas already created");
        TG_CUDA(ctx, cudaMalloc(&ctx->arena_local[k], bytes));   // plain cudaMalloc: pool memory cannot be exported
        cudaIpcMemHandle_t h;
        TG_CUDA(ctx, cudaIpcGetMemHandle(&h, ctx->arena_local[k]));
        memcpy(handles_out + k * TGPU_IPC_HANDLE_BYTES, &h, TGPU_IPC_HANDLE_BYTES);
    }
    ctx->arena_bytes = bytes;
    return TGPU_OK;
}

extern "C" int tgpu_comm_arena_open(tgpu_ctx* ctx, const uint8_t* all_handles)
{
    if (!ctx || !all_handles) return TGPU_ERR_INVALID_ARGUMENT;
    if (!ctx->arena_local[0]) return tg_fail(ctx, TGPU_ERR_ILLEGAL_STATE, "tgpu_comm_arena_create has not been called");
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    for (int k = 0; k < TGPU_NUM_ARENAS; k++) {
        ctx->arena_peer[k].assign(ctx->world, nullptr);
        for (int r = 0; r < ctx->world; r++) {
            if (r == ctx->rank) { ctx->arena_peer[k][r] = ctx->arena_local[k]; continue; }
            cudaIpcMemHandle_t h;
            memcpy(&h, all_handles + ((size_t)r * TGPU_NUM_ARENAS + k) * TGPU_IPC_HANDLE_BYTES, TGPU_IPC_HANDLE_BYTES);
            TG_CUDA(ctx, cudaIpcOpenMemHandle(&ctx->arena_peer[k][r], h, cudaIpcMemLazyEnablePeerAccess));
        }
    }
    return TGPU_OK;
}

// ------------------------------------------------------------------------------------------------
// General exchange: everything the PagePartitioner can emit - variable-width columns, rows replicated to every partition
// (nullChannel rows and the single replicatesAnyRow row, PagePartitioner.java:229-241,401-416), more than XMAXC / 2 columns.  The
// operator itself partitions the page (its sort + compose path), the per-destination pages travel as ncclSend/ncclRecv per buffer
// (values, offsets + bytes, validity bitmap), and the chunks received from rank 0..W-1 are concatenated in rank order, which is the
// row order the fixed-width paths produce.  Three host round trips (part sizes, the all-gathered size matrix, the final sync): this
// is the completeness path, the multi-split paths above are the fast ones.
// ------------------------------------------------------------------------------------------------
namespace {
// the type of a column's values: a DICT32 or RLE column's is its dictionary's
int32_t value_type(const tgpu_column& col)
{
    return (col.type == TGPU_DICT32 || col.type == TGPU_RLE) && col.dictionary ? col.dictionary->type : col.type;
}

bool exchange_needs_general_path(const PartitionOp* p, const tgpu_page* page)
{
    if (p->null_channel >= 0 || p->replicates_any_row) return true;
    if (2 * page->num_columns > XMAXC) return true;
    for (int c = 0; c < page->num_columns; c++) {
        int type = value_type(page->columns[c]);
        if (type == TGPU_UTF8 || type == TGPU_INT128) return true;
    }
    return false;
}

// The checks the blocking and the split-phase exchange share.  *general: the page takes the general exchange, because the
// multi-split does not carry its shape or has fewer partitions than there are ranks.
int exchange_prologue(tgpu_ctx* ctx, const PartitionOp* p, const tgpu_page* page, bool* general)
{
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    if (!ctx->comm) return tg_fail(ctx, TGPU_ERR_ILLEGAL_STATE, "tgpu_comm_init has not been called");
    const int W = ctx->world;
    if (p->partition_count != W) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "partition count %d != world size %d", p->partition_count, W);
    if (page->num_rows > (int64_t)INT32_MAX) return tg_fail(ctx, TGPU_ERR_INVALID_ARGUMENT, "page has more than 2^31-1 positions");
    *general = exchange_needs_general_path(p, page) || W > XMAXP;
    return TGPU_OK;
}

// The count matrix: the `per_rank` int64 entries every rank holds in d_mine, all-gathered into a host matrix with one row per
// rank, in rank order.  One device-to-host copy and one wait.
int count_matrix(tgpu_ctx* ctx, const DevBuf& d_mine, size_t per_rank, std::vector<long long>* matrix)
{
    const int W = ctx->world;
    DevBuf d_all;
    TG_TRY(d_all.alloc(ctx, (size_t)W * per_rank * 8));
    if (W > 1) TG_NCCL(ctx, g_nccl.all_gather(d_mine.p, d_all.p, per_rank, NCCL_INT64, ctx->comm, ctx->stream));
    else TG_CUDA(ctx, cudaMemcpyAsync(d_all.p, d_mine.p, per_rank * 8, cudaMemcpyDeviceToDevice, ctx->stream));
    matrix->resize((size_t)W * per_rank);
    TG_CUDA(ctx, cudaMemcpyAsync(matrix->data(), d_all.p, (size_t)W * per_rank * 8, cudaMemcpyDeviceToHost, ctx->stream));
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return TGPU_OK;
}

// per column: does any rank's page carry NULLs (entry first + c of each rank's row of V entries), so that it needs a NULL-byte lane
std::vector<bool> null_lanes(const std::vector<long long>& matrix, int W, int V, int first, int C)
{
    std::vector<bool> any(C, false);
    for (int c = 0; c < C; c++)
        for (int r = 0; r < W; r++) any[c] = any[c] || matrix[(size_t)r * V + first + c] != 0;
    return any;
}

// Where the rows of a peer-store or split-phase exchange land in a destination's arena: one 256-byte aligned region per lane,
// as many rows long as the destination receives, in lane order; inside a region the rows of lower-ranked senders come first.
// Every sender and the receiver derive it from the same count matrix (entry d of each rank's row: its rows for destination d), so
// they agree byte for byte.
struct ArenaLayout {
    std::vector<long long> total_recv_of, first_row;    // per destination: rows it receives, and where this rank's start
    std::vector<size_t> es;                             // per lane: bytes per row

    ArenaLayout(const std::vector<long long>& matrix, int W, int V, int me, const std::vector<XchgLane>& lanes) : total_recv_of(W, 0), first_row(W, 0)
    {
        for (int d = 0; d < W; d++)
            for (int r = 0; r < W; r++) {
                total_recv_of[d] += matrix[(size_t)r * V + d];
                if (r < me) first_row[d] += matrix[(size_t)r * V + d];
            }
        for (auto& lane : lanes) es.push_back(lane_bytes(lane));
    }
    size_t region_off(int d, size_t lane) const
    {
        size_t off = 0;
        for (size_t l = 0; l < lane; l++) off += (((size_t)total_recv_of[d] * es[l]) + 255) & ~(size_t)255;
        return off;
    }
    size_t bytes(int d) const { return region_off(d, es.size()); }
    // where this rank's rows of lane l go in the arena of destination d
    char* dst(void* arena, int d, size_t l) const { return (char*)arena + region_off(d, l) + (size_t)first_row[d] * es[l]; }
};

// part[d]: the rows this rank has for rank d (nullptr = none); the parts must stay alive until this returns
int exchange_pages(tgpu_ctx* ctx, const std::vector<const DevPage*>& part, const std::vector<int32_t>& types, tgpu_page** out)
{
    const int W = ctx->world, me = ctx->rank, C = (int)types.size();
    // 2. sizes: per destination {rows, then per column: has validity, first offset, value bytes}
    const int V = 1 + 3 * C;
    std::vector<long long> mine((size_t)W * V, 0);
    for (int d = 0; d < W; d++) {
        if (!part[d]) continue;
        const DevPage& pg = *part[d];
        mine[(size_t)d * V] = pg.rows;
        for (int c = 0; c < C; c++) {
            const DevColumn& col = pg.cols[c];
            mine[(size_t)d * V + 1 + 3 * c] = col.validity ? 1 : 0;
            if (col.type == TGPU_UTF8 && pg.rows > 0) {
                int32_t ends[2] = {0, 0};
                TG_CUDA(ctx, cudaMemcpyAsync(&ends[0], col.offsets, 4, cudaMemcpyDeviceToHost, ctx->stream));
                TG_CUDA(ctx, cudaMemcpyAsync(&ends[1], col.offsets + pg.rows, 4, cudaMemcpyDeviceToHost, ctx->stream));
                TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
                mine[(size_t)d * V + 2 + 3 * c] = ends[0];
                mine[(size_t)d * V + 3 + 3 * c] = ends[1] - ends[0];
            }
        }
    }
    std::vector<long long> all;
    {
        DevBuf d_mine;
        TG_TRY(d_mine.alloc(ctx, mine.size() * 8));
        TG_CUDA(ctx, cudaMemcpyAsync(d_mine.p, mine.data(), mine.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
        TG_TRY(count_matrix(ctx, d_mine, mine.size(), &all));
    }
    auto info = [&](int sender, int dest, int k) { return all[((size_t)sender * W + dest) * V + k]; };
    long long total_recv = 0;
    for (int r = 0; r < W; r++) total_recv += info(r, me, 0);
    if (total_recv > (long long)INT32_MAX) return tg_fail(ctx, TGPU_ERR_INSUFFICIENT_RESOURCES, "exchange output exceeds 2^31-1 rows on rank %d", me);
    // 3. receive chunks: one DevColumn per (sender, column); this rank's own part is used in place
    std::vector<std::vector<DevColumn>> chunk(W, std::vector<DevColumn>(C));
    for (int r = 0; r < W; r++) {
        const long long rows = info(r, me, 0);
        if (r == me) {
            if (part[me]) chunk[r] = part[me]->cols;        // (shares the buffers)
            continue;
        }
        for (int c = 0; c < C && rows > 0; c++) {
            DevColumn& col = chunk[r][c];
            col.type = types[c];
            col.length = rows;
            if (types[c] == TGPU_UTF8) {
                const long long first = info(r, me, 2 + 3 * c), bytes = info(r, me, 3 + 3 * c);
                col.own_offsets = std::make_shared<DevBuf>();
                TG_TRY(col.own_offsets->alloc(ctx, (size_t)(rows + 1) * 4));
                col.offsets = col.own_offsets->as<int32_t>();
                col.own_data = std::make_shared<DevBuf>();
                TG_TRY(col.own_data->alloc(ctx, (size_t)std::max<long long>(bytes, 1)));
                col.data = (const char*)col.own_data->p - first;            // the sender's offsets stay as they are
                col.data_bytes = bytes;
            }
            else {
                col.own_data = std::make_shared<DevBuf>();
                TG_TRY(col.own_data->alloc(ctx, (size_t)rows * col.elem_size()));
                col.data = col.own_data->p;
            }
            if (info(r, me, 1 + 3 * c)) {
                col.own_validity = std::make_shared<DevBuf>();
                TG_TRY(col.own_validity->alloc(ctx, (size_t)((rows + 7) / 8)));
                col.validity = col.own_validity->as<uint8_t>();
            }
        }
    }
    // 4. one NCCL group: every buffer of every part to its destination, every chunk buffer from its sender (same order on both sides)
    if (W > 1) {
        TG_NCCL(ctx, g_nccl.group_start());
        for (int peer = 0; peer < W; peer++) {
            if (peer == me) continue;
            if (part[peer] && part[peer]->rows > 0) {
                const DevPage& pg = *part[peer];
                for (int c = 0; c < C; c++) {
                    const DevColumn& col = pg.cols[c];
                    if (col.type == TGPU_UTF8) {
                        const long long first = mine[(size_t)peer * V + 2 + 3 * c], bytes = mine[(size_t)peer * V + 3 + 3 * c];
                        TG_NCCL(ctx, g_nccl.send(col.offsets, (size_t)(pg.rows + 1) * 4, NCCL_INT8, peer, ctx->comm, ctx->stream));
                        if (bytes > 0) TG_NCCL(ctx, g_nccl.send((const char*)col.data + first, (size_t)bytes, NCCL_INT8, peer, ctx->comm, ctx->stream));
                    }
                    else TG_NCCL(ctx, g_nccl.send(col.data, (size_t)pg.rows * col.elem_size(), NCCL_INT8, peer, ctx->comm, ctx->stream));
                    if (col.validity) TG_NCCL(ctx, g_nccl.send(col.validity, (size_t)((pg.rows + 7) / 8), NCCL_INT8, peer, ctx->comm, ctx->stream));
                }
            }
            const long long rows = info(peer, me, 0);
            for (int c = 0; c < C && rows > 0; c++) {
                DevColumn& col = chunk[peer][c];
                if (col.type == TGPU_UTF8) {
                    TG_NCCL(ctx, g_nccl.recv(col.own_offsets->p, (size_t)(rows + 1) * 4, NCCL_INT8, peer, ctx->comm, ctx->stream));
                    if (col.data_bytes > 0) TG_NCCL(ctx, g_nccl.recv(col.own_data->p, (size_t)col.data_bytes, NCCL_INT8, peer, ctx->comm, ctx->stream));
                }
                else TG_NCCL(ctx, g_nccl.recv(col.own_data->p, (size_t)rows * col.elem_size(), NCCL_INT8, peer, ctx->comm, ctx->stream));
                if (col.validity) TG_NCCL(ctx, g_nccl.recv(col.own_validity->p, (size_t)((rows + 7) / 8), NCCL_INT8, peer, ctx->comm, ctx->stream));
            }
        }
        TG_NCCL(ctx, g_nccl.group_end());
    }
    // 5. the output page: chunks in sender order
    DevPage outp;
    outp.rows = total_recv;
    outp.cols.resize(C);
    for (int c = 0; c < C; c++) {
        std::vector<const DevColumn*> parts;
        for (int r = 0; r < W; r++)
            if (info(r, me, 0) > 0) parts.push_back(&chunk[r][c]);
        if (parts.empty()) {
            // nothing arrived: an empty column of the right type
            DevColumn e;
            e.type = types[c];
            e.own_data = std::make_shared<DevBuf>();
            TG_TRY(e.own_data->alloc(ctx, 8));
            e.data = e.own_data->p;
            if (types[c] == TGPU_UTF8) {
                e.own_offsets = std::make_shared<DevBuf>();
                TG_TRY(e.own_offsets->alloc(ctx, 4));
                TG_CUDA(ctx, cudaMemsetAsync(e.own_offsets->p, 0, 4, ctx->stream));
                e.offsets = e.own_offsets->as<int32_t>();
            }
            outp.cols[c] = std::move(e);
        }
        else if (parts.size() == 1) outp.cols[c] = *parts[0];
        else TG_TRY(tg_concat_columns(ctx, parts, &outp.cols[c]));
    }
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));      // the caller releases the parts next: the sends must have left them
    OwnedPage* o = tg_make_owned_page(std::move(outp));
    *out = &o->hdr;
    return TGPU_OK;
}

std::vector<int32_t> value_types_of(const tgpu_page* page)
{
    std::vector<int32_t> types(page->num_columns);
    for (int c = 0; c < page->num_columns; c++) types[c] = value_type(page->columns[c]);
    return types;
}

int exchange_general(tgpu_ctx* ctx, PartitionOp* p, const tgpu_page* page, tgpu_page** out)
{
    const int W = ctx->world;
    // 1. partition locally: at most one page per destination
    TG_TRY(p->add_input(page));
    std::vector<std::unique_ptr<OwnedPage>> owned(W);
    for (size_t i = p->next_out; i < p->pending.size(); i++) {
        OwnedPage* o = p->pending[i];
        if (o->partition < 0 || o->partition >= W || owned[o->partition]) { delete o; continue; }
        owned[o->partition].reset(o);
    }
    p->pending.clear();
    p->next_out = 0;
    std::vector<const DevPage*> part(W, nullptr);
    for (int d = 0; d < W; d++)
        if (owned[d]) part[d] = &owned[d]->page;
    return exchange_pages(ctx, part, value_types_of(page), out);
}
}  // namespace

extern "C" int tgpu_exchange_partitioned(tgpu_ctx* ctx, tgpu_op* partitioner, const tgpu_page* page, tgpu_page** out)
{
    return tgpu_exchange_partitioned_fenced(ctx, partitioner, page, nullptr, out);
}

extern "C" int tgpu_exchange_partitioned_fenced(tgpu_ctx* ctx, tgpu_op* partitioner, const tgpu_page* page, tgpu_ctx* consumer, tgpu_page** out)
{
    PartitionOp* p = dynamic_cast<PartitionOp*>(partitioner);
    if (!ctx || !p || !page || !out) return TGPU_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    bool general = false;
    TG_TRY(exchange_prologue(ctx, p, page, &general));
    if (general) return exchange_general(ctx, p, page, out);
    const int W = ctx->world, me = ctx->rank;
    const int64_t n = page->num_rows;
    DevPage in;
    TG_TRY(tg_ingest_page(ctx, page, &in));
    PhaseTrace trace{ctx, "exchange rank " + std::to_string(me)};
    const int C = (int)in.cols.size();
    // 1. partition ids + per-CTA histograms + offsets (stable multi-split, no sort)
    const XchgGeom geom = xchg_geom(ctx, n, W, W > 1);
    const int grid = geom.nchunks;
    DevBuf pids, hist, block_off, d_totals;
    TG_TRY(pids.alloc(ctx, (size_t)std::max<int64_t>(n, 1)));
    TG_TRY(hist.alloc(ctx, (size_t)grid * W * 4));
    TG_TRY(block_off.alloc(ctx, (size_t)grid * W * 8));
    TG_TRY(d_totals.alloc(ctx, (size_t)(W + C) * 8));
    std::vector<long long> send_vec(W + C, 0);     // W send counts, then one "has NULLs" flag per column
    if (n > 0) {
        KeyCols k;
        TG_TRY(p->key_cols(in, &k));
        TG_TRY(xchg_launch_hist(ctx, geom, k, n, p->bucket_count, p->bucket_to_partition.empty() ? nullptr : p->d_b2p.as<int32_t>(), W, pids.as<uint8_t>(),
                                hist.as<unsigned int>()));
        TG_LAUNCH(ctx, xchg_offsets_kernel, W, 256, 0, hist.as<unsigned int>(), grid, W, block_off.as<long long>(), d_totals.as<long long>());
        TG_CUDA(ctx, cudaMemcpyAsync(send_vec.data(), d_totals.p, (size_t)W * 8, cudaMemcpyDeviceToHost, ctx->stream));
        TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    trace.mark("hist+offsets");
    for (int c = 0; c < C; c++) send_vec[W + c] = in.cols[c].validity ? 1 : 0;
    // 2. count matrix: every rank learns what every rank sends to whom (and which columns carry NULLs anywhere)
    const int V = W + C;
    std::vector<long long> matrix;
    DevBuf d_send;
    TG_TRY(d_send.alloc(ctx, (size_t)V * 8));
    TG_CUDA(ctx, cudaMemcpyAsync(d_send.p, send_vec.data(), (size_t)V * 8, cudaMemcpyHostToDevice, ctx->stream));
    TG_TRY(count_matrix(ctx, d_send, V, &matrix));
    trace.mark("count all-gather");
    std::vector<long long> send_off(W + 1, 0), recv_counts(W), recv_off(W + 1, 0);
    for (int r = 0; r < W; r++) {
        send_off[r + 1] = send_off[r] + send_vec[r];
        recv_counts[r] = matrix[(size_t)r * V + me];
        recv_off[r + 1] = recv_off[r] + recv_counts[r];
    }
    const long long total_recv = recv_off[W];
    if (total_recv > (long long)INT32_MAX) return tg_fail(ctx, TGPU_ERR_INSUFFICIENT_RESOURCES, "exchange output exceeds 2^31-1 rows on rank %d", me);
    // 3. one scatter pass writes every column (and the NULL bytes of nullable columns) partition-contiguously
    const std::vector<XchgLane> lanes = xchg_lanes(in, null_lanes(matrix, W, V, W, C));
    // Peer-memory path: every rank knows every destination's arena layout, so the scatter kernel stores each row directly at its
    // final address in the destination GPU's arena.
    const ArenaLayout layout(matrix, W, V, me, lanes);
    bool p2p = !ctx->arena_peer[0].empty() && !getenv("TGPU_EXCHANGE_NCCL");
    for (int d = 0; d < W && p2p; d++) p2p = layout.bytes(d) <= ctx->arena_bytes;
    const int arena = (int)(ctx->arena_epoch % TGPU_NUM_ARENAS);
    std::vector<DevBuf> send(lanes.size());
    std::vector<std::shared_ptr<DevBuf>> recv(lanes.size());
    std::vector<char*> h_dst(lanes.size() * W);
    for (size_t l = 0; l < lanes.size(); l++) {
        const size_t es = lane_bytes(lanes[l]);
        if (p2p) {
            for (int d = 0; d < W; d++) h_dst[l * W + d] = layout.dst(ctx->arena_peer[arena][d], d, l);
            continue;
        }
        TG_TRY(send[l].alloc(ctx, (size_t)std::max<int64_t>(n, 1) * es));
        recv[l] = std::make_shared<DevBuf>();
        TG_TRY(recv[l]->alloc(ctx, (size_t)std::max<long long>(total_recv, 1) * es));
        for (int r = 0; r < W; r++) h_dst[l * W + r] = (char*)send[l].p + send_off[r] * es;
        // rows that stay on this GPU are scattered straight into their final place in the receive buffer
        h_dst[l * W + me] = (char*)recv[l]->p + recv_off[me] * es;
    }
    trace.mark("buffer allocation");
    DevBuf d_dst;
    XchgCols xc;
    TG_TRY(xchg_cols(ctx, lanes, h_dst, &d_dst, &xc));
    if (n > 0) TG_TRY(xchg_launch_scatter(ctx, geom, pids.as<uint8_t>(), n, W, block_off.as<long long>(), xc));
    trace.mark("scatter");
    std::vector<char*> base(lanes.size());
    DevPage outp;
    if (p2p) {
        // the rows are already in the destination arenas; a 1-element all-reduce on the stream is the barrier that tells
        // every rank that all its senders' scatter kernels have completed
        if (consumer && consumer != ctx) {
            // The barrier below tells every peer that it may overwrite the arena this rank's consumer read the exchange before
            // last from: do not enter it before everything the consumer context has enqueued so far (its probe of that page)
            // is done.  The wait is on the device - this exchange's scatter and the consumer's probe overlap.
            if (!consumer->fence_ev) TG_CUDA(ctx, cudaEventCreateWithFlags(&consumer->fence_ev, cudaEventDisableTiming));
            TG_CUDA(ctx, cudaEventRecord(consumer->fence_ev, consumer->stream));
            TG_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, consumer->fence_ev, 0));
        }
        DevBuf token;
        TG_TRY(token.alloc(ctx, 16));
        TG_CUDA(ctx, cudaMemsetAsync(token.p, 0, 16, ctx->stream));
        TG_NCCL(ctx, g_nccl.all_reduce(token.p, (char*)token.p + 8, 1, NCCL_INT64, 0 /* ncclSum */, ctx->comm, ctx->stream));
        trace.mark("p2p scatter + barrier");
        ctx->arena_epoch++;
        for (size_t l = 0; l < lanes.size(); l++) base[l] = (char*)ctx->arena_local[arena] + layout.region_off(me, l);
        TG_TRY(xchg_page(ctx, lanes, base, total_recv, nullptr, &outp));     // aliases the arena: valid until the second-next exchange on this context
    }
    else {
        // 4. all-to-all with explicit counts: one NCCL group for every column
        TG_NCCL(ctx, g_nccl.group_start());
        for (size_t l = 0; l < lanes.size(); l++) {
            const size_t es = lane_bytes(lanes[l]);
            for (int r = 0; r < W; r++) {
                if (r == me) continue;
                if (send_vec[r] > 0)
                    TG_NCCL(ctx, g_nccl.send((const char*)send[l].p + send_off[r] * es, (size_t)send_vec[r] * es, NCCL_INT8, r, ctx->comm, ctx->stream));
                if (recv_counts[r] > 0)
                    TG_NCCL(ctx, g_nccl.recv((char*)recv[l]->p + recv_off[r] * es, (size_t)recv_counts[r] * es, NCCL_INT8, r, ctx->comm, ctx->stream));
            }
        }
        TG_NCCL(ctx, g_nccl.group_end());
        trace.mark("nccl send/recv");
        for (size_t l = 0; l < lanes.size(); l++) base[l] = (char*)recv[l]->p;
        TG_TRY(xchg_page(ctx, lanes, base, total_recv, &recv, &outp));
    }
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));   // send buffers are released after the transfers have left them
    OwnedPage* o = tg_make_owned_page(std::move(outp));
    *out = &o->hdr;
    return TGPU_OK;
}

// ------------------------------------------------------------------------------------------------
// broadcast exchange: FIXED_BROADCAST_DISTRIBUTION (M/sql/planner/SystemPartitioningHandle.java:51) - the build side of a REPLICATED
// join: BroadcastOutputBuffer hands every page to every consumer (M/execution/buffer/BroadcastOutputBuffer.java), so every rank ends up
// with all rows.  Here: one all-gather of the row counts, then ncclSend/ncclRecv of every column (NULL bytes for nullable ones).
// ------------------------------------------------------------------------------------------------
namespace {
__global__ void validity_to_bytes_kernel(const uint8_t* __restrict__ validity, int64_t n, uint8_t* __restrict__ is_null)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) is_null[i] = tg_valid(validity, i) ? 0 : 1;
}
}  // namespace

extern "C" int tgpu_exchange_broadcast(tgpu_ctx* ctx, const tgpu_page* page, tgpu_page** out)
{
    if (!ctx || !page || !out) return TGPU_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    const int W = ctx->comm ? ctx->world : 1;     // no communicator: a single-GPU plan, the "broadcast" is a copy
    DevPage in;
    TG_TRY(tg_ingest_page(ctx, page, &in));
    const int C = (int)in.cols.size();
    bool variable_width = false;
    for (auto& c : in.cols) variable_width = variable_width || c.elem_size() == 0;
    if (variable_width) {
        // variable-width columns: every rank's page goes to every rank through the general exchange (offsets + bytes per chunk)
        if (W == 1) {
            OwnedPage* o = tg_make_owned_page(std::move(in));
            *out = &o->hdr;
            return TGPU_OK;
        }
        std::vector<const DevPage*> part(W, &in);
        return exchange_pages(ctx, part, value_types_of(page), out);
    }
    const int64_t n = in.rows;
    // count matrix: rows and one "has NULLs" flag per column from every rank
    const int V = 1 + C;
    std::vector<long long> mine(V, 0), matrix;
    mine[0] = n;
    for (int c = 0; c < C; c++) mine[1 + c] = in.cols[c].validity ? 1 : 0;
    if (W > 1) {
        DevBuf d_mine;
        TG_TRY(d_mine.alloc(ctx, (size_t)V * 8));
        TG_CUDA(ctx, cudaMemcpyAsync(d_mine.p, mine.data(), (size_t)V * 8, cudaMemcpyHostToDevice, ctx->stream));
        TG_TRY(count_matrix(ctx, d_mine, V, &matrix));
    }
    else matrix = mine;
    const int my_rank = W > 1 ? ctx->rank : 0;
    std::vector<long long> off(W + 1, 0);
    for (int r = 0; r < W; r++) off[r + 1] = off[r] + matrix[(size_t)r * V];
    const long long total = off[W];
    if (total > (long long)INT32_MAX) return tg_fail(ctx, TGPU_ERR_INSUFFICIENT_RESOURCES, "broadcast output exceeds 2^31-1 rows");
    std::vector<XchgLane> lanes = xchg_lanes(in, null_lanes(matrix, W, V, 1, C));
    std::vector<std::shared_ptr<DevBuf>> recv(lanes.size());
    std::vector<DevBuf> staged(lanes.size());
    std::vector<char*> base(lanes.size());
    for (size_t l = 0; l < lanes.size(); l++) {
        XchgLane& lane = lanes[l];
        const size_t es = lane_bytes(lane);
        recv[l] = std::make_shared<DevBuf>();
        TG_TRY(recv[l]->alloc(ctx, (size_t)std::max<long long>(total, 1) * es));
        base[l] = (char*)recv[l]->p;
        if (lane.nulls) {
            // this rank's NULL bytes (all zero when its own page has no validity buffer), copied as 1-byte cells
            TG_TRY(staged[l].alloc(ctx, (size_t)std::max<int64_t>(n, 1)));
            if (lane.src && n > 0)
                TG_LAUNCH(ctx, validity_to_bytes_kernel, tg_grid(ctx, n, 1024, 8), 256, 0, (const uint8_t*)lane.src, n, staged[l].as<uint8_t>());
            else TG_CUDA(ctx, cudaMemsetAsync(staged[l].p, 0, (size_t)std::max<int64_t>(n, 1), ctx->stream));
            lane.src = staged[l].p;
        }
        if (n > 0) TG_CUDA(ctx, cudaMemcpyAsync(base[l] + (size_t)off[my_rank] * es, lane.src, (size_t)n * es, cudaMemcpyDeviceToDevice, ctx->stream));
    }
    if (W > 1) TG_NCCL(ctx, g_nccl.group_start());
    for (size_t l = 0; l < lanes.size(); l++)
        for (int r = 0; r < W && W > 1; r++) {
            if (r == my_rank) continue;
            const size_t es = lane_bytes(lanes[l]);
            if (n > 0) TG_NCCL(ctx, g_nccl.send(lanes[l].src, (size_t)n * es, NCCL_INT8, r, ctx->comm, ctx->stream));
            long long cnt = matrix[(size_t)r * V];
            if (cnt > 0) TG_NCCL(ctx, g_nccl.recv(base[l] + (size_t)off[r] * es, (size_t)cnt * es, NCCL_INT8, r, ctx->comm, ctx->stream));
        }
    if (W > 1) TG_NCCL(ctx, g_nccl.group_end());
    DevPage outp;
    TG_TRY(xchg_page(ctx, lanes, base, total, &recv, &outp));
    TG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));   // staged NULL bytes and the borrowed input are the caller's again
    OwnedPage* o = tg_make_owned_page(std::move(outp));
    *out = &o->hdr;
    return TGPU_OK;
}

// ------------------------------------------------------------------------------------------------
// split-phase exchange: SMs partition, copy engines move, the caller's next kernels overlap the transfer
// ------------------------------------------------------------------------------------------------
struct tgpu_exchange {
    std::vector<XchgLane> lanes;
    std::vector<size_t> region_off;   // of every lane inside this rank's arena
    std::vector<DevBuf> send;         // per lane: rows for peer destinations, destination-major
    DevBuf token;                     // the barrier's all-reduce buffer
    int arena = 0;
    long long total_recv = 0;
    cudaEvent_t done = nullptr;
    tgpu_page* ready = nullptr;       // the general (blocking) path ran inside begin: the finished page
    ~tgpu_exchange() { if (done) cudaEventDestroy(done); }
};

extern "C" int tgpu_exchange_begin(tgpu_ctx* ctx, tgpu_op* partitioner, const tgpu_page* page, tgpu_exchange** out)
{
    PartitionOp* p = dynamic_cast<PartitionOp*>(partitioner);
    if (!ctx || !p || !page || !out) return TGPU_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    bool general = false;
    TG_TRY(exchange_prologue(ctx, p, page, &general));
    if (!ctx->comm2) return tg_fail(ctx, TGPU_ERR_NOT_SUPPORTED, "split-phase exchange needs ncclCommSplit (NCCL >= 2.18)");
    if (ctx->arena_peer[0].empty()) return tg_fail(ctx, TGPU_ERR_ILLEGAL_STATE, "split-phase exchange needs arenas (tgpu_comm_arena_create/open)");
    if (ctx->exchanges_in_flight >= 2) return tg_fail(ctx, TGPU_ERR_ILLEGAL_STATE, "more than two exchanges in flight on one context");
    if (general) {
        // shapes the copy-engine form does not carry (variable width, replicated rows): the blocking general exchange runs here, _end
        // hands its page over.  Every rank takes this branch for the same exchange (the shape is a property of the plan, not of the data).
        std::unique_ptr<tgpu_exchange> g(new tgpu_exchange());
        TG_TRY(exchange_general(ctx, p, page, &g->ready));
        ctx->exchanges_in_flight++;
        *out = g.release();
        return TGPU_OK;
    }
    const int W = ctx->world, me = ctx->rank;
    const int64_t n = page->num_rows;
    DevPage in;
    TG_TRY(tg_ingest_page(ctx, page, &in));
    const int C = (int)in.cols.size();
    // 1. partition ids, histograms, offsets.  Every destination of the scatter is LOCAL memory here (send buffers and this
    //    rank's own arena), so the warp-granular kernels apply.
    const XchgGeom geom = xchg_geom(ctx, n, W, false);
    const int grid = geom.nchunks;
    DevBuf pids, hist, block_off, d_totals;
    TG_TRY(hist.alloc(ctx, (size_t)grid * W * 4));
    TG_TRY(block_off.alloc(ctx, (size_t)grid * W * 8));
    TG_TRY(d_totals.alloc(ctx, (size_t)(W + C) * 8));
    const int V = W + C;
    KeyCols k;
    memset(&k, 0, sizeof(k));
    const int32_t* b2p = p->bucket_to_partition.empty() ? nullptr : p->d_b2p.as<int32_t>();
    bool ids_from_key = false;
    // the vector this rank contributes to the count matrix is assembled ON THE DEVICE (W send counts from the offsets kernel, then one
    // "has NULLs" flag per column), so the host waits once per exchange - for the all-gathered matrix - not twice
    std::vector<long long> flags(V, 0);
    for (int c = 0; c < C; c++) flags[W + c] = in.cols[c].validity ? 1 : 0;
    TG_CUDA(ctx, cudaMemcpyAsync(d_totals.p, flags.data(), (size_t)V * 8, cudaMemcpyHostToDevice, ctx->stream));
    if (n > 0) {
        TG_TRY(p->key_cols(in, &k));
        ids_from_key = xchg_ids_from_key(geom, k);
        if (!ids_from_key) TG_TRY(pids.alloc(ctx, (size_t)n));
        TG_TRY(xchg_launch_hist(ctx, geom, k, n, p->bucket_count, b2p, W, ids_from_key ? nullptr : pids.as<uint8_t>(), hist.as<unsigned int>()));
        TG_LAUNCH(ctx, xchg_offsets_kernel, W, 256, 0, hist.as<unsigned int>(), grid, W, block_off.as<long long>(), d_totals.as<long long>());
    }
    // 2. count matrix
    std::vector<long long> matrix;
    TG_TRY(count_matrix(ctx, d_totals, V, &matrix));
    const long long* send_vec = &matrix[(size_t)me * V];
    std::vector<long long> send_off(W + 1, 0);
    for (int r = 0; r < W; r++) send_off[r + 1] = send_off[r] + send_vec[r];
    std::vector<XchgLane> lanes = xchg_lanes(in, null_lanes(matrix, W, V, W, C));
    const ArenaLayout layout(matrix, W, V, me, lanes);
    if (layout.total_recv_of[me] > (long long)INT32_MAX) return tg_fail(ctx, TGPU_ERR_INSUFFICIENT_RESOURCES, "exchange output exceeds 2^31-1 rows on rank %d", me);
    for (int d = 0; d < W; d++)
        if (layout.bytes(d) > ctx->arena_bytes) return tg_fail(ctx, TGPU_ERR_INSUFFICIENT_RESOURCES, "rank %d would receive more than its arena holds", d);
    std::unique_ptr<tgpu_exchange> x(new tgpu_exchange());
    x->lanes = std::move(lanes);
    x->total_recv = layout.total_recv_of[me];
    x->arena = (int)(ctx->arena_epoch % TGPU_NUM_ARENAS);
    // 3. scatter: peer-bound rows into send buffers (destination-major), rows that stay into their final place
    const size_t L = x->lanes.size();
    x->send.resize(L);
    std::vector<char*> h_dst(L * W);
    for (size_t l = 0; l < L; l++) {
        const size_t es = layout.es[l];
        x->region_off.push_back(layout.region_off(me, l));
        TG_TRY(x->send[l].alloc(ctx, (size_t)std::max<int64_t>(n, 1) * es));
        for (int d = 0; d < W; d++) h_dst[l * W + d] = (char*)x->send[l].p + (size_t)send_off[d] * es;
        h_dst[l * W + me] = layout.dst(ctx->arena_local[x->arena], me, l);
    }
    DevBuf d_dst;
    XchgCols xc;
    TG_TRY(xchg_cols(ctx, x->lanes, h_dst, &d_dst, &xc));
    if (n > 0) TG_TRY(xchg_launch_scatter(ctx, geom, ids_from_key ? nullptr : pids.as<uint8_t>(), n, W, block_off.as<long long>(), xc, &k, p->bucket_count, b2p));
    // 4. hand over to the copy engines.  The event also orders the transfer behind everything enqueued on this context so far:
    //    the readers of the arena this exchange's peers will overwrite NEXT (see the header).
    TG_CUDA(ctx, cudaEventCreateWithFlags(&x->done, cudaEventDisableTiming));
    TG_CUDA(ctx, cudaEventRecord(x->done, ctx->stream));
    TG_CUDA(ctx, cudaStreamWaitEvent(ctx->copy_stream, x->done, 0));
    for (int step = 1; step < W; step++) {
        const int d = (me + step) % W;          // staggered: at any moment every receiver has one sender per step
        if (send_vec[d] == 0) continue;
        for (size_t l = 0; l < L; l++) {
            const size_t es = layout.es[l];
            const char* src = (const char*)x->send[l].p + (size_t)send_off[d] * es;
            TG_CUDA(ctx, cudaMemcpyAsync(layout.dst(ctx->arena_peer[x->arena][d], d, l), src, (size_t)send_vec[d] * es, cudaMemcpyDefault, ctx->copy_stream));
        }
    }
    // 5. barrier: when it completes here, every peer's copies into this rank's arena have completed
    TG_TRY(x->token.alloc(ctx, 16));
    TG_CUDA(ctx, cudaMemsetAsync(x->token.p, 0, 16, ctx->copy_stream));
    TG_NCCL(ctx, g_nccl.all_reduce(x->token.p, (char*)x->token.p + 8, 1, NCCL_INT64, 0 /* ncclSum */, ctx->comm2, ctx->copy_stream));
    TG_CUDA(ctx, cudaEventRecord(x->done, ctx->copy_stream));
    // temporaries of this function (pids, histograms, pointer table) are released in stream order on ctx->stream, behind the
    // scatter; the send buffers and the barrier token are used by the copy stream and live in the handle until _end
    ctx->arena_epoch++;
    ctx->exchanges_in_flight++;
    *out = x.release();
    return TGPU_OK;
}

extern "C" int tgpu_exchange_end(tgpu_ctx* ctx, tgpu_exchange* exchange, tgpu_page** out)
{
    if (!ctx || !exchange || !out) return TGPU_ERR_INVALID_ARGUMENT;
    *out = nullptr;
    std::unique_ptr<tgpu_exchange> x(exchange);
    ctx->exchanges_in_flight--;
    TG_CUDA(ctx, cudaSetDevice(ctx->device));
    if (x->ready) { *out = x->ready; return TGPU_OK; }
    // the received rows are complete once this rank's barrier has run; everything below is ordered behind it on ctx->stream
    TG_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, x->done, 0));
    std::vector<char*> base;
    for (size_t off : x->region_off) base.push_back((char*)ctx->arena_local[x->arena] + off);
    DevPage outp;
    TG_TRY(xchg_page(ctx, x->lanes, base, x->total_recv, nullptr, &outp));     // aliases the arena: valid until the second-next exchange on this context
    OwnedPage* po = tg_make_owned_page(std::move(outp));
    *out = &po->hdr;
    // the send buffers are returned to this context's allocator here: their next use is ordered behind the wait above
    return TGPU_OK;
}
