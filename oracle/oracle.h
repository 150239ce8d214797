/*
 * oracle.h — CPU restatement of the reference (trinodb/trino @ b5a4f5aa) algorithms on the
 * columnar operator hot path.
 *
 * THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only tests/, __graft_entry__.smoke() and
 * bench.py's cpu_baseline / --impl reference legs may load liboracle.so.  The product
 * (libtrino_gpu.so) never links, loads or calls anything in this directory.
 *
 * Parity pinning status (see DESIGN.md §Oracle):
 *   - XXH64: pinned on the reference's own golden vectors
 *     (core/trino-main/src/test/java/io/trino/operator/scalar/TestVarbinaryFunctions.java:776-780)
 *     plus the published xxHash vectors (io.airlift:slice is not vendored under trinodb/trino).
 *   - murmur3 fmix64: restated in-repo at M/operator/join/PagesHash.java:44-50 (pinned by source).
 *   - group ids / join rows / partition lists: pinned on the behavioural cases of the reference's unit
 *     tests (TestGroupByHash, TestHashJoinOperator, TestPagePartitioner) restated in tests/golden/.
 *   - the reference (Java) cannot be built or run in this environment (no JDK): no oracle/_ref.
 *
 * Paths: M/ = core/trino-main/src/main/java/io/trino/, S/ = core/trino-spi/src/main/java/io/trino/spi/.
 * Pages use the same Arrow-layout structs as the product ABI (include/trino_gpu.h), host memory only.
 */
#ifndef TRINO_ORACLE_H
#define TRINO_ORACLE_H

#include <stdint.h>
#include "../include/trino_gpu.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- scalar hash functions (SURVEY.md Appendix A) */
uint64_t orc_hash_long(int64_t v);                 /* S/type/AbstractLongType.java:121-125 */
uint64_t orc_hash_double(double d);                /* S/type/DoubleType.java:199-206 */
uint64_t orc_hash_real(float f);                   /* S/type/RealType.java:151-159 */
uint64_t orc_xxh64(const void* data, int64_t len, uint64_t seed); /* io.airlift.slice.XxHash64 (public XXH64) */
uint64_t orc_xxh64_long(int64_t v);                /* XxHash64.hash(long) = XXH64 of the 8 LE bytes, seed 0 */
uint64_t orc_murmur3(uint64_t x);                  /* M/operator/join/PagesHash.java:44-50 */
uint64_t orc_combine_hash(uint64_t prev, uint64_t v); /* M/operator/scalar/CombineHashFunction.java:29-32 */
int32_t orc_array_size(int64_t expected, double f);   /* fastutil 8.5.18 HashCommon.arraySize; -1 when > 2^30 */
int32_t orc_join_hash_array_size(int64_t n);       /* M/operator/IncrementalLoadFactorHashArraySizeSupplier.java:40-47, multiplier 1 */
int32_t orc_process_raw_hash(int64_t raw_hash, int32_t partition_count); /* M/operator/HashGenerator.java:41-46 */
int32_t orc_local_partition(int64_t raw_hash, int32_t partition_count);  /* M/operator/exchange/LocalPartitionGenerator.java:76-80 */

/* row hashes of a page: M/operator/InterpretedHashGenerator.java:102-110 (null -> 0, h = 31*h + H_type) */
void orc_row_hashes(const tgpu_page* page, const int32_t* channels, int32_t num_channels, int64_t* out);

/* ---- GroupByHash: ids dense, 0-based, first-seen order (M/operator/GroupByHash.java:118-125).
 * kind 0 = auto (GroupByHash.createGroupByHash :82-100: single BIGINT key -> BigintGroupByHash, else FlatGroupByHash),
 * 1 = force BigintGroupByHash (M/operator/BigintGroupByHash.java:191-311), 2 = force FlatHash (M/operator/FlatHash.java:238-423) */
typedef struct orc_groupby orc_groupby;
orc_groupby* orc_groupby_create(int32_t kind, int32_t expected_size);
void orc_groupby_destroy(orc_groupby* g);
/* returns 0, or -3 when the table would exceed 2^30 slots (GENERIC_INSUFFICIENT_RESOURCES) */
int32_t orc_groupby_get_group_ids(orc_groupby* g, const tgpu_page* page, const int32_t* key_channels, int32_t num_keys, int32_t* out_ids);
int32_t orc_groupby_group_count(const orc_groupby* g);
int32_t orc_groupby_capacity(const orc_groupby* g);

/* ---- grouped accumulators: sequential left fold in row order
 * (M/operator/aggregation/GroupedAggregator.java:77-101 + the @InputFunctions cited in trino_gpu.h).
 * state arrays are sized by the caller to group_count. */
void orc_agg_sum_double(const int32_t* gids, int64_t n, const double* v, const uint8_t* validity, const uint8_t* mask_sel, double* sum, uint8_t* nonnull);
void orc_agg_avg_double(const int32_t* gids, int64_t n, const double* v, const uint8_t* validity, const uint8_t* mask_sel, double* sum, int64_t* count);
void orc_agg_count(const int32_t* gids, int64_t n, const uint8_t* validity, const uint8_t* mask_sel, int64_t* count);
/* returns 0 or -4 on overflow (Math.addExact) */
int32_t orc_agg_sum_bigint(const int32_t* gids, int64_t n, const int64_t* v, const uint8_t* validity, const uint8_t* mask_sel, int64_t* sum, uint8_t* nonnull);
void orc_agg_sum_decimal(const int32_t* gids, int64_t n, const int64_t* values, int32_t is_short, const uint8_t* validity, const uint8_t* mask_sel,
                         int64_t* decimal, int64_t* overflow, uint8_t* nonnull);
void orc_agg_sum_decimal_combine(int64_t* decimal, int64_t* overflow, uint8_t* nonnull, const int64_t* other_decimal, int64_t other_overflow);
int32_t orc_decimal_sum_overflows(int64_t high, int64_t low, int64_t overflow);
void orc_agg_minmax_double(const int32_t* gids, int64_t n, const double* v, const uint8_t* validity, int32_t is_max, double* acc, uint8_t* nonnull);
void orc_agg_minmax_bigint(const int32_t* gids, int64_t n, const int64_t* v, const uint8_t* validity, int32_t is_max, int64_t* acc, uint8_t* nonnull);

/* ---- hash join (M/operator/join/BigintPagesHash.java, DefaultPagesHash.java, ArrayPositionLinks.java, JoinHash.java) */
typedef struct orc_join orc_join;
/* build over one concatenated build page; address index == row number (M/operator/SyntheticAddress.java).
 * force_default == 1 selects DefaultPagesHash even for a single BIGINT key (as JoinHashSupplier.java:162-168 does above 2^20 rows);
 * force_default == 2 keeps the BigintPagesHash layout at any size (the timing leg: it is the faster of the two on a CPU) */
orc_join* orc_join_build(const tgpu_page* build, const int32_t* key_channels, int32_t num_keys, int32_t force_default);
void orc_join_destroy(orc_join* j);
int32_t orc_join_hash_size(const orc_join* j);
int32_t orc_join_has_links(const orc_join* j);               /* !positionLinks.isEmpty() */
void orc_join_copy_links(const orc_join* j, int32_t* out);   /* -1 = end of chain */
/* JoinProbe.fillCache + LookupSource.getJoinPosition: chain head address index or -1 per probe row
 * (NULL in any key column -> -1, M/operator/join/unspilled/JoinProbe.java:154-171) */
void orc_join_positions(const orc_join* j, const tgpu_page* probe, const int32_t* key_channels, int32_t* out);
/* PageJoiner.processProbe expansion (M/operator/join/unspilled/PageJoiner.java:138-258): emits
 * (probe row, build row) pairs in reference order; build row -1 = appendNullForBuild.
 * Returns the number of pairs (call with capacity 0 to count). */
int64_t orc_join_expand(const orc_join* j, const int32_t* join_positions, int64_t num_probe_rows, int32_t join_type, int32_t single_match,
                        int32_t* out_probe, int32_t* out_build, int64_t capacity);

/* HashSemiJoinOperator.process (M/operator/HashSemiJoinOperator.java:181-199) over a ChannelSet of BIGINT values
 * (M/operator/ChannelSet.java:43-61, FlatSet.java:120-153: size counts the NULL once).  validity: Arrow bitmaps or NULL.
 * out_value[i] = the BOOLEAN, out_null[i] = 1 when the result is NULL. */
void orc_semi_join_bigint(const int64_t* set_values, const uint8_t* set_validity, int64_t set_rows, const int64_t* probe, const uint8_t* probe_validity,
                          int64_t probe_rows, int8_t* out_value, uint8_t* out_null);
/* the same over a DOUBLE (kind 1) or REAL (kind 2) channel given as raw IEEE bits: IDENTICAL membership (NaN is a member like any other) */
void orc_semi_join_float(int32_t kind, const void* set_values, const uint8_t* set_validity, int64_t set_rows, const void* probe, const uint8_t* probe_validity,
                         int64_t probe_rows, int8_t* out_value, uint8_t* out_null);
/* multi-threaded probe timing leg for the CPU baseline: `threads` workers each take 8192-row pages
 * (BigintPagesHash.getAddressIndex(int[],Page) 3-phase batching); returns seconds */
double orc_join_probe_timed(const orc_join* j, const int64_t* probe_keys, int64_t n, int32_t threads, int32_t* out,
                            const int32_t* build_payload, int32_t* out_payload);
/* force BigintPagesHash layout (keys[] + values[]) regardless of size: the timing leg probes BIGINT keys */

/* ---- the stable CPU timing arm: a PartitionedLookupSource (M/operator/join/unspilled/PartitionedLookupSource.java:97-186) of
 * `partitions` (rounded up to a power of two) lookup sources, each built by its own builder thread over its own slice of the build
 * side (one HashBuilderOperator per partition behind the local exchange, LocalPartitionGenerator.java:76-80; BigintPagesHash up to
 * 2^20 positions per partition, DefaultPagesHash above, JoinHashSupplier.java:162-168), probed by a persistent pool of `threads`
 * drivers on 8192-row pages.  Single BIGINT join channel without NULLs, unique build keys, one INT32 build output channel. */
typedef struct orc_pjoin orc_pjoin;
orc_pjoin* orc_pjoin_build(const int64_t* build_keys, const int32_t* build_payload, int64_t n, int32_t partitions, int32_t threads, double* seconds_out);
void orc_pjoin_destroy(orc_pjoin* j);
int32_t orc_pjoin_partitions(const orc_pjoin* j);
int32_t orc_pjoin_threads(const orc_pjoin* j);
/* zero-fill a caller-allocated probe-side array with the page -> worker assignment of orc_pjoin_probe (NUMA first touch) */
void orc_pjoin_touch(orc_pjoin* j, void* base, int64_t bytes_per_row, int64_t n);
/* one pass of the probe drivers: out_positions[i] = encodePartitionedJoinPosition(partition, joinPosition) or -1
 * (PartitionedLookupSource.java:259-262), out_payload[i] = the build output value of the match (0 when none).  Outputs are
 * caller-allocated (pre-touched); nothing is allocated or spawned inside the timed region.  Returns seconds. */
double orc_pjoin_probe(orc_pjoin* j, const int64_t* probe_keys, int64_t n, int64_t* out_positions, int32_t* out_payload);
/* decodePartition / decodeJoinPosition (:264-275) mapped back to rows of the unpartitioned build side, for verification */
void orc_pjoin_decode(const orc_pjoin* j, const int64_t* positions, int64_t n, int32_t* out_rows);

/* ---- PagePartitioner (M/operator/output/PagePartitioner.java:133-162,229-433) */
/* partition id per row: bucketToPartition[processRawHash(rowHash, bucketCount)] */
void orc_partition_ids(const tgpu_page* page, const int32_t* key_channels, int32_t num_keys, int32_t bucket_count,
                       const int32_t* bucket_to_partition, int32_t* out);
/* per-partition position lists in reference order.  `any_row_replicated` is the
 * hasAnyRowBeenReplicated state (in/out).  out_offsets has partition_count+1 entries;
 * out_positions must hold num_rows + (partition_count * (1 + null rows)) entries. */
void orc_partition_positions(const tgpu_page* page, const int32_t* key_channels, int32_t num_keys, int32_t bucket_count,
                             const int32_t* bucket_to_partition, int32_t partition_count, int32_t null_channel,
                             int32_t replicates_any_row, int32_t* any_row_replicated,
                             int64_t* out_offsets, int32_t* out_positions);

/* ---- TPC-H Q1 pipeline (scan -> filter -> project -> GROUP BY) structured like the reference:
 * `threads` drivers each run filter (M/sql/gen/columnar/ColumnarFilter.java:43-53), unfused FP64
 * projections (M/type/DoubleOperators.java:66-86), FlatHash group ids on 1024-row batches
 * (M/operator/FlatGroupByHash.java:515-540) and one accumulator pass per aggregate
 * (M/operator/aggregation/GroupedAggregator.java:77-101) as a PARTIAL step, then a FINAL merge.
 * Keys are VARCHAR(1) (hashed with XXH64 of the byte).  Output rows in first-seen group order of the
 * thread-0-first merge; out arrays sized max_groups.  Returns seconds spent (wall). */
typedef struct orc_q1_result {
    int32_t num_groups;
    int8_t returnflag[16];
    int8_t linestatus[16];
    double sum_qty[16], sum_base_price[16], sum_disc_price[16], sum_charge[16];
    double avg_qty[16], avg_price[16], avg_disc[16];
    int64_t count_order[16];
} orc_q1_result;
double orc_q1_run(int64_t n, const int32_t* shipdate, const int8_t* returnflag, const int8_t* linestatus,
                  const double* quantity, const double* extendedprice, const double* discount, const double* tax,
                  int32_t shipdate_cutoff, int32_t threads, orc_q1_result* out);

/* ---- synthetic generators, identical to the device generators (SURVEY.md §8d) */
uint64_t orc_splitmix64(uint64_t x);
void orc_synth_orders_keys(int64_t n_total, int64_t first, int64_t count, uint64_t seed, int32_t shuffle, int64_t* out);
int64_t orc_synth_lineitem_rows(int64_t n_orders);
void orc_synth_lineitem_keys(int64_t n_orders, int64_t first, int64_t count, uint64_t seed, int32_t shuffle, int64_t* out);
void orc_synth_lineitem_q1(int64_t n, int64_t first, uint64_t seed, int32_t* shipdate, int8_t* returnflag, int8_t* linestatus,
                           double* quantity, double* extendedprice, double* discount, double* tax);

void orc_synth_orders_custkeys(int64_t n_total, int64_t first, int64_t count, uint64_t seed, int32_t shuffle, int64_t n_customers, uint64_t cust_seed, int64_t* out);
/* returns the number of rows whose two nullable keys are both present */
int64_t orc_synth_store_sales(int64_t n, int64_t first, uint64_t seed, int64_t* date_sk, int64_t* item_sk, int64_t* customer_sk, uint8_t* customer_valid,
                              int64_t* store_sk, uint8_t* store_valid, double* net_paid);

int32_t orc_hardware_threads(void);

#ifdef __cplusplus
}
#endif
#endif
