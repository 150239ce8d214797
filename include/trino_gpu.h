/*
 * trino_gpu.h — C ABI of libtrino_gpu.so: the H100 (sm_90a) implementation of Trino's
 * columnar operator hot path.
 *
 * The reference has no FFI for this path (SURVEY.md §8b): operators are Java classes that
 * implement io.trino.operator.Operator / OperatorFactory.  Every entry point below is what a
 * thin Java Operator (see INTEGRATION.md, java/) binds through Panama/JNI, and each cites the
 * reference interface it stands in for (paths relative to
 * trinodb/trino/core/trino-main/src/main/java/io/trino/ = M/, .../trino-spi/.../spi/ = S/).
 *
 * Conventions
 *   - plain C, plain pointers and sizes; no C++/torch types.
 *   - every call returns TGPU_OK (0) or a negative tgpu_status; tgpu_last_error() gives text.
 *   - a handle is used by one thread at a time (mirrors @NotThreadSafe Operator, M/operator/Driver.java:298);
 *     distinct handles may be used concurrently.
 *   - pages are Arrow-layout column buffers.  Host pages are copied to the device inside
 *     add_input; pages flagged TGPU_PAGE_DEVICE already live in HBM and are consumed in place.
 *   - lifetime of TGPU_PAGE_DEVICE inputs.  When the input IS a page this library returned (the tgpu_page* of
 *     tgpu_op_get_output / tgpu_exchange_*, passed on unchanged: GPU -> GPU operator chaining), the consumer shares
 *     ownership of its buffers and the caller may release the page right after add_input, as Operator.addInput
 *     allows (M/operator/Operator.java:60-66).  Any other device page (descriptors the caller built around its own
 *     device memory) is BORROWED: the memory must stay allocated while an operator can still read it - until the
 *     lookup source is released for a join build side (PagesIndex keeps block references, M/operator/PagesIndex.java:224-256),
 *     until the output page is released for operators that pass input blocks through (LookupJoinOperator 1:1 outputs,
 *     HashSemiJoinOperator, pass-through projections, a single-partition PartitionedOutput), and until add_input
 *     returns otherwise.  Pages returned by the exchange alias a receive arena and follow the arena rule stated there.
 *   - there is NO CPU fallback: without a CUDA device every create call fails with TGPU_ERR_CUDA.
 */
#ifndef TRINO_GPU_H
#define TRINO_GPU_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------ status / error codes */
typedef enum tgpu_status {
    TGPU_OK = 0,
    TGPU_ERR_INVALID_ARGUMENT = -1,       /* IllegalArgumentException / checkArgument */
    TGPU_ERR_CUDA = -2,                   /* GENERIC_INTERNAL_ERROR: device failure, no device, OOM on device */
    TGPU_ERR_INSUFFICIENT_RESOURCES = -3, /* GENERIC_INSUFFICIENT_RESOURCES (M/operator/BigintGroupByHash.java:242, M/operator/PagesIndex.java:247) */
    TGPU_ERR_NUMERIC_VALUE_OUT_OF_RANGE = -4, /* NUMERIC_VALUE_OUT_OF_RANGE (M/type/BigintOperators.java:52-84) */
    TGPU_ERR_DIVISION_BY_ZERO = -5,       /* DIVISION_BY_ZERO (M/type/BigintOperators.java:96-106) */
    TGPU_ERR_NOT_SUPPORTED = -6,          /* NOT_SUPPORTED: caller keeps the Java operator */
    TGPU_ERR_ILLEGAL_STATE = -7           /* IllegalStateException / checkState (protocol misuse) */
} tgpu_status;

/* ------------------------------------------------------------------ columnar data model
 * Stands in for S/Page.java:31 and the Block family (S/block/LongArrayBlock.java:36-41,
 * IntArrayBlock, ShortArrayBlock, ByteArrayBlock, VariableWidthBlock.java:41-46,
 * DictionaryBlock.java:37-40, RunLengthEncodedBlock.java:71-72).                       */
typedef enum tgpu_type {
    TGPU_INT64 = 1,    /* BIGINT, short DECIMAL, TIMESTAMP(millis)…  (LongArrayBlock)          */
    TGPU_INT32 = 2,    /* INTEGER, DATE                              (IntArrayBlock)           */
    TGPU_INT16 = 3,    /* SMALLINT                                   (ShortArrayBlock)         */
    TGPU_INT8 = 4,     /* TINYINT, BOOLEAN                           (ByteArrayBlock)          */
    TGPU_FLOAT64 = 5,  /* DOUBLE, raw IEEE bits in a LongArrayBlock (S/type/DoubleType.java:205) */
    TGPU_UTF8 = 7,     /* VARCHAR / CHAR / VARBINARY: int32 offsets[length+1] + bytes          */
    TGPU_DICT32 = 8,   /* DictionaryBlock: data = int32 ids[length], dictionary = value column */
    TGPU_RLE = 9,      /* RunLengthEncodedBlock: dictionary = 1-row value column, broadcast    */
    TGPU_INT128 = 10,  /* long DECIMAL(p > 18): Int128ArrayBlock's long[] - 16 bytes per position, the HIGH (signed) word first, then the
                          LOW word (S/block/Int128ArrayBlock.java:123-133).  Moves through every operator; hashes and compares as
                          LongDecimalType does (S/type/LongDecimalType.java:203-247); group-by / join / partition key; sum() input and
                          output (DecimalSumAggregation).  The expression evaluator does not compute on it.                          */
    TGPU_FLOAT32 = 11  /* REAL: the float's raw IEEE bits in an IntArrayBlock (S/type/RealType.java:104-121).  Moves through every
                          operator; partition / join / group-by key with RealType's operators (hash :151-159 over floatToIntBits with
                          -0.0 collapsed; EQUAL :145-149 - NaN matches nothing; IDENTICAL :172-185 - NaN is identical to NaN).  Join and
                          group-by widen the key to its (exact) double internally; a semi-join set over REAL or DOUBLE answers NaN
                          probes by IDENTICAL like the ChannelSet.  Aggregates and expressions over REAL and REAL dynamic-filter
                          domains answer TGPU_ERR_NOT_SUPPORTED.                                                                   */
} tgpu_type;

enum {
    TGPU_COL_NULLS_BYTEMAP = 1 /* `validity` points at Java's boolean[] valueIsNull (1 byte/position,
                                  1 = NULL) instead of an Arrow LSB bitmap (1 bit/position, 1 = valid) */
};

typedef struct tgpu_column {
    int32_t type;                         /* tgpu_type */
    int32_t flags;                        /* TGPU_COL_* */
    int64_t length;                       /* positions */
    const void* data;                     /* values; int32 ids for DICT32; bytes for UTF8; unused for RLE */
    const int32_t* offsets;               /* UTF8 only: length+1 entries */
    const uint8_t* validity;              /* NULL = no nulls */
    const struct tgpu_column* dictionary; /* DICT32: dictionary values; RLE: the single value */
} tgpu_column;

enum {
    TGPU_PAGE_DEVICE = 1 /* all buffers referenced by the page are device pointers (GPU->GPU operator
                            chaining and the device-resident benchmark path) */
};

typedef struct tgpu_page {
    int32_t num_columns;
    int32_t flags;                        /* TGPU_PAGE_* */
    int64_t num_rows;                     /* Page.getPositionCount() */
    const tgpu_column* columns;
} tgpu_page;

typedef struct tgpu_ctx tgpu_ctx;         /* one per (process, device): stream, memory pool, error slot */
typedef struct tgpu_op tgpu_op;           /* one Operator instance */
typedef struct tgpu_lookup tgpu_lookup;   /* built join table: LookupSource (M/operator/join/LookupSource.java:24-68) */

/* ------------------------------------------------------------------ context */
int tgpu_ctx_create(int device, tgpu_ctx** out);
void tgpu_ctx_destroy(tgpu_ctx* ctx);
const char* tgpu_last_error(const tgpu_ctx* ctx);     /* message of the last failing call on ctx */
const char* tgpu_status_name(int status);             /* Trino StandardErrorCode name */
int tgpu_ctx_synchronize(tgpu_ctx* ctx);              /* cudaStreamSynchronize on the ctx stream */
void* tgpu_ctx_stream(tgpu_ctx* ctx);                 /* the cudaStream_t every kernel of ctx is launched on */
int64_t tgpu_ctx_kernel_launches(const tgpu_ctx* ctx);/* number of kernels this library launched on ctx */
int tgpu_device_count(void);
/* tuning knob: cudaLimitMaxL2FetchGranularity (32/64/128 bytes pulled from HBM per missing L2 sector) */
int tgpu_ctx_set_l2_fetch_granularity(tgpu_ctx* ctx, int bytes);
int tgpu_ctx_get_l2_fetch_granularity(tgpu_ctx* ctx, int* bytes);

/* device memory helpers for the device-resident path (bench, GPU->GPU chaining, tests) */
int tgpu_malloc(tgpu_ctx* ctx, size_t bytes, void** out);
int tgpu_free(tgpu_ctx* ctx, void* ptr);
int tgpu_memcpy_h2d(tgpu_ctx* ctx, void* dst, const void* src, size_t bytes);
int tgpu_memcpy_d2h(tgpu_ctx* ctx, void* dst, const void* src, size_t bytes);
int tgpu_host_alloc_pinned(size_t bytes, void** out);
int tgpu_host_free_pinned(void* ptr);
/* write a buffer larger than L2 (bench hygiene between timed iterations) */
int tgpu_flush_l2(tgpu_ctx* ctx);
/* device timing on the ctx stream (cudaEvent pair) */
int tgpu_timer_start(tgpu_ctx* ctx);
int tgpu_timer_stop_ms(tgpu_ctx* ctx, float* ms);
/* device time (CUDA events on the ctx stream) of the dominant kernel launched by the last operator call */
int tgpu_ctx_last_kernel_ms(tgpu_ctx* ctx, float* ms);

/* ------------------------------------------------------------------ expressions (PageProcessor)
 * Stands in for the compiled PageFilter/PageProjection pair produced by
 * ExpressionCompiler.compilePageProcessor (M/sql/gen/ExpressionCompiler.java:50-85) from the
 * RowExpression trees at M/sql/planner/LocalExecutionPlanner.java:2111-2127.
 * A program is three-address code over per-row temporaries; operands are an input channel, an
 * immediate, or a temporary.  Value types inside the VM: BIGINT (all integer widths are sign-extended
 * on load), DOUBLE, BOOLEAN; every value carries a null flag (SQL three-valued logic).          */
typedef enum tgpu_expr_op {
    TGPU_EX_MOV = 0,
    TGPU_EX_ADD = 1, TGPU_EX_SUB = 2, TGPU_EX_MUL = 3, TGPU_EX_DIV = 4, TGPU_EX_MOD = 5, TGPU_EX_NEG = 6,
    TGPU_EX_EQ = 10, TGPU_EX_NE = 11, TGPU_EX_LT = 12, TGPU_EX_LE = 13, TGPU_EX_GT = 14, TGPU_EX_GE = 15,
    TGPU_EX_AND = 20, TGPU_EX_OR = 21, TGPU_EX_NOT = 22,
    TGPU_EX_IS_NULL = 23, TGPU_EX_IS_NOT_NULL = 24,
    TGPU_EX_BETWEEN = 25,          /* a BETWEEN b AND c: c in operand `c` */
    TGPU_EX_CAST_BIGINT_TO_DOUBLE = 30,
    TGPU_EX_CAST_DOUBLE_TO_BIGINT = 31, /* Math.round semantics, range-checked (M/type/DoubleOperators.java) */
    TGPU_EX_IN = 40                /* a IN (const list): b.imm = index into in_lists, all operands of `vtype` */
} tgpu_expr_op;

typedef enum tgpu_vtype { TGPU_V_BIGINT = 0, TGPU_V_DOUBLE = 1, TGPU_V_BOOLEAN = 2 } tgpu_vtype;
typedef enum tgpu_operand_kind { TGPU_OPND_NONE = 0, TGPU_OPND_COLUMN = 1, TGPU_OPND_TEMP = 2, TGPU_OPND_CONST = 3, TGPU_OPND_NULL = 4 } tgpu_operand_kind;

typedef struct tgpu_operand {
    int32_t kind;                         /* tgpu_operand_kind */
    int32_t index;                        /* channel or temp slot */
    union { int64_t i64; double f64; } imm;
} tgpu_operand;

typedef struct tgpu_expr_insn {
    int32_t op;                           /* tgpu_expr_op */
    int32_t vtype;                        /* tgpu_vtype of the OPERANDS (result of comparisons is BOOLEAN) */
    int32_t dst;                          /* temp slot written, 0..TGPU_MAX_TEMPS-1 */
    int32_t reserved;
    tgpu_operand a, b, c;
} tgpu_expr_insn;

#define TGPU_MAX_TEMPS 8
#define TGPU_MAX_INSNS 64
#define TGPU_MAX_CHANNELS 32

typedef struct tgpu_in_list { int32_t count; const int64_t* values; /* raw bits for DOUBLE */ } tgpu_in_list;

typedef struct tgpu_projection {
    int32_t kind;        /* 0 = pass an input channel through (any type incl. UTF8/DICT/RLE, like InputPageProjection);
                            1 = computed: value of temp `index` after the program ran */
    int32_t index;       /* channel or temp */
    int32_t vtype;       /* computed only: result type (BIGINT->INT64, DOUBLE->FLOAT64, BOOLEAN->INT8) */
} tgpu_projection;

typedef struct tgpu_expr_program {
    int32_t num_insns;
    const tgpu_expr_insn* insns;
    int32_t filter_temp;                  /* temp holding the BOOLEAN filter result, or -1 = no filter.
                                             NULL or FALSE rejects the row (M/sql/gen/columnar/ColumnarFilter.java:27-30) */
    int32_t num_filter_insns;             /* insns [0, num_filter_insns) compute the filter and run for every row; the
                                             remaining insns (projections) run, and may raise errors, only for selected
                                             rows (PageProcessor filters first: M/operator/project/PageProcessor.java:126-142) */
    int32_t num_projections;
    const tgpu_projection* projections;
    int32_t num_in_lists;
    const tgpu_in_list* in_lists;
} tgpu_expr_program;

/* FilterAndProjectOperator (M/operator/FilterAndProjectOperator.java:60-95) over a PageProcessor
 * (M/operator/project/PageProcessor.java:105-142).  Output: one page per non-empty input page.  */
int tgpu_filter_project_create(tgpu_ctx* ctx, const tgpu_expr_program* program, tgpu_op** out);

/* ------------------------------------------------------------------ hash aggregation
 * Stands in for HashAggregationOperator (M/operator/HashAggregationOperator.java:346-498) +
 * InMemoryHashAggregationBuilder (M/operator/aggregation/builder/InMemoryHashAggregationBuilder.java:141-300)
 * + GroupByHash (M/operator/GroupByHash.java:82-125) + the grouped accumulators
 * (M/operator/aggregation/GroupedAggregator.java:77-117).                                        */
typedef enum tgpu_agg_function {
    TGPU_AGG_COUNT_STAR = 0,  /* CountAggregation.java:36-51    -> BIGINT                       */
    TGPU_AGG_COUNT = 1,       /* CountColumn.java               -> BIGINT (non-null inputs)     */
    TGPU_AGG_SUM = 2,         /* DoubleSumAggregation.java:37-63 / BigintSumAggregation.java:38-59 (checked) */
    TGPU_AGG_AVG = 3,         /* DoubleAverageAggregations.java:37-63 (DOUBLE input) / LongAverage (BIGINT input) */
    TGPU_AGG_MIN = 4,
    TGPU_AGG_MAX = 5,
    TGPU_AGG_SUM_DECIMAL = 6, /* DecimalSumAggregation.java:44-146: input TGPU_INT64 (short decimal) or TGPU_INT128 (long decimal) -> DECIMAL(38, s)
                                 as TGPU_INT128; "Decimal overflow" (NUMERIC_VALUE_OUT_OF_RANGE) when the sum leaves +-10^38                   */
    TGPU_AGG_AVG_DECIMAL = 7  /* DecimalAverageAggregation.java:54-176: same inputs -> DECIMAL(p, s) of the input: sum / count rounded HALF_UP, as
                                 TGPU_INT64 for a short decimal and TGPU_INT128 for a long one (tgpu_agg_fn.reserved names the result type in a
                                 FINAL step, where the state no longer tells)                                                                   */
} tgpu_agg_function;

typedef enum tgpu_agg_step {   /* M/sql/planner/plan/AggregationNode.java:361-402 */
    TGPU_STEP_SINGLE = 0,      /* raw input -> final output                                   */
    TGPU_STEP_PARTIAL = 1,     /* raw input -> intermediate state columns                     */
    TGPU_STEP_FINAL = 2,       /* intermediate state columns -> final output                  */
    TGPU_STEP_INTERMEDIATE = 3 /* intermediate -> intermediate                                */
} tgpu_agg_step;

typedef struct tgpu_agg_fn {
    int32_t function;          /* tgpu_agg_function */
    int32_t input_channel;     /* -1 for count(*).  For FINAL/INTERMEDIATE: first channel of the state columns */
    int32_t mask_channel;      /* -1 or a BOOLEAN channel (AggregationMask, M/operator/aggregation/AggregationMask.java:30-100) */
    int32_t reserved;          /* TGPU_AGG_AVG_DECIMAL: tgpu_type of the result (TGPU_INT64 / TGPU_INT128); 0 = as the input channel */
} tgpu_agg_fn;

/* Intermediate state layout emitted by PARTIAL and consumed by FINAL (one or two flat columns per
 * aggregate, the Arrow-side flattening of the reference's state serializers):
 *   count/count(*) : INT64 count
 *   sum            : value (INT64 or FLOAT64), NULL when no input rows (NullableDoubleState / NullableLongState)
 *   avg            : INT64 count, FLOAT64 sum (LongAndDoubleState)
 *   min/max        : value, NULL when no input rows
 *   sum (decimal)  : TGPU_INT128 sum, INT64 overflow (LongDecimalWithOverflowState: total = sum + overflow * 2^128); the sum is NULL
 *                    when no input rows
 *   avg (decimal)  : TGPU_INT128 sum, INT64 overflow, INT64 count (LongDecimalWithOverflowAndLongState)
 * Variable-width (TGPU_UTF8) group-by keys are supported: each such key column owns a device string dictionary
 * (csrc/strdict.cuh, the AppendOnlyVariableWidthData analogue of M/operator/FlatHash.java:309-348); identity is exact
 * (full-byte comparison, colliding strings rehash), output key columns are UTF8 again.                                 */
typedef struct tgpu_agg_spec {
    int32_t num_keys;
    const int32_t* key_channels;  /* groupByChannels */
    int32_t step;                 /* tgpu_agg_step */
    int32_t num_aggs;
    const tgpu_agg_fn* aggs;
    int64_t expected_groups;      /* expectedGroups, sizes the table like arraySize(expected, 0.75) */
    int64_t max_partial_bytes;    /* task.max-partial-aggregation-memory (PARTIAL flush threshold); 0 = never flush */
    /* optional fused pre-stage: filter + projections evaluated in registers in the same kernel that
       aggregates, so projected columns never reach HBM (ScanFilterAndProject -> HashAggregation chain of Q1).
       When set, key_channels / input_channel refer to the program's projection outputs.        */
    const tgpu_expr_program* pre;
    /* global grouping sets (GROUPING SETS / ROLLUP / CUBE with an empty set): when no row reaches a SINGLE / FINAL step the operator
       emits one default row per listed id - the $group_id key holds the id, the other keys are NULL, count is 0 and every other
       aggregate NULL (HashAggregationOperator.getGlobalAggregationOutput, M/operator/HashAggregationOperator.java:466-470,537-567).
       group_id_key indexes key_channels (groupIdChannel); input_channel_types (tgpu_type per aggregation-input channel - the
       operator's source types at LocalExecutionPlanner.java:4086-4089) shapes those rows, as no page was ever seen.  All optional. */
    int32_t num_global_group_ids;
    const int32_t* global_group_ids;      /* globalAggregationGroupIds */
    int32_t group_id_key;
    int32_t num_input_channels;
    const int32_t* input_channel_types;
    /* adaptive partial aggregation (PARTIAL / INTERMEDIATE steps only, else INVALID_ARGUMENT - the reference's
       checkArgument at M/operator/HashAggregationOperator.java:296).  When the shared controller says partial aggregation is
       disabled at the moment a new aggregation builder would be created (:358-372), the operator runs that builder as a
       SkipAggregationBuilder (M/operator/aggregation/partial/SkipAggregationBuilder.java:103-131): add_input takes ONE page,
       needs_input turns false, get_output returns one page of the same row count - the key channels passed through, and per
       aggregate the intermediate state of a group that holds just that row.  NULL = no controller.  Not owned by the operator. */
    struct tgpu_partial_agg_controller* partial_aggregation_controller;
} tgpu_agg_spec;

/* PartialAggregationController (M/operator/aggregation/partial/PartialAggregationController.java:35-103): one per plan node
 * and task, shared by that node's drivers; thread-safe.  Partial aggregation is switched off once at least
 * 1.5 x max_partial_memory_bytes of input were aggregated and unique rows / input rows exceeds the threshold, and switched back
 * on (counters reset) after 300 x max_partial_memory_bytes of input.  The operators call on_flush themselves
 * (HashAggregationOperator.closeAggregationBuilder :512-523); the entry point is public for callers that mix CPU and GPU
 * drivers under one controller.  unique_rows_produced < 0 stands for OptionalLong.empty() (a skipped builder). Needs no GPU. */
typedef struct tgpu_partial_agg_controller tgpu_partial_agg_controller;
int tgpu_partial_agg_controller_create(int64_t max_partial_memory_bytes, double unique_rows_ratio_threshold, tgpu_partial_agg_controller** out);
void tgpu_partial_agg_controller_destroy(tgpu_partial_agg_controller* controller);
int tgpu_partial_agg_controller_is_disabled(const tgpu_partial_agg_controller* controller);
void tgpu_partial_agg_controller_on_flush(tgpu_partial_agg_controller* controller, int64_t bytes_processed, int64_t rows_processed, int64_t unique_rows_produced);
/* AggregationMetrics.recordInputRowsProcessedWithPartialAggregationDisabled: rows this operator passed through un-aggregated */
int tgpu_agg_rows_with_partial_aggregation_disabled(tgpu_op* op, int64_t* out);

int tgpu_agg_create(tgpu_ctx* ctx, const tgpu_agg_spec* spec, tgpu_op** out);
/* diagnostics (needs no GPU): generate the kernel specialised for `spec` over input channels of the given tgpu_types
 * (bit c of nullable_mask = channel c carries NULLs), compile it with NVRTC for sm_90a; returns the cubin size and
 * the generated source (or the compiler log on failure) */
int tgpu_jit_selftest_agg(const tgpu_agg_spec* spec, const int32_t* channel_types, int32_t num_channels, uint32_t nullable_mask,
                          int64_t* cubin_bytes, char* source_out, int64_t source_cap);
/* Same for the FilterAndProject kernels generated from `program` (tg_fp_filter_jit / tg_fp_project_jit). */
int tgpu_jit_selftest_filter_project(const tgpu_expr_program* program, const int32_t* channel_types, int32_t num_channels, uint32_t nullable_mask,
                                     int64_t* cubin_bytes, char* source_out, int64_t source_cap);
/* GroupByHash.getGroupCount() */
int tgpu_agg_group_count(tgpu_op* op, int64_t* out);

/* GroupByHash.getGroupIds(Page) alone (M/operator/GroupByHash.java:118-125): dense ids in
 * first-seen order for the key columns of `page`, written to `out_group_ids` (host or device to
 * match the page).  The table persists in the handle across calls, like the Java object.        */
int tgpu_groupby_hash_create(tgpu_ctx* ctx, int32_t num_keys, const int32_t* key_channels, int64_t expected_groups, tgpu_op** out);
int tgpu_groupby_hash_get_group_ids(tgpu_op* op, const tgpu_page* page, int32_t* out_group_ids);

/* ------------------------------------------------------------------ hash join
 * Build: HashBuilderOperator (M/operator/join/unspilled/HashBuilderOperator.java:253-333) over
 * PagesIndex (M/operator/PagesIndex.java:224-256,523-542) producing a JoinHash
 * (M/operator/join/JoinHash.java) = PagesHash (BigintPagesHash.java:62-141 / DefaultPagesHash.java:61-144)
 * + ArrayPositionLinks (M/operator/join/ArrayPositionLinks.java:45-104).
 * Probe: LookupJoinOperator (M/operator/join/unspilled/LookupJoinOperator.java:52-80) =
 * JoinProbe.fillCache (JoinProbe.java:112-180) + PageJoiner (PageJoiner.java:93-258) +
 * LookupJoinPageBuilder (LookupJoinPageBuilder.java:89-160).                                     */
typedef enum tgpu_join_type {  /* M/operator/join/LookupJoinOperatorFactory.JoinType */
    TGPU_JOIN_INNER = 0,
    TGPU_JOIN_PROBE_OUTER = 1,
    TGPU_JOIN_LOOKUP_OUTER = 2,   /* JoinOperatorType.lookupOuterJoin: INNER on the probe side + visited build positions */
    TGPU_JOIN_FULL_OUTER = 3      /* JoinOperatorType.fullOuterJoin: PROBE_OUTER on the probe side + visited build positions */
} tgpu_join_type;

typedef struct tgpu_join_build_spec {
    int32_t num_key_channels;
    const int32_t* key_channels;      /* hashChannels of the build pages */
    int32_t num_output_channels;
    const int32_t* output_channels;   /* build columns appended to each output row */
    int64_t expected_positions;       /* expectedPositions (sizing hint only) */
} tgpu_join_build_spec;

typedef struct tgpu_join_probe_spec {
    int32_t join_type;                /* tgpu_join_type */
    int32_t output_single_match;      /* outputSingleMatch (semi-join style: first match only) */
    int32_t num_key_channels;
    const int32_t* key_channels;      /* probeJoinChannels */
    int32_t num_output_channels;
    const int32_t* output_channels;   /* probeOutputChannels; output page = these, then the build output channels */
} tgpu_join_probe_spec;

int tgpu_join_build_create(tgpu_ctx* ctx, const tgpu_join_build_spec* spec, tgpu_op** out);
/* valid after finish(): lendPartitionLookupSource (PartitionedLookupSourceFactory.java:100).  The
 * lookup stays alive until tgpu_lookup_release, independent of the build operator handle.       */
int tgpu_join_build_get_lookup(tgpu_op* build, tgpu_lookup** out);
void tgpu_lookup_release(tgpu_lookup* lookup);
int64_t tgpu_lookup_position_count(const tgpu_lookup* lookup);   /* LookupSource.getJoinPositionCount */
int64_t tgpu_lookup_memory_bytes(const tgpu_lookup* lookup);     /* getInMemorySizeInBytes */
int tgpu_lookup_has_duplicates(const tgpu_lookup* lookup);       /* !positionLinks.isEmpty() */
int tgpu_join_probe_create(tgpu_ctx* ctx, const tgpu_join_probe_spec* spec, tgpu_lookup* lookup, tgpu_op** out);
/* LookupJoinPageBuilder.build (M/operator/join/LookupJoinPageBuilder.java:144-150) returns the probe blocks themselves when
 * every probe row produced exactly one output row.  With this switch on, a HOST probe page only has its join-key channel
 * uploaded; when the output is such a 1:1 page its pass-through columns carry no device data (data == NULL): the caller
 * substitutes its own input blocks (tgpu_page_passthrough_channel) and passes data == NULL for them to
 * tgpu_page_copy_to_host.  When rows were dropped or repeated the remaining channels are uploaded after all and the output is
 * complete.  Off by default (every output column is materialised on the device); single-channel BIGINT-family keys only. */
int tgpu_join_probe_set_passthrough_by_reference(tgpu_op* probe, int32_t enable);

/* LookupOuterOperator (M/operator/join/LookupOuterOperator.java:170-206, OuterLookupSource.java:109-196): a source operator
 * that, once every LOOKUP_OUTER / FULL_OUTER probe of `lookup` has finished (the caller's outerPositionsFuture), returns the build
 * rows no probe emitted, in build position order: `num_probe_outputs` all-NULL columns of the given tgpu_type, then the build
 * output channels.  One page; getOutput then returns NULL and isFinished is true. */
int tgpu_join_outer_create(tgpu_ctx* ctx, tgpu_lookup* lookup, const int32_t* probe_output_types, int32_t num_probe_outputs, tgpu_op** out);

/* HashSemiJoinOperator (M/operator/HashSemiJoinOperator.java:155-201): `lookup` is built by a hash builder over the filtering
 * source's join channel (SetBuilderOperator's ChannelSet; no output channels needed).  Output = the input page's columns + one
 * BOOLEAN (TGPU_INT8) column: NULL probe key -> false if the set is empty else NULL; otherwise contained -> true, not contained ->
 * NULL if the set holds a NULL else false.  DOUBLE / REAL keys: membership is IDENTICAL as in the ChannelSet's FlatSet
 * (M/operator/FlatSet.java:54,374) - a NaN probe key is contained iff the set holds a NaN, -0.0 and +0.0 are one member. */
int tgpu_semi_join_create(tgpu_ctx* ctx, tgpu_lookup* lookup, int32_t probe_join_channel, tgpu_op** out);

/* DynamicFilterSourceOperator / JoinDomainBuilder (M/operator/DynamicFilterSourceOperator.java, M/operator/JoinDomainBuilder.java):
 * the domain of the build-side join key read off the finished table: min, max and number of distinct non-NULL keys, and the keys
 * themselves (ascending) when there are at most `max_values` of them (distinct_out > max_values: only min/max are meaningful, the
 * reference's fallback to a range).  Single BIGINT-family key only. */
int tgpu_lookup_key_domain(tgpu_ctx* ctx, tgpu_lookup* lookup, int64_t max_values, int64_t* min_out, int64_t* max_out, int64_t* distinct_out,
                           int64_t* values_out, int32_t* has_null_out);

/* DynamicPageFilter (M/sql/gen/columnar/DynamicPageFilter.java:47-211): the probe-side half of dynamic filtering.  One Domain per
 * filtered channel = `null_allowed` + a value set (Domain.includesNullableValue): ALL, NONE, one inclusive range [min, max]
 * (integer family, and DOUBLE by value), or DISCRETE values (integer family; any order, sorted here).  Filters apply in the given order to
 * the surviving rows (DynamicFilterEvaluator.evaluate :160-178); a filter that, after >= 2047 input positions, passes more than
 * selectivity_threshold of them is switched off (EffectiveFilterProfiler :181-210).  A Range with an exclusive upper bound over integers is
 * passed as max = bound - 1.  Zero domains = TupleDomain.all() (every page passes through); TupleDomain.none() = one NONE domain.
 * Output: the input page restricted to the selected rows, in input order (all blocks pass through when every row is selected).
 * tgpu_dynamic_filter_update installs a narrowed predicate (DynamicFilter.getCurrentPredicate after an update: a new evaluator with a
 * fresh profiler, :100-108). */
typedef enum tgpu_domain_kind { TGPU_DOMAIN_ALL = 0, TGPU_DOMAIN_NONE = 1, TGPU_DOMAIN_RANGE = 2, TGPU_DOMAIN_DISCRETE = 3 } tgpu_domain_kind;
typedef struct tgpu_domain {
    int32_t channel;
    int32_t null_allowed;      /* Domain.isNullAllowed() */
    int32_t kind;              /* tgpu_domain_kind */
    int32_t num_values;        /* DISCRETE */
    int64_t min, max;          /* RANGE (raw IEEE bits for a DOUBLE channel); derived for DISCRETE */
    const int64_t* values;     /* DISCRETE */
} tgpu_domain;
int tgpu_dynamic_filter_create(tgpu_ctx* ctx, const tgpu_domain* domains, int32_t num_domains, double selectivity_threshold, tgpu_op** out);
int tgpu_dynamic_filter_update(tgpu_op* op, const tgpu_domain* domains, int32_t num_domains);
int tgpu_dynamic_filter_is_effective(tgpu_op* op, int32_t filter, int32_t* out);

/* LookupSource.getJoinPosition(int[] positions, Page hashChannelsPage, Page allChannelsPage, long[] result)
 * (M/operator/join/JoinHash.java:100-143): for every row of `keys_page` (only the key columns, in
 * key order) the address index of the chain head or -1.  `out_positions` is int32[num_rows], host or
 * device to match the page.  This is the index-only probe the headline metric times.            */
int tgpu_lookup_get_join_positions(tgpu_ctx* ctx, const tgpu_lookup* lookup, const tgpu_page* keys_page, int32_t* out_positions);
/* PositionLinks.next for every build position (ArrayPositionLinks.java:101-104); -1 terminates */
int tgpu_lookup_copy_position_links(tgpu_ctx* ctx, const tgpu_lookup* lookup, int32_t* out_links_host);

/* ------------------------------------------------------------------ partitioned output / exchange
 * Stands in for PartitionedOutputOperator (M/operator/output/PartitionedOutputOperator.java:335-357)
 * + PagePartitioner (M/operator/output/PagePartitioner.java:133-162,229-433) with the
 * SystemPartitionFunction.HASH bucket function (M/sql/planner/HashBucketFunction.java:43-46,
 * M/operator/HashGenerator.java:25-46, M/operator/BucketPartitionFunction.java:45-64).
 * get_output returns one page per non-empty partition per input page; the partition id of the
 * page returned last is read with tgpu_partition_last_output_partition.                          */
enum {
    TGPU_PARTITION_HASH_BUCKET = 0, /* HashBucketFunction over HashGenerator.processRawHash (the inter-stage FIXED_HASH_DISTRIBUTION)   */
    TGPU_PARTITION_LOCAL = 1        /* LocalPartitionGenerator (M/operator/exchange/LocalPartitionGenerator.java:45-77; built by
                                       LocalExchange.java:252 and PartitionedLookupSource.java:103): (int) XxHash64.hash(Long.reverse(raw))
                                       & (bucket_count - 1); bucket_count must be a power of two, bucket_to_partition must be NULL     */
};

typedef struct tgpu_partition_spec {
    int32_t num_key_channels;
    const int32_t* key_channels;          /* partitionChannels; an entry < 0 takes its value from key_constants */
    int32_t bucket_count;                 /* HashBucketFunction bucketCount / LocalPartitionGenerator partitionCount */
    const int32_t* bucket_to_partition;   /* bucket_count entries, NULL = identity */
    int32_t null_channel;                 /* -1 or channel whose NULL rows are replicated to every partition */
    int32_t replicates_any_row;           /* replicatesAnyRow */
    int32_t partition_function;           /* TGPU_PARTITION_* */
    const tgpu_column* key_constants;     /* partitionConstants (PagePartitioner.java:78-101,436-451): NULL, or num_key_channels host columns
                                             of which entry i is read when key_channels[i] < 0 - ONE position holding the constant (its
                                             NullableValue; a NULL constant hashes to 0 like every NULL).  The reference wraps it in a
                                             RunLengthEncodedBlock per page; here its type hash is taken once, at create time.          */
} tgpu_partition_spec;

int tgpu_partition_create(tgpu_ctx* ctx, const tgpu_partition_spec* spec, tgpu_op** out);
int tgpu_partition_last_output_partition(tgpu_op* op, int32_t* out);
/* HashGenerator.getPartitions equivalent: partition id per row (after bucket_to_partition) */
int tgpu_partition_get_partitions(tgpu_op* op, const tgpu_page* page, int32_t* out_partitions);

/* multi-GPU exchange: one process per GPU.  Rank discovery / id distribution is the host's job
 * (torch.distributed here, Trino's task RPC in a Java deployment); the data path is NCCL send/recv
 * over NVLink (all-to-all with explicit counts).  Replaces PartitionedOutputBuffer + HTTP pull
 * (M/execution/buffer/PartitionedOutputBuffer.java, M/operator/DirectExchangeClient.java).       */
#define TGPU_COMM_ID_BYTES 128
int tgpu_comm_get_unique_id(uint8_t id[TGPU_COMM_ID_BYTES]);
int tgpu_comm_init(tgpu_ctx* ctx, const uint8_t id[TGPU_COMM_ID_BYTES], int rank, int world);
int tgpu_comm_destroy(tgpu_ctx* ctx);
/* Peer-memory exchange (NVLink P2P): every rank allocates two receive arenas of `bytes` each and exports their CUDA IPC
 * handles; the host distributes the handles (all-gather) and every rank maps all of them.  With arenas in place
 * tgpu_exchange_partitioned scatters rows STRAIGHT INTO THE DESTINATION GPU'S HBM from the partitioning kernel (no send
 * buffer, no separate transfer) and synchronises with one tiny NCCL all-reduce.  The returned page then aliases an arena
 * and stays valid until the second-next exchange on this context; exchanges that do not fit fall back to NCCL send/recv. */
#define TGPU_IPC_HANDLE_BYTES 64
#define TGPU_NUM_ARENAS 3   /* receive arenas per context; an exchanged page stays valid until the SECOND-next exchange on the context
                               (with three arenas a peer may overwrite page j's arena once this rank entered the barrier of exchange j+2) */
int tgpu_comm_arena_create(tgpu_ctx* ctx, size_t bytes, uint8_t handles_out[TGPU_NUM_ARENAS * TGPU_IPC_HANDLE_BYTES]);
int tgpu_comm_arena_open(tgpu_ctx* ctx, const uint8_t* all_handles /* world x 2 x TGPU_IPC_HANDLE_BYTES, rank-major */);
/* Hash-partition a device-resident page into `world` partitions and exchange: partition p goes to
 * rank p.  Returns the concatenation (in rank order) of what every rank sent here, as a
 * library-owned device page.  Fixed-width pages of a non-replicating partitioner take the multi-split transports (peer-memory
 * stores / copy engines / NCCL); pages with variable-width (TGPU_UTF8) columns, more than 24 columns, and partitioners that
 * replicate rows (null_channel rows and the replicatesAnyRow row reach EVERY rank, PagePartitioner.java:229-241,401-416) take the
 * general path: the partitioner's own per-partition pages travel buffer by buffer through ncclSend/ncclRecv and the received
 * chunks are concatenated in rank order - same rows, same order, library-owned buffers (no arena aliasing).                    */
int tgpu_exchange_partitioned(tgpu_ctx* ctx, tgpu_op* partitioner, const tgpu_page* page, tgpu_page** out);
/* Same, for a pipeline in which another context of this process (`consumer`, e.g. the one running the LookupJoinOperator)
 * reads the exchanged pages: the exchange does not enter its closing barrier - after which peers may overwrite the arena of the
 * exchange before last - until everything enqueued on `consumer` so far has completed.  The wait happens on the device, so this
 * exchange's partition/scatter passes overlap the consumer's kernels.  consumer == NULL: identical to tgpu_exchange_partitioned. */
int tgpu_exchange_partitioned_fenced(tgpu_ctx* ctx, tgpu_op* partitioner, const tgpu_page* page, tgpu_ctx* consumer, tgpu_page** out);

/* Broadcast exchange: the REPLICATED join distribution (FIXED_BROADCAST_DISTRIBUTION, M/sql/planner/SystemPartitioningHandle.java:51;
 * BroadcastOutputBuffer hands every page to every consumer): every rank receives the concatenation, in rank order, of the pages all
 * ranks passed in - the whole (small) build side on every GPU.  Collective: every rank calls it, also with an empty page.  Pages
 * with variable-width columns go through the general exchange's chunk transfer.  With world == 1 it returns a copy of the page. */
int tgpu_exchange_broadcast(tgpu_ctx* ctx, const tgpu_page* page, tgpu_page** out);

/* Split-phase exchange for pipelines (one context): _begin partitions the page (multi-split into per-destination send
 * buffers; rows that stay are written to their final place), then hands the transfer to the copy engines - one peer copy per
 * (destination, column) over NVLink on a side stream, closed by a barrier on a second communicator - and returns while it
 * runs; the SMs are free for the caller's next kernels on this context (e.g. the probe of the previous page).  _end makes the
 * context's stream wait for the transfer and returns the received page (same rows, order and lifetime rules as
 * tgpu_exchange_partitioned).  At most two exchanges may be in flight (begun, not ended) per context, and work that reads a
 * received page must be enqueued on this context before the second-next _begin: with TGPU_NUM_ARENAS = 3 that is what keeps a
 * peer from overwriting an arena that is still being read.  Requires arenas (tgpu_comm_arena_create/open). */
typedef struct tgpu_exchange tgpu_exchange;
int tgpu_exchange_begin(tgpu_ctx* ctx, tgpu_op* partitioner, const tgpu_page* page, tgpu_exchange** out);
int tgpu_exchange_end(tgpu_ctx* ctx, tgpu_exchange* exchange, tgpu_page** out);

/* ------------------------------------------------------------------ Operator protocol
 * One-to-one with M/operator/Operator.java:21-102.                                              */
int tgpu_op_needs_input(tgpu_op* op, int* out);                  /* needsInput() */
int tgpu_op_add_input(tgpu_op* op, const tgpu_page* page);       /* addInput(Page): copies; caller keeps ownership */
int tgpu_op_get_output(tgpu_op* op, tgpu_page** out);            /* getOutput(): *out = NULL when nothing is ready */
int tgpu_op_finish(tgpu_op* op);                                 /* finish(): re-entrant (Driver.java:380-388) */
int tgpu_op_is_finished(tgpu_op* op, int* out);                  /* isFinished() */
int64_t tgpu_op_memory_bytes(tgpu_op* op);                       /* bytes to report through LocalMemoryContext.setBytes */
void tgpu_op_close(tgpu_op* op);                                 /* close() */

/* output pages are library-owned device pages (flags has TGPU_PAGE_DEVICE) until released */
void tgpu_page_release(tgpu_ctx* ctx, tgpu_page* page);
/* copy a device page into caller-provided host buffers: `host` must describe the same schema with
 * buffers large enough (UTF8: data capacity from tgpu_page_utf8_bytes)                          */
int tgpu_page_copy_to_host(tgpu_ctx* ctx, const tgpu_page* device_page, tgpu_page* host);

/* The reference's page wire format, uncompressed and unencrypted (PagesSerdeUtil.writeRawPage / CompressingEncryptingPageSerializer
 * with CompressionCodec.NONE; M/execution/buffer/PagesSerdeUtil.java:44-76, S/block/LongArrayBlockEncoding.java:61-133,
 * S/block/EncoderUtil.java:35-70, S/block/VariableWidthBlockEncoding.java:57-146): lets a GPU stage exchange pages with Java
 * tasks over the existing HTTP exchange.  Block encodings: LONG_ARRAY, INT_ARRAY (also REAL), SHORT_ARRAY, BYTE_ARRAY, VARIABLE_WIDTH,
 * INT128_ARRAY (S/block/Int128ArrayBlockEncoding.java:52-84); dictionary / RLE inputs are written flat.  Parity: tests/test_gpu_serde.py.
 * serialize: `out` is host memory of `capacity` bytes (tgpu_page_serialized_size_bound gives a bound), *bytes_out the length.
 * deserialize: `types[c]` is the tgpu_type of channel c (the wire names the block encoding, not the SQL type). */
int64_t tgpu_page_serialized_size_bound(const tgpu_page* page);
int tgpu_page_serialize(tgpu_ctx* ctx, const tgpu_page* page, uint8_t* out, int64_t capacity, int64_t* bytes_out);
int tgpu_page_deserialize(tgpu_ctx* ctx, const uint8_t* data, int64_t length, const int32_t* types, int32_t num_types, tgpu_page** out);
int64_t tgpu_page_utf8_bytes(tgpu_ctx* ctx, const tgpu_page* device_page, int32_t channel);
/* LookupJoinPageBuilder.build :144-150 returns probe blocks directly when the output covers the probe page 1:1, and
 * InputPageProjection returns its input block: *input_channel = the input channel this output column is an unchanged view
 * of (the host already holds that block and need not copy it back), or -1.  Columns of tgpu_page_copy_to_host whose host
 * `data` pointer is NULL are skipped. */
int tgpu_page_passthrough_channel(const tgpu_page* device_page, int32_t channel, int32_t* input_channel);

/* ------------------------------------------------------------------ synthetic data (bench/tests)
 * Counter-based generators (x_i = splitmix64(seed ^ i)) so the CPU oracle and the GPU produce
 * identical TPC-H-shaped columns without a transfer (SURVEY.md §8d).                            */
int tgpu_synth_orders_keys(tgpu_ctx* ctx, int64_t n_total, int64_t first, int64_t count, uint64_t seed, int shuffle, int64_t* out_device);
int64_t tgpu_synth_lineitem_rows(int64_t n_orders);
int tgpu_synth_lineitem_keys(tgpu_ctx* ctx, int64_t n_orders, int64_t first, int64_t count, uint64_t seed, int shuffle, int64_t* out_device);
int tgpu_synth_lineitem_q1(tgpu_ctx* ctx, int64_t n, int64_t first, uint64_t seed,
                           int32_t* shipdate, int8_t* returnflag, int8_t* linestatus,
                           double* quantity, double* extendedprice, double* discount, double* tax);

/* partitioned 3-way join (BASELINE.json configs[3]): o_custkey of the same orders rows tgpu_synth_orders_keys makes (uniform over the two
 * thirds of the customers that have orders, custkey % 3 != 0); dense key sequences (c_custkey, dimension surrogate keys) */
int tgpu_synth_orders_custkeys(tgpu_ctx* ctx, int64_t n_total, int64_t first, int64_t count, uint64_t seed, int shuffle, int64_t n_customers,
                               uint64_t cust_seed, int64_t* out_device);
int tgpu_synth_sequence(tgpu_ctx* ctx, int64_t first_value, int64_t count, int64_t* out_device);
/* INT32 sequence: the offsets of a VARCHAR(1) column whose bytes are the INT8 code column itself (Q1 with the reference's key types) */
int tgpu_synth_sequence32(tgpu_ctx* ctx, int32_t first_value, int64_t count, int32_t* out_device);
/* star join (BASELINE.json configs[4]): rows [first, first + n) of a TPC-DS store_sales-shaped fact table: ss_sold_date_sk over a
 * 1 823-day window, ss_item_sk 1..300 000, ss_customer_sk 1..12 M and ss_store_sk 1..1 002 with 4.5 % NULLs each (Arrow validity
 * bitmaps, (n + 7) / 8 bytes), ss_net_paid FLOAT64.  *rows_with_both_keys = rows whose two nullable keys are both present. */
int tgpu_synth_store_sales(tgpu_ctx* ctx, int64_t n, int64_t first, uint64_t seed, int64_t* date_sk, int64_t* item_sk, int64_t* customer_sk,
                           uint8_t* customer_valid, int64_t* store_sk, uint8_t* store_valid, double* net_paid, int64_t* rows_with_both_keys);

/* bench / test hygiene: wrapping 64-bit sum of a fixed-width device column (raw bits for FLOAT64; value % mod when mod > 0; NULL rows
 * skipped).  bench.py's N > 1 pass checks the partitioned join with it: sum(build payload) == sum(probe key % 2557), key sum and row
 * count conserved across the exchange.  One small reduction kernel, independent of the aggregation operator it cross-checks. */
int tgpu_column_sum(tgpu_ctx* ctx, const tgpu_column* device_column, int64_t mod, int64_t* out_sum);

#ifdef __cplusplus
}
#endif
#endif /* TRINO_GPU_H */
