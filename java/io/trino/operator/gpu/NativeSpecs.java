/*
 * Builders of the native spec structs of include/trino_gpu.h (tgpu_agg_spec, tgpu_join_build_spec, tgpu_join_probe_spec,
 * tgpu_partition_spec, tgpu_expr_program) from the plain values LocalExecutionPlanner holds at the construction sites
 * (M/sql/planner/LocalExecutionPlanner.java:4040-4118 aggregation, :2930-3069 join, :556-633 partitioned output, :2111-2153 filter/project).
 * Field order, widths and padding follow the C declarations; every create call returns a tgpu_op*.  NOT compiled here (no JDK).
 */
package io.trino.operator.gpu;

import io.trino.operator.gpu.GpuHashAggregationOperatorFactory.GpuAggregate;
import io.trino.sql.planner.plan.AggregationNode.Step;

import java.lang.foreign.Arena;
import java.lang.foreign.MemoryLayout;
import java.lang.foreign.MemorySegment;
import java.lang.foreign.StructLayout;
import java.util.List;

import static java.lang.foreign.ValueLayout.ADDRESS;
import static java.lang.foreign.ValueLayout.JAVA_BYTE;
import static java.lang.foreign.ValueLayout.JAVA_INT;
import static java.lang.foreign.ValueLayout.JAVA_LONG;

public final class NativeSpecs
{
    private NativeSpecs() {}

    // tgpu_agg_fn { int32 function; int32 input_channel; int32 mask_channel; int32 reserved }
    static final StructLayout AGG_FN = MemoryLayout.structLayout(JAVA_INT, JAVA_INT, JAVA_INT, JAVA_INT);
    // tgpu_agg_spec { int32 num_keys; (pad) ; int32* key_channels; int32 step; int32 num_aggs; tgpu_agg_fn* aggs; int64 expected_groups;
    //                 int64 max_partial_bytes; tgpu_expr_program* pre; int32 num_global_group_ids; (pad); int32* global_group_ids;
    //                 int32 group_id_key; int32 num_input_channels; int32* input_channel_types; tgpu_partial_agg_controller* controller }
    static final StructLayout AGG_SPEC = MemoryLayout.structLayout(
            JAVA_INT.withName("num_keys"), MemoryLayout.paddingLayout(4), ADDRESS.withName("key_channels"),
            JAVA_INT.withName("step"), JAVA_INT.withName("num_aggs"), ADDRESS.withName("aggs"),
            JAVA_LONG.withName("expected_groups"), JAVA_LONG.withName("max_partial_bytes"), ADDRESS.withName("pre"),
            JAVA_INT.withName("num_global_group_ids"), MemoryLayout.paddingLayout(4), ADDRESS.withName("global_group_ids"),
            JAVA_INT.withName("group_id_key"), JAVA_INT.withName("num_input_channels"), ADDRESS.withName("input_channel_types"),
            ADDRESS.withName("partial_aggregation_controller"));
    // tgpu_join_build_spec { int32 num_key_channels; int32* key_channels; int32 num_output_channels; int32* output_channels; int64 expected_positions }
    static final StructLayout JOIN_BUILD_SPEC = MemoryLayout.structLayout(
            JAVA_INT, MemoryLayout.paddingLayout(4), ADDRESS, JAVA_INT, MemoryLayout.paddingLayout(4), ADDRESS, JAVA_LONG);
    // tgpu_join_probe_spec { int32 join_type; int32 output_single_match; int32 num_key_channels; int32* key_channels; int32 num_output_channels; int32* output_channels }
    static final StructLayout JOIN_PROBE_SPEC = MemoryLayout.structLayout(
            JAVA_INT, JAVA_INT, JAVA_INT, MemoryLayout.paddingLayout(4), ADDRESS, JAVA_INT, MemoryLayout.paddingLayout(4), ADDRESS);
    // tgpu_partition_spec { int32 num_key_channels; int32* key_channels; int32 bucket_count; int32* bucket_to_partition; int32 null_channel; int32 replicates_any_row;
    //                       int32 partition_function; tgpu_column* key_constants }
    static final StructLayout PARTITION_SPEC = MemoryLayout.structLayout(
            JAVA_INT, MemoryLayout.paddingLayout(4), ADDRESS, JAVA_INT, MemoryLayout.paddingLayout(4), ADDRESS, JAVA_INT, JAVA_INT,
            JAVA_INT, MemoryLayout.paddingLayout(4), ADDRESS);
    // tgpu_bytes { int32 length; (pad); uint8* data }
    static final StructLayout BYTES = MemoryLayout.structLayout(JAVA_INT.withName("length"), MemoryLayout.paddingLayout(4), ADDRESS.withName("data"));
    // tgpu_like_pattern { tgpu_bytes pattern; tgpu_bytes escape /* length 0 = no ESCAPE */ }: a `$like` whose `$like_pattern` argument is a constant
    static final StructLayout LIKE_PATTERN = MemoryLayout.structLayout(BYTES.withName("pattern"), BYTES.withName("escape"));
    // tgpu_expr_program { int32 num_insns; (pad); tgpu_expr_insn* insns; int32 filter_temp; int32 num_filter_insns; int32 num_projections; (pad);
    //                     tgpu_projection* projections; int32 num_in_lists; (pad); tgpu_in_list* in_lists; int32 num_strings; (pad); tgpu_bytes* strings;
    //                     int32 num_like_patterns; (pad); tgpu_like_pattern* like_patterns; tgpu_decimal_signature* decimal_signatures;
    //                     int32 num_decimal_constants; (pad); int64* decimal_constants }  (112 bytes; a zeroed tail = no strings, no decimals)
    static final StructLayout EXPR_PROGRAM = MemoryLayout.structLayout(
            JAVA_INT.withName("num_insns"), MemoryLayout.paddingLayout(4), ADDRESS.withName("insns"),
            JAVA_INT.withName("filter_temp"), JAVA_INT.withName("num_filter_insns"), JAVA_INT.withName("num_projections"), MemoryLayout.paddingLayout(4),
            ADDRESS.withName("projections"), JAVA_INT.withName("num_in_lists"), MemoryLayout.paddingLayout(4), ADDRESS.withName("in_lists"),
            JAVA_INT.withName("num_strings"), MemoryLayout.paddingLayout(4), ADDRESS.withName("strings"),
            JAVA_INT.withName("num_like_patterns"), MemoryLayout.paddingLayout(4), ADDRESS.withName("like_patterns"),
            ADDRESS.withName("decimal_signatures"), JAVA_INT.withName("num_decimal_constants"), MemoryLayout.paddingLayout(4),
            ADDRESS.withName("decimal_constants"));
    // DECIMAL operands: TGPU_V_DECIMAL = 4; casts TGPU_EX_CAST_TO_DECIMAL = 32, _DECIMAL_TO_BIGINT = 33, _DECIMAL_TO_DOUBLE = 34.
    // tgpu_decimal_type { int8 precision, scale }; tgpu_decimal_signature { a, b, c, result } (8 bytes): the bound types of the resolved
    // function ($operator$add(decimal(p1,s1), decimal(p2,s2)):decimal(p,s) and the like), one per instruction
    public static final int V_DECIMAL = 4;
    public static final int EX_CAST_TO_DECIMAL = 32;
    public static final int EX_CAST_DECIMAL_TO_BIGINT = 33;
    public static final int EX_CAST_DECIMAL_TO_DOUBLE = 34;
    static final StructLayout DECIMAL_TYPE = MemoryLayout.structLayout(JAVA_BYTE.withName("precision"), JAVA_BYTE.withName("scale"));
    static final StructLayout DECIMAL_SIGNATURE = MemoryLayout.structLayout(DECIMAL_TYPE.withName("a"), DECIMAL_TYPE.withName("b"),
            DECIMAL_TYPE.withName("c"), DECIMAL_TYPE.withName("result"));
    // String functions (operand type TGPU_V_VARCHAR = 3): the resolved function of a call maps to one opcode.  length(varchar) -> EX_LENGTH;
    // substr / substring(varchar, bigint[, bigint]) -> EX_SUBSTR (the two-argument form leaves operand c TGPU_OPND_NONE); ltrim / rtrim /
    // trim(varchar) with one argument -> EX_LTRIM / EX_RTRIM / EX_TRIM; concat(varchar, ...) and `||` -> a left-deep chain of binary
    // EX_CONCATs, at most 8 pieces.  A computed projection of vtype 3 yields a UTF8 column.  CHAR(n) arguments and the trims with a
    // character list keep the Java operator.
    public static final int V_VARCHAR = 3;
    public static final int EX_LENGTH = 50;
    public static final int EX_SUBSTR = 51;
    public static final int EX_LTRIM = 52;
    public static final int EX_RTRIM = 53;
    public static final int EX_TRIM = 54;
    public static final int EX_CONCAT = 55;
    public static final int MAX_CONCAT_PIECES = 8;
    // Conditional special forms (SpecialForm IF, SWITCH / WHEN, COALESCE, NULL_IF of SqlToRowExpressionTranslator) lower onto two opcodes
    // whose vtype is the result type (BIGINT, DOUBLE, BOOLEAN or DECIMAL; a VARCHAR result keeps the Java operator): EX_IF(a, b, c) is
    // a ? b : c with a BOOLEAN condition (c TGPU_OPND_NULL for a CASE without ELSE), EX_COALESCE(a, b) the first non-NULL operand.
    //   IF(c, r, e) and a searched CASE: the right-deep chain IF(c1, r1, IF(c2, r2, ... e)).
    //   SWITCH(v, WHEN(w1, r1), ..., e): v into a temp t, then IF(EQ(t, w1), r1, IF(EQ(t, w2), r2, ... e)), t the FIRST operand of each
    //   EQ, so that v's error comes first and a NULL v reaches e without any w's error.
    //   COALESCE(a1, ..., an): COALESCE(a1, COALESCE(a2, ... an)).
    //   NULL_IF(a, b): a into a temp t, then IF(EQ(cast(t), cast(b)), NULL, t) with the casts of the resolved EQUAL's argument type.
    // For DECIMAL the signature's selected operands and result are the one (coerced) result type.  Join filters keep the Java operator.
    public static final int EX_IF = 60;
    public static final int EX_COALESCE = 61;

    /** the opcode of a one-call string function (by its resolved name and argument count), or -1 when it keeps the Java operator */
    public static int stringFunctionOpcode(String name, int arity)
    {
        return switch (name) {
            case "length" -> arity == 1 ? EX_LENGTH : -1;
            case "substr", "substring" -> arity == 2 || arity == 3 ? EX_SUBSTR : -1;
            case "ltrim" -> arity == 1 ? EX_LTRIM : -1;
            case "rtrim" -> arity == 1 ? EX_RTRIM : -1;
            case "trim" -> arity == 1 ? EX_TRIM : -1;
            case "concat", "$operator$concat" -> arity >= 2 && arity <= MAX_CONCAT_PIECES ? EX_CONCAT : -1;
            default -> -1;
        };
    }

    public static final int PARTITION_HASH_BUCKET = 0;    // HashBucketFunction (M/sql/planner/HashBucketFunction.java:43-46)
    public static final int PARTITION_LOCAL = 1;          // LocalPartitionGenerator (M/operator/exchange/LocalPartitionGenerator.java:45-77)

    static MemorySegment ints(Arena arena, List<Integer> values)
    {
        MemorySegment segment = arena.allocate(JAVA_INT, Math.max(1, values.size()));
        for (int i = 0; i < values.size(); i++) {
            segment.setAtIndex(JAVA_INT, i, values.get(i));
        }
        return segment;
    }

    private static MemorySegment create(GpuContexts.Handle gpu, java.lang.invoke.MethodHandle factory, MemorySegment spec, Arena arena)
            throws Throwable
    {
        MemorySegment out = arena.allocate(ADDRESS);
        int status = (int) factory.invokeExact(gpu.context(), spec, out);
        if (status != 0) {
            throw GpuOperator.failure(status, gpu.context());
        }
        return out.get(ADDRESS, 0);
    }

    /** Step -> tgpu_agg_step (M/sql/planner/plan/AggregationNode.java:361-402) */
    static int stepCode(Step step)
    {
        return switch (step) {
            case SINGLE -> 0;
            case PARTIAL -> 1;
            case FINAL -> 2;
            case INTERMEDIATE -> 3;
        };
    }

    public static MemorySegment createAggregation(GpuContexts.Handle gpu, List<Integer> groupByChannels, Step step, List<GpuAggregate> aggregates, int expectedGroups,
            long maxPartialMemory, List<Integer> globalAggregationGroupIds, int groupIdKey, int[] inputChannelTypes, MemorySegment preProgram,
            MemorySegment partialAggregationController)
    {
        try (Arena arena = Arena.ofConfined()) {
            MemorySegment spec = aggregationSpec(arena, step, aggregates, inputChannelTypes, preProgram);
            spec.set(JAVA_INT, 0, groupByChannels.size());
            spec.set(ADDRESS, 8, ints(arena, groupByChannels));
            spec.set(JAVA_LONG, 32, expectedGroups);
            spec.set(JAVA_LONG, 40, maxPartialMemory);
            spec.set(JAVA_INT, 56, globalAggregationGroupIds.size());
            spec.set(ADDRESS, 64, ints(arena, globalAggregationGroupIds));
            spec.set(JAVA_INT, 72, groupIdKey);
            spec.set(ADDRESS, 88, partialAggregationController);       // MemorySegment.NULL = Optional.empty()
            return create(gpu, TrinoGpuLibrary.AGG_CREATE, spec, arena);
        }
        catch (RuntimeException e) {
            throw e;
        }
        catch (Throwable e) {
            throw new RuntimeException(e);
        }
    }

    /** AggregationOperator (tgpu_aggregation_create): no keys, no flush threshold, no grouping sets, no controller */
    public static MemorySegment createGlobalAggregation(GpuContexts.Handle gpu, Step step, List<GpuAggregate> aggregates, int[] inputChannelTypes, MemorySegment preProgram)
    {
        try (Arena arena = Arena.ofConfined()) {
            MemorySegment spec = aggregationSpec(arena, step, aggregates, inputChannelTypes, preProgram);
            spec.set(JAVA_INT, 72, -1);                                 // group_id_key
            return create(gpu, TrinoGpuLibrary.AGGREGATION_CREATE, spec, arena);
        }
        catch (RuntimeException e) {
            throw e;
        }
        catch (Throwable e) {
            throw new RuntimeException(e);
        }
    }

    // tgpu_agg_spec with the fields both aggregation operators read; the others zero / NULL
    private static MemorySegment aggregationSpec(Arena arena, Step step, List<GpuAggregate> aggregates, int[] inputChannelTypes, MemorySegment preProgram)
    {
        MemorySegment fns = arena.allocate(AGG_FN, Math.max(1, aggregates.size()));
        for (int i = 0; i < aggregates.size(); i++) {
            GpuAggregate aggregate = aggregates.get(i);
            long at = i * AGG_FN.byteSize();
            fns.set(JAVA_INT, at, aggregate.function());
            fns.set(JAVA_INT, at + 4, aggregate.inputChannel());
            fns.set(JAVA_INT, at + 8, aggregate.maskChannel());
            fns.set(JAVA_INT, at + 12, aggregate.resultType());      // avg(decimal) in a FINAL step: TGPU_INT64 / TGPU_INT128, else 0
        }
        MemorySegment types = arena.allocate(JAVA_INT, Math.max(1, inputChannelTypes.length));
        for (int i = 0; i < inputChannelTypes.length; i++) {
            types.setAtIndex(JAVA_INT, i, inputChannelTypes[i]);
        }
        MemorySegment spec = arena.allocate(AGG_SPEC);                 // zero-filled: no keys, NULL pointers
        spec.set(JAVA_INT, 16, stepCode(step));
        spec.set(JAVA_INT, 20, aggregates.size());
        spec.set(ADDRESS, 24, fns);
        spec.set(ADDRESS, 48, preProgram);
        spec.set(JAVA_INT, 76, inputChannelTypes.length);
        spec.set(ADDRESS, 80, types);
        return spec;
    }

    public static MemorySegment createJoinBuild(GpuContexts.Handle gpu, List<Integer> hashChannels, List<Integer> outputChannels, long expectedPositions)
    {
        try (Arena arena = Arena.ofConfined()) {
            MemorySegment spec = arena.allocate(JOIN_BUILD_SPEC);
            spec.set(JAVA_INT, 0, hashChannels.size());
            spec.set(ADDRESS, 8, ints(arena, hashChannels));
            spec.set(JAVA_INT, 16, outputChannels.size());
            spec.set(ADDRESS, 24, ints(arena, outputChannels));
            spec.set(JAVA_LONG, 32, expectedPositions);
            return create(gpu, TrinoGpuLibrary.JOIN_BUILD_CREATE, spec, arena);
        }
        catch (RuntimeException e) {
            throw e;
        }
        catch (Throwable e) {
            throw new RuntimeException(e);
        }
    }

    /** HashBuilderOperatorFactory with a filterFunctionFactory: `filter` is a tgpu_expr_program over the join-sources layout, buildLayoutSize its build channels */
    public static MemorySegment createJoinBuildFiltered(GpuContexts.Handle gpu, List<Integer> hashChannels, List<Integer> outputChannels, long expectedPositions,
            MemorySegment filter, int buildLayoutSize)
    {
        try (Arena arena = Arena.ofConfined()) {
            MemorySegment spec = arena.allocate(JOIN_BUILD_SPEC);
            spec.set(JAVA_INT, 0, hashChannels.size());
            spec.set(ADDRESS, 8, ints(arena, hashChannels));
            spec.set(JAVA_INT, 16, outputChannels.size());
            spec.set(ADDRESS, 24, ints(arena, outputChannels));
            spec.set(JAVA_LONG, 32, expectedPositions);
            MemorySegment out = arena.allocate(ADDRESS);
            int status = (int) TrinoGpuLibrary.JOIN_BUILD_CREATE_FILTERED.invokeExact(gpu.context(), spec, filter, buildLayoutSize, out);
            if (status != 0) {
                throw GpuOperator.failure(status, gpu.context());
            }
            return out.get(ADDRESS, 0);
        }
        catch (RuntimeException e) {
            throw e;
        }
        catch (Throwable e) {
            throw new RuntimeException(e);
        }
    }

    /** joinType: 0 INNER, 1 PROBE_OUTER, 2 LOOKUP_OUTER, 3 FULL_OUTER (LookupJoinOperatorFactory.JoinType) */
    public static MemorySegment createJoinProbe(GpuContexts.Handle gpu, MemorySegment lookup, int joinType, boolean outputSingleMatch, List<Integer> probeJoinChannels,
            List<Integer> probeOutputChannels)
    {
        try (Arena arena = Arena.ofConfined()) {
            MemorySegment spec = arena.allocate(JOIN_PROBE_SPEC);
            spec.set(JAVA_INT, 0, joinType);
            spec.set(JAVA_INT, 4, outputSingleMatch ? 1 : 0);
            spec.set(JAVA_INT, 8, probeJoinChannels.size());
            spec.set(ADDRESS, 16, ints(arena, probeJoinChannels));
            spec.set(JAVA_INT, 24, probeOutputChannels.size());
            spec.set(ADDRESS, 32, ints(arena, probeOutputChannels));
            MemorySegment out = arena.allocate(ADDRESS);
            int status = (int) TrinoGpuLibrary.JOIN_PROBE_CREATE.invokeExact(gpu.context(), spec, lookup, out);
            if (status != 0) {
                throw GpuOperator.failure(status, gpu.context());
            }
            return out.get(ADDRESS, 0);
        }
        catch (RuntimeException e) {
            throw e;
        }
        catch (Throwable e) {
            throw new RuntimeException(e);
        }
    }

    /**
     * keyConstants: MemorySegment.NULL, or the tgpu_column array of a ONE-position page that holds, at index i, the partition constant of
     * partition channel i when partitionChannels.get(i) is negative (PagePartitioner.java:78-101: NullableValue.asBlock()); the library reads
     * it inside this call only.
     */
    public static MemorySegment createPartitioner(GpuContexts.Handle gpu, List<Integer> partitionChannels, int bucketCount, int[] bucketToPartition, int nullChannel,
            boolean replicatesAnyRow, int partitionFunction, MemorySegment keyConstants)
    {
        try (Arena arena = Arena.ofConfined()) {
            MemorySegment spec = arena.allocate(PARTITION_SPEC);
            spec.set(JAVA_INT, 0, partitionChannels.size());
            spec.set(ADDRESS, 8, ints(arena, partitionChannels));
            spec.set(JAVA_INT, 16, bucketCount);
            MemorySegment b2p = MemorySegment.NULL;
            if (bucketToPartition != null) {
                b2p = arena.allocate(JAVA_INT, bucketToPartition.length);
                for (int i = 0; i < bucketToPartition.length; i++) {
                    b2p.setAtIndex(JAVA_INT, i, bucketToPartition[i]);
                }
            }
            spec.set(ADDRESS, 24, b2p);
            spec.set(JAVA_INT, 32, nullChannel);
            spec.set(JAVA_INT, 36, replicatesAnyRow ? 1 : 0);
            spec.set(JAVA_INT, 40, partitionFunction);
            spec.set(ADDRESS, 48, keyConstants);
            return create(gpu, TrinoGpuLibrary.PARTITION_CREATE, spec, arena);
        }
        catch (RuntimeException e) {
            throw e;
        }
        catch (Throwable e) {
            throw new RuntimeException(e);
        }
    }
}
