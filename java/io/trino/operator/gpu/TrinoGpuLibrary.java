/*
 * Panama (java.lang.foreign) binding of libtrino_gpu.so — the reference-side stub a Trino maintainer would add.
 * NOT compiled in this repository (the build image has no JDK); kept deliberately small and 1:1 with include/trino_gpu.h.
 * JVM flag already present in the reference build: --enable-native-access=ALL-UNNAMED (R/.mvn/jvm.config).
 */
package io.trino.operator.gpu;

import java.lang.foreign.Arena;
import java.lang.foreign.FunctionDescriptor;
import java.lang.foreign.Linker;
import java.lang.foreign.MemorySegment;
import java.lang.foreign.SymbolLookup;
import java.lang.invoke.MethodHandle;

import static java.lang.foreign.ValueLayout.ADDRESS;
import static java.lang.foreign.ValueLayout.JAVA_DOUBLE;
import static java.lang.foreign.ValueLayout.JAVA_INT;
import static java.lang.foreign.ValueLayout.JAVA_LONG;

public final class TrinoGpuLibrary
{
    private static final Linker LINKER = Linker.nativeLinker();
    private static final SymbolLookup LIB = SymbolLookup.libraryLookup(System.getProperty("trino.gpu.library", "libtrino_gpu.so"), Arena.global());

    private static MethodHandle handle(String name, FunctionDescriptor descriptor)
    {
        return LINKER.downcallHandle(LIB.find(name).orElseThrow(() -> new UnsatisfiedLinkError(name)), descriptor);
    }

    // int tgpu_ctx_create(int device, tgpu_ctx** out)
    static final MethodHandle CTX_CREATE = handle("tgpu_ctx_create", FunctionDescriptor.of(JAVA_INT, JAVA_INT, ADDRESS));
    static final MethodHandle CTX_DESTROY = handle("tgpu_ctx_destroy", FunctionDescriptor.ofVoid(ADDRESS));
    static final MethodHandle LAST_ERROR = handle("tgpu_last_error", FunctionDescriptor.of(ADDRESS, ADDRESS));
    static final MethodHandle STATUS_NAME = handle("tgpu_status_name", FunctionDescriptor.of(ADDRESS, JAVA_INT));
    static final MethodHandle HOST_ALLOC_PINNED = handle("tgpu_host_alloc_pinned", FunctionDescriptor.of(JAVA_INT, JAVA_LONG, ADDRESS));
    static final MethodHandle HOST_FREE_PINNED = handle("tgpu_host_free_pinned", FunctionDescriptor.of(JAVA_INT, ADDRESS));
    static final MethodHandle PAGE_UTF8_BYTES = handle("tgpu_page_utf8_bytes", FunctionDescriptor.of(JAVA_LONG, ADDRESS, ADDRESS, JAVA_INT));
    static final MethodHandle LOOKUP_POSITION_COUNT = handle("tgpu_lookup_position_count", FunctionDescriptor.of(JAVA_LONG, ADDRESS));
    static final MethodHandle LOOKUP_MEMORY_BYTES = handle("tgpu_lookup_memory_bytes", FunctionDescriptor.of(JAVA_LONG, ADDRESS));
    // operator factories
    static final MethodHandle FILTER_PROJECT_CREATE = handle("tgpu_filter_project_create", FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS, ADDRESS));
    static final MethodHandle AGG_CREATE = handle("tgpu_agg_create", FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS, ADDRESS));
    static final MethodHandle AGGREGATION_CREATE = handle("tgpu_aggregation_create", FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS, ADDRESS));
    // PartialAggregationController lives in the library so that GPU operators report their flushes without an upcall
    static final MethodHandle PA_CONTROLLER_CREATE = handle("tgpu_partial_agg_controller_create", FunctionDescriptor.of(JAVA_INT, JAVA_LONG, JAVA_DOUBLE, ADDRESS));
    static final MethodHandle PA_CONTROLLER_DESTROY = handle("tgpu_partial_agg_controller_destroy", FunctionDescriptor.ofVoid(ADDRESS));
    static final MethodHandle PA_CONTROLLER_IS_DISABLED = handle("tgpu_partial_agg_controller_is_disabled", FunctionDescriptor.of(JAVA_INT, ADDRESS));
    static final MethodHandle AGG_ROWS_WITH_PA_DISABLED = handle("tgpu_agg_rows_with_partial_aggregation_disabled", FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS));
    static final MethodHandle JOIN_BUILD_CREATE = handle("tgpu_join_build_create", FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS, ADDRESS));
    static final MethodHandle JOIN_BUILD_CREATE_FILTERED = handle("tgpu_join_build_create_filtered", FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS, ADDRESS, JAVA_INT, ADDRESS));
    static final MethodHandle JOIN_BUILD_GET_LOOKUP = handle("tgpu_join_build_get_lookup", FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS));
    static final MethodHandle JOIN_PROBE_CREATE = handle("tgpu_join_probe_create", FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS, ADDRESS, ADDRESS));
    static final MethodHandle LOOKUP_RELEASE = handle("tgpu_lookup_release", FunctionDescriptor.ofVoid(ADDRESS));
    // LookupJoinPageBuilder.build :144-150: probe blocks of a 1:1 page stay on the heap, only the join key is uploaded
    static final MethodHandle JOIN_PROBE_BY_REFERENCE = handle("tgpu_join_probe_set_passthrough_by_reference", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT));
    static final MethodHandle PAGE_PASSTHROUGH_CHANNEL = handle("tgpu_page_passthrough_channel", FunctionDescriptor.of(JAVA_INT, ADDRESS, JAVA_INT, ADDRESS));
    // LookupOuterOperator / HashSemiJoinOperator / DynamicFilterSourceOperator counterparts
    static final MethodHandle JOIN_OUTER_CREATE = handle("tgpu_join_outer_create", FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS, ADDRESS, JAVA_INT, ADDRESS));
    static final MethodHandle SEMI_JOIN_CREATE = handle("tgpu_semi_join_create", FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS, JAVA_INT, ADDRESS));
    static final MethodHandle LOOKUP_KEY_DOMAIN = handle("tgpu_lookup_key_domain",
            FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS, JAVA_LONG, ADDRESS, ADDRESS, ADDRESS, ADDRESS, ADDRESS));
    // exchange between two GPU stages inside one box (replaces PartitionedOutputOperator -> OutputBuffer -> HTTP -> ExchangeOperator)
    static final MethodHandle EXCHANGE_BEGIN = handle("tgpu_exchange_begin", FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS, ADDRESS, ADDRESS));
    static final MethodHandle EXCHANGE_END = handle("tgpu_exchange_end", FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS, ADDRESS));
    static final MethodHandle PARTITION_CREATE = handle("tgpu_partition_create", FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS, ADDRESS));
    static final MethodHandle PARTITION_LAST_OUTPUT = handle("tgpu_partition_last_output_partition", FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS));
    // Operator protocol (M/operator/Operator.java:21-102)
    static final MethodHandle OP_NEEDS_INPUT = handle("tgpu_op_needs_input", FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS));
    static final MethodHandle OP_ADD_INPUT = handle("tgpu_op_add_input", FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS));
    static final MethodHandle OP_GET_OUTPUT = handle("tgpu_op_get_output", FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS));
    static final MethodHandle OP_FINISH = handle("tgpu_op_finish", FunctionDescriptor.of(JAVA_INT, ADDRESS));
    static final MethodHandle OP_IS_FINISHED = handle("tgpu_op_is_finished", FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS));
    static final MethodHandle OP_MEMORY_BYTES = handle("tgpu_op_memory_bytes", FunctionDescriptor.of(JAVA_LONG, ADDRESS));
    static final MethodHandle OP_CLOSE = handle("tgpu_op_close", FunctionDescriptor.ofVoid(ADDRESS));
    static final MethodHandle PAGE_RELEASE = handle("tgpu_page_release", FunctionDescriptor.ofVoid(ADDRESS, ADDRESS));
    static final MethodHandle PAGE_COPY_TO_HOST = handle("tgpu_page_copy_to_host", FunctionDescriptor.of(JAVA_INT, ADDRESS, ADDRESS, ADDRESS));

    private TrinoGpuLibrary() {}

    static String lastError(MemorySegment ctx)
    {
        try {
            return ((MemorySegment) LAST_ERROR.invokeExact(ctx)).reinterpret(1024).getString(0);
        }
        catch (Throwable e) {
            throw new RuntimeException(e);
        }
    }
}
