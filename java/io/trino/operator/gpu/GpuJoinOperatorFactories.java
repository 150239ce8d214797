/*
 * GPU counterparts of the join, filter/project and partitioned-output factories, instantiated at the LocalExecutionPlanner sites named
 * in SURVEY.md §8(b): hash build (M/sql/planner/LocalExecutionPlanner.java:3038-3054), probe (OperatorFactories.join called at :3061-3069),
 * filter/project (:2111-2153), partitioned output (:556-633).  The planner takes these branches only for shapes the library supports
 * (a join filter function only as a translated program, no sort channel; SystemPartitionFunction.HASH; expressions of BIGINT/DOUBLE/BOOLEAN
 * operators) and keeps the
 * Java factories otherwise - TGPU_ERR_NOT_SUPPORTED never reaches a running query.  NOT compiled here (no JDK).
 */
package io.trino.operator.gpu;

import io.trino.operator.DriverContext;
import io.trino.operator.Operator;
import io.trino.operator.OperatorContext;
import io.trino.operator.OperatorFactory;
import io.trino.operator.join.JoinBridgeManager;
import io.trino.operator.join.LookupSource;
import io.trino.operator.join.unspilled.PartitionedLookupSourceFactory;
import io.trino.spi.Page;
import io.trino.sql.planner.plan.PlanNodeId;

import java.lang.foreign.Arena;
import java.lang.foreign.MemorySegment;
import java.util.List;
import java.util.Optional;

import static com.google.common.base.Preconditions.checkState;
import static com.google.common.util.concurrent.MoreExecutors.directExecutor;
import static java.lang.foreign.ValueLayout.ADDRESS;

public final class GpuJoinOperatorFactories
{
    private GpuJoinOperatorFactories() {}

    /** HashBuilderOperatorFactory (M/operator/join/unspilled/HashBuilderOperator.java:55-140): one builder, partition 0 of the bridge */
    public static final class GpuHashBuilderOperatorFactory
            implements OperatorFactory
    {
        private final int operatorId;
        private final PlanNodeId planNodeId;
        private final JoinBridgeManager<PartitionedLookupSourceFactory> bridgeManager;
        private final int[] inputTypes;
        private final List<Integer> hashChannels;
        private final List<Integer> outputChannels;
        private final long expectedPositions;
        // filterFunctionFactory's RowExpression translated by GpuExpressionTranslator to a tgpu_expr_program (filter only) over
        // createJoinSourcesLayout(buildLayout, probeLayout), kept alive by the factory, and buildLayout.size(); empty = no join filter function
        private final Optional<MemorySegment> filter;
        private final int buildLayoutSize;
        private boolean closed;

        public GpuHashBuilderOperatorFactory(int operatorId, PlanNodeId planNodeId, JoinBridgeManager<PartitionedLookupSourceFactory> bridgeManager, int[] inputTypes,
                List<Integer> hashChannels, List<Integer> outputChannels, long expectedPositions)
        {
            this(operatorId, planNodeId, bridgeManager, inputTypes, hashChannels, outputChannels, expectedPositions, Optional.empty(), inputTypes.length);
        }

        public GpuHashBuilderOperatorFactory(int operatorId, PlanNodeId planNodeId, JoinBridgeManager<PartitionedLookupSourceFactory> bridgeManager, int[] inputTypes,
                List<Integer> hashChannels, List<Integer> outputChannels, long expectedPositions, Optional<MemorySegment> filter, int buildLayoutSize)
        {
            this.operatorId = operatorId;
            this.planNodeId = planNodeId;
            this.bridgeManager = bridgeManager;
            this.inputTypes = inputTypes.clone();
            this.hashChannels = List.copyOf(hashChannels);
            this.outputChannels = List.copyOf(outputChannels);
            this.expectedPositions = expectedPositions;
            this.filter = filter;
            this.buildLayoutSize = buildLayoutSize;
        }

        @Override
        public Operator createOperator(DriverContext driverContext)
        {
            checkState(!closed, "Factory is already closed");
            OperatorContext operatorContext = driverContext.addOperatorContext(operatorId, planNodeId, "GpuHashBuilderOperator");
            GpuContexts.Handle gpu = GpuContexts.forCurrentDriver(driverContext);
            MemorySegment op = filter.isPresent()
                    ? NativeSpecs.createJoinBuildFiltered(gpu, hashChannels, outputChannels, expectedPositions, filter.get(), buildLayoutSize)
                    : NativeSpecs.createJoinBuild(gpu, hashChannels, outputChannels, expectedPositions);
            PartitionedLookupSourceFactory bridge = bridgeManager.getJoinBridge();
            return new GpuOperator(operatorContext, gpu.context(), op, gpu.marshaller(inputTypes), new int[0])
            {
                private boolean lent;

                @Override
                public void finish()
                {
                    super.finish();      // flushes the last batch, builds the table on the device
                    if (lent) {
                        return;
                    }
                    lent = true;
                    try (Arena arena = Arena.ofConfined()) {
                        MemorySegment out = arena.allocate(ADDRESS);
                        check((int) TrinoGpuLibrary.JOIN_BUILD_GET_LOOKUP.invokeExact(this.op, out));
                        GpuLookupSource source = new GpuLookupSource(out.get(ADDRESS, 0));
                        // HashBuilderOperator.finishInput :310-333: hand the lookup source to the bridge; probes obtain it from createLookupSource()
                        bridge.lendPartitionLookupSource(0, () -> source).addListener(source::close, directExecutor());
                    }
                    catch (Throwable e) {
                        throw new RuntimeException(e);
                    }
                }

                @Override
                public Page getOutput()
                {
                    return null;
                }
            };
        }

        @Override
        public void noMoreOperators()
        {
            closed = true;
        }

        @Override
        public OperatorFactory duplicate()
        {
            throw new UnsupportedOperationException("Parallel hash build cannot be duplicated");     // as the reference (:131-135)
        }
    }

    /** LookupJoinOperatorFactory: probe pages against the table the bridge delivers; 1:1 outputs return the probe blocks themselves */
    public static final class GpuLookupJoinOperatorFactory
            implements OperatorFactory
    {
        private final int operatorId;
        private final PlanNodeId planNodeId;
        private final JoinBridgeManager<PartitionedLookupSourceFactory> bridgeManager;
        private final int[] probeTypes;
        private final int[] outputTypes;
        private final int joinType;
        private final boolean outputSingleMatch;
        private final List<Integer> probeJoinChannels;
        private final List<Integer> probeOutputChannels;
        private boolean closed;

        public GpuLookupJoinOperatorFactory(int operatorId, PlanNodeId planNodeId, JoinBridgeManager<PartitionedLookupSourceFactory> bridgeManager, int[] probeTypes,
                int[] outputTypes, int joinType, boolean outputSingleMatch, List<Integer> probeJoinChannels, List<Integer> probeOutputChannels)
        {
            this.operatorId = operatorId;
            this.planNodeId = planNodeId;
            this.bridgeManager = bridgeManager;
            this.probeTypes = probeTypes.clone();
            this.outputTypes = outputTypes.clone();
            this.joinType = joinType;
            this.outputSingleMatch = outputSingleMatch;
            this.probeJoinChannels = List.copyOf(probeJoinChannels);
            this.probeOutputChannels = List.copyOf(probeOutputChannels);
            bridgeManager.incrementProbeFactoryCount();
        }

        @Override
        public Operator createOperator(DriverContext driverContext)
        {
            checkState(!closed, "Factory is already closed");
            OperatorContext operatorContext = driverContext.addOperatorContext(operatorId, planNodeId, "GpuLookupJoinOperator");
            GpuContexts.Handle gpu = GpuContexts.forCurrentDriver(driverContext);
            PartitionedLookupSourceFactory bridge = bridgeManager.getJoinBridge();
            bridgeManager.probeOperatorCreated();
            LookupSource lookupSource;
            try {
                // the Driver only schedules the probe once the build pipeline has finished (the bridge's future is the blocking point of
                // the Java LookupJoinOperator: WorkProcessor blocked on lookupSourceProvider); here it is complete by construction
                lookupSource = bridge.createLookupSource().get();
            }
            catch (Exception e) {
                throw new RuntimeException(e);
            }
            MemorySegment lookup = ((GpuLookupSource) lookupSource).handle();
            MemorySegment op = NativeSpecs.createJoinProbe(gpu, lookup, joinType, outputSingleMatch, probeJoinChannels, probeOutputChannels);
            try {
                // host pages: upload the join key only, pass-through probe blocks stay on the heap (LookupJoinPageBuilder.build :144-150)
                int status = (int) TrinoGpuLibrary.JOIN_PROBE_BY_REFERENCE.invokeExact(op, 1);
                if (status != 0) {
                    throw GpuOperator.failure(status, gpu.context());
                }
            }
            catch (RuntimeException e) {
                throw e;
            }
            catch (Throwable e) {
                throw new RuntimeException(e);
            }
            return new GpuOperator(operatorContext, gpu.context(), op, gpu.marshaller(probeTypes), outputTypes)
            {
                @Override
                public void close()
                {
                    super.close();
                    lookupSource.close();
                    bridgeManager.probeOperatorClosed();
                }
            };
        }

        @Override
        public void noMoreOperators()
        {
            closed = true;
            bridgeManager.probeOperatorFactoryClosed();
        }

        @Override
        public OperatorFactory duplicate()
        {
            return new GpuLookupJoinOperatorFactory(operatorId, planNodeId, bridgeManager, probeTypes, outputTypes, joinType, outputSingleMatch, probeJoinChannels,
                    probeOutputChannels);
        }
    }

    /**
     * FilterAndProjectOperator (M/operator/FilterAndProjectOperator.java:60-95).  `program` is a tgpu_expr_program built by
     * GpuExpressionTranslator from translatedFilter / translatedProjections (LocalExecutionPlanner.java:2111-2114), kept alive by the factory.
     */
    public static final class GpuFilterAndProjectOperatorFactory
            implements OperatorFactory
    {
        private final int operatorId;
        private final PlanNodeId planNodeId;
        private final MemorySegment program;
        private final int[] inputTypes;
        private final int[] outputTypes;
        private boolean closed;

        public GpuFilterAndProjectOperatorFactory(int operatorId, PlanNodeId planNodeId, MemorySegment program, int[] inputTypes, int[] outputTypes)
        {
            this.operatorId = operatorId;
            this.planNodeId = planNodeId;
            this.program = program;
            this.inputTypes = inputTypes.clone();
            this.outputTypes = outputTypes.clone();
        }

        @Override
        public Operator createOperator(DriverContext driverContext)
        {
            checkState(!closed, "Factory is already closed");
            OperatorContext operatorContext = driverContext.addOperatorContext(operatorId, planNodeId, "GpuFilterAndProjectOperator");
            GpuContexts.Handle gpu = GpuContexts.forCurrentDriver(driverContext);
            try (Arena arena = Arena.ofConfined()) {
                MemorySegment out = arena.allocate(ADDRESS);
                int status = (int) TrinoGpuLibrary.FILTER_PROJECT_CREATE.invokeExact(gpu.context(), program, out);
                if (status != 0) {
                    throw GpuOperator.failure(status, gpu.context());
                }
                return new GpuOperator(operatorContext, gpu.context(), out.get(ADDRESS, 0), gpu.marshaller(inputTypes), outputTypes);
            }
            catch (RuntimeException e) {
                throw e;
            }
            catch (Throwable e) {
                throw new RuntimeException(e);
            }
        }

        @Override
        public void noMoreOperators()
        {
            closed = true;
        }

        @Override
        public OperatorFactory duplicate()
        {
            return new GpuFilterAndProjectOperatorFactory(operatorId, planNodeId, program, inputTypes, outputTypes);
        }
    }

    /**
     * PartitionedOutputOperator (M/operator/output/PartitionedOutputOperator.java:335-357) for SystemPartitionFunction.HASH: the device
     * partitions the page; every output page is enqueued into the OutputBuffer under tgpu_partition_last_output_partition.  Between two
     * GPU stages of one box the exchange itself stays on the device (tgpu_exchange_begin/_end, INTEGRATION.md §5) and this operator
     * is not on the path.
     */
    public static final class GpuPartitionedOutputOperatorFactory
            implements OperatorFactory
    {
        private final int operatorId;
        private final PlanNodeId planNodeId;
        private final int[] types;
        private final List<Integer> partitionChannels;
        private final int bucketCount;
        private final int[] bucketToPartition;
        private final int nullChannel;
        private final boolean replicatesAnyRow;
        private final Page partitionConstants;           // null, or ONE position: block i = NullableValue.asBlock() of partition channel i (any block where it is a real channel)
        private final int[] partitionConstantTypes;
        private final java.util.function.BiConsumer<Integer, Page> enqueue;      // OutputBuffer.enqueue(partition, serialized pages) of the task

        public GpuPartitionedOutputOperatorFactory(int operatorId, PlanNodeId planNodeId, int[] types, List<Integer> partitionChannels, int bucketCount,
                int[] bucketToPartition, int nullChannel, boolean replicatesAnyRow, Page partitionConstants, int[] partitionConstantTypes,
                java.util.function.BiConsumer<Integer, Page> enqueue)
        {
            this.partitionConstants = partitionConstants;
            this.partitionConstantTypes = partitionConstantTypes;
            this.operatorId = operatorId;
            this.planNodeId = planNodeId;
            this.types = types.clone();
            this.partitionChannels = List.copyOf(partitionChannels);
            this.bucketCount = bucketCount;
            this.bucketToPartition = bucketToPartition;
            this.nullChannel = nullChannel;
            this.replicatesAnyRow = replicatesAnyRow;
            this.enqueue = enqueue;
        }

        @Override
        public Operator createOperator(DriverContext driverContext)
        {
            OperatorContext operatorContext = driverContext.addOperatorContext(operatorId, planNodeId, "GpuPartitionedOutputOperator");
            GpuContexts.Handle gpu = GpuContexts.forCurrentDriver(driverContext);
            MemorySegment op;
            try (Arena arena = Arena.ofConfined()) {
                MemorySegment constants = MemorySegment.NULL;
                if (partitionConstants != null) {
                    io.trino.spi.block.PageMarshaller constantMarshaller = gpu.marshaller(partitionConstantTypes);
                    constantMarshaller.append(partitionConstants);
                    constants = constantMarshaller.flush(arena).get(java.lang.foreign.ValueLayout.ADDRESS, 16);      // tgpu_page.columns
                }
                op = NativeSpecs.createPartitioner(gpu, partitionChannels, bucketCount, bucketToPartition, nullChannel, replicatesAnyRow,
                        NativeSpecs.PARTITION_HASH_BUCKET, constants);
            }
            return new GpuOperator(operatorContext, gpu.context(), op, gpu.marshaller(types), types)
            {
                @Override
                protected int tagOf(MemorySegment devicePage)
                        throws Throwable
                {
                    try (Arena arena = Arena.ofConfined()) {
                        MemorySegment out = arena.allocate(java.lang.foreign.ValueLayout.JAVA_INT);
                        check((int) TrinoGpuLibrary.PARTITION_LAST_OUTPUT.invokeExact(this.op, out));   // partition of the page get_output just returned
                        return out.get(java.lang.foreign.ValueLayout.JAVA_INT, 0);
                    }
                }

                @Override
                public Page getOutput()
                {
                    // a sink: every partition page goes into the output buffer, nothing flows downstream (PartitionedOutputOperator.getOutput :352-356)
                    Page page;
                    while ((page = super.getOutput()) != null) {
                        enqueue.accept(lastOutputTag, page);
                    }
                    return null;
                }
            };
        }

        @Override
        public void noMoreOperators() {}

        @Override
        public OperatorFactory duplicate()
        {
            return new GpuPartitionedOutputOperatorFactory(operatorId, planNodeId, types, partitionChannels, bucketCount, bucketToPartition, nullChannel, replicatesAnyRow, partitionConstants, partitionConstantTypes, enqueue);
        }
    }
}
