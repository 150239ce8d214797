/*
 * Drop-in for AggregationOperator.AggregationOperatorFactory (M/operator/AggregationOperator.java:43-88): aggregation without GROUP BY
 * keys, instantiated where LocalExecutionPlanner.planGlobalAggregation (:3978-4011) and the statistics aggregations of table writes
 * (:3347-3357, :3424-3434) create the reference's factory (see INTEGRATION.md §2).  One output page of one row after finish(), also over
 * empty input.  NOT compiled here.
 */
package io.trino.operator.gpu;

import io.trino.operator.DriverContext;
import io.trino.operator.Operator;
import io.trino.operator.OperatorContext;
import io.trino.operator.OperatorFactory;
import io.trino.operator.gpu.GpuHashAggregationOperatorFactory.GpuAggregate;
import io.trino.sql.planner.plan.AggregationNode.Step;
import io.trino.sql.planner.plan.PlanNodeId;

import java.lang.foreign.MemorySegment;
import java.util.List;

import static com.google.common.base.Preconditions.checkState;

public class GpuAggregationOperatorFactory
        implements OperatorFactory
{
    private final int operatorId;
    private final PlanNodeId planNodeId;
    private final int[] inputTypes;              // tgpu_type per source channel: shapes the output row when no page arrives
    private final int[] outputTypes;             // one (SINGLE/FINAL) or the state columns (PARTIAL/INTERMEDIATE) per aggregate
    private final Step step;
    private final List<GpuAggregate> aggregates;
    private boolean closed;

    public GpuAggregationOperatorFactory(int operatorId, PlanNodeId planNodeId, int[] inputTypes, int[] outputTypes, Step step, List<GpuAggregate> aggregates)
    {
        this.operatorId = operatorId;
        this.planNodeId = planNodeId;
        this.inputTypes = inputTypes.clone();
        this.outputTypes = outputTypes.clone();
        this.step = step;
        this.aggregates = List.copyOf(aggregates);
    }

    @Override
    public Operator createOperator(DriverContext driverContext)
    {
        checkState(!closed, "Factory is already closed");
        OperatorContext operatorContext = driverContext.addOperatorContext(operatorId, planNodeId, "GpuAggregationOperator");
        GpuContexts.Handle gpu = GpuContexts.forCurrentDriver(driverContext);
        MemorySegment op = NativeSpecs.createGlobalAggregation(gpu, step, aggregates, inputTypes, MemorySegment.NULL);
        return new GpuOperator(operatorContext, gpu.context(), op, gpu.marshaller(inputTypes), outputTypes);
    }

    @Override
    public void noMoreOperators()
    {
        closed = true;
    }

    @Override
    public OperatorFactory duplicate()
    {
        return new GpuAggregationOperatorFactory(operatorId, planNodeId, inputTypes, outputTypes, step, aggregates);
    }
}
