/*
 * Base of every GPU-backed operator: the Operator protocol (M/operator/Operator.java:21-102) over a tgpu_op handle.
 * Input pages are batched by the PageMarshaller (a Java page is <= 8192 rows, a device launch wants ~1 M): addInput appends to the
 * batch and crosses the boundary once per batch; getOutput splits a device page back into <= 8192-row Java pages.
 * NOT compiled here (no JDK); tests/harness/driver_loop.cpp exercises the same call sequence against the real library.
 *
 * isBlocked(): every tgpu call returns when its result is on the host or its work is enqueued; the only waits are the stream
 * synchronisations inside getOutput (milliseconds - far below the 1 s driver quantum, M/operator/Driver.java:298), so the operator is
 * never "blocked" in the ListenableFuture sense and keeps the default NOT_BLOCKED.  The yield signal is honoured at batch granularity:
 * a batch is at most BATCH_ROWS rows.
 */
package io.trino.operator.gpu;

import com.google.common.util.concurrent.ListenableFuture;
import io.trino.memory.context.LocalMemoryContext;
import io.trino.operator.Operator;
import io.trino.operator.OperatorContext;
import io.trino.spi.Page;
import io.trino.spi.TrinoException;
import io.trino.spi.block.Block;
import io.trino.spi.block.PageMarshaller;

import java.lang.foreign.Arena;
import java.lang.foreign.MemorySegment;
import java.util.ArrayDeque;
import java.util.ArrayList;
import java.util.List;

import static io.trino.spi.StandardErrorCode.DIVISION_BY_ZERO;
import static io.trino.spi.StandardErrorCode.GENERIC_INSUFFICIENT_RESOURCES;
import static io.trino.spi.StandardErrorCode.GENERIC_INTERNAL_ERROR;
import static io.trino.spi.StandardErrorCode.INVALID_CAST_ARGUMENT;
import static io.trino.spi.StandardErrorCode.INVALID_FUNCTION_ARGUMENT;
import static io.trino.spi.StandardErrorCode.NOT_SUPPORTED;
import static io.trino.spi.StandardErrorCode.NUMERIC_VALUE_OUT_OF_RANGE;
import static java.lang.foreign.ValueLayout.ADDRESS;
import static java.lang.foreign.ValueLayout.JAVA_INT;
import static java.lang.foreign.ValueLayout.JAVA_LONG;

public class GpuOperator
        implements Operator
{
    protected final OperatorContext operatorContext;
    protected final LocalMemoryContext memoryContext;
    protected final MemorySegment ctx;       // tgpu_ctx* of the driver thread (GpuContexts.forCurrentDriver)
    protected final MemorySegment op;        // tgpu_op*
    private final PageMarshaller marshaller;
    private final int[] outputTypes;         // tgpu_type per output channel
    private final ArrayDeque<Page> ready = new ArrayDeque<>();
    private final ArrayDeque<Integer> readyTags = new ArrayDeque<>();   // per ready page: tagOf(device page it came from)
    protected int lastOutputTag;
    /** input pages of the batch in flight, for the blocks an operator passes through unchanged (tgpu_page_passthrough_channel) */
    private final List<Page> inFlight = new ArrayList<>();
    private boolean finishing;

    protected GpuOperator(OperatorContext operatorContext, MemorySegment ctx, MemorySegment op, PageMarshaller marshaller, int[] outputTypes)
    {
        this.operatorContext = operatorContext;
        this.memoryContext = operatorContext.localUserMemoryContext();
        this.ctx = ctx;
        this.op = op;
        this.marshaller = marshaller;
        this.outputTypes = outputTypes.clone();
    }

    @Override
    public OperatorContext getOperatorContext()
    {
        return operatorContext;
    }

    @Override
    public ListenableFuture<Void> isBlocked()
    {
        return NOT_BLOCKED;
    }

    @Override
    public boolean needsInput()
    {
        if (finishing || !ready.isEmpty()) {
            return false;
        }
        try (Arena arena = Arena.ofConfined()) {
            MemorySegment out = arena.allocate(JAVA_INT);
            check((int) TrinoGpuLibrary.OP_NEEDS_INPUT.invokeExact(op, out));
            return out.get(JAVA_INT, 0) != 0;
        }
        catch (Throwable e) {
            throw propagate(e);
        }
    }

    @Override
    public void addInput(Page page)
    {
        inFlight.add(page);
        if (marshaller.append(page)) {
            flushBatch();
        }
    }

    private void flushBatch()
    {
        if (!marshaller.hasBatch()) {
            return;
        }
        try (Arena arena = Arena.ofConfined()) {
            MemorySegment nativePage = marshaller.flush(arena);     // one tgpu_page over the pinned staging region
            check((int) TrinoGpuLibrary.OP_ADD_INPUT.invokeExact(op, nativePage));
            memoryContext.setBytes((long) TrinoGpuLibrary.OP_MEMORY_BYTES.invokeExact(op));
            drain(arena);
        }
        catch (Throwable e) {
            throw propagate(e);
        }
        finally {
            inFlight.clear();
        }
    }

    /** moves every device page the native operator has ready into `ready` as Java pages */
    private void drain(Arena arena)
            throws Throwable
    {
        while (true) {
            MemorySegment out = arena.allocate(ADDRESS);
            check((int) TrinoGpuLibrary.OP_GET_OUTPUT.invokeExact(op, out));
            MemorySegment devicePage = out.get(ADDRESS, 0);
            if (devicePage.equals(MemorySegment.NULL)) {
                return;
            }
            try {
                MemorySegment header = devicePage.reinterpret(PageMarshaller.PAGE.byteSize());
                long rows = header.get(JAVA_LONG, 8);
                MemorySegment columns = header.get(ADDRESS, 16).reinterpret(PageMarshaller.COLUMN.byteSize() * outputTypes.length);
                int[] passthrough = new int[outputTypes.length];
                long[] utf8Bytes = new long[outputTypes.length];
                boolean[] hasNulls = new boolean[outputTypes.length];
                Block[][] passthroughBlocks = new Block[outputTypes.length][];
                MemorySegment channelOut = arena.allocate(JAVA_INT);
                for (int channel = 0; channel < outputTypes.length; channel++) {
                    check((int) TrinoGpuLibrary.PAGE_PASSTHROUGH_CHANNEL.invokeExact(devicePage, channel, channelOut));
                    passthrough[channel] = channelOut.get(JAVA_INT, 0);
                    hasNulls[channel] = !columns.get(ADDRESS, channel * PageMarshaller.COLUMN.byteSize() + 32).equals(MemorySegment.NULL);
                    if (outputTypes[channel] == PageMarshaller.UTF8 && passthrough[channel] < 0) {
                        utf8Bytes[channel] = (long) TrinoGpuLibrary.PAGE_UTF8_BYTES.invokeExact(ctx, devicePage, channel);
                    }
                    if (passthrough[channel] >= 0) {
                        // LookupJoinPageBuilder.build :144-150: the probe blocks themselves, page by page of the batch in flight
                        Block[] blocks = new Block[inFlight.size()];
                        for (int i = 0; i < blocks.length; i++) {
                            blocks[i] = inFlight.get(i).getBlock(passthrough[channel]);
                        }
                        passthroughBlocks[channel] = blocks;
                    }
                }
                PageMarshaller.OutputShape shape = new PageMarshaller.OutputShape(outputTypes, rows, utf8Bytes);
                MemorySegment hostPage = marshaller.describeLanding(shape, passthrough, arena);
                check((int) TrinoGpuLibrary.PAGE_COPY_TO_HOST.invokeExact(ctx, devicePage, hostPage));
                boolean aligned = passthroughBlocks.length > 0 && java.util.Arrays.stream(passthroughBlocks).anyMatch(java.util.Objects::nonNull);
                // pass-through blocks keep the input page boundaries; otherwise cut at 8192 rows (PageProcessor.java:58 / LookupJoinPageBuilder.java:55-60)
                int tag = tagOf(devicePage);
                for (Page page : PageMarshaller.toPages(hostPage, shape, hasNulls, passthroughBlocks, aligned ? inFlight.get(0).getPositionCount() : 8192)) {
                    ready.add(page);
                    readyTags.add(tag);
                }
            }
            finally {
                TrinoGpuLibrary.PAGE_RELEASE.invokeExact(ctx, devicePage);
            }
        }
    }

    @Override
    public Page getOutput()
    {
        if (ready.isEmpty() && finishing) {
            flushBatch();
            try (Arena arena = Arena.ofConfined()) {
                drain(arena);
            }
            catch (Throwable e) {
                throw propagate(e);
            }
        }
        Integer tag = readyTags.poll();
        lastOutputTag = tag == null ? 0 : tag;
        return ready.poll();
    }

    /** per device page, read right after tgpu_op_get_output (e.g. the partition id of a partitioned-output page) */
    protected int tagOf(MemorySegment devicePage)
            throws Throwable
    {
        return 0;
    }

    @Override
    public void finish()
    {
        if (finishing) {
            return;     // re-entrant (M/operator/Driver.java:380-388)
        }
        flushBatch();
        finishing = true;
        try {
            check((int) TrinoGpuLibrary.OP_FINISH.invokeExact(op));
        }
        catch (Throwable e) {
            throw propagate(e);
        }
    }

    @Override
    public boolean isFinished()
    {
        if (!ready.isEmpty()) {
            return false;
        }
        try (Arena arena = Arena.ofConfined()) {
            MemorySegment out = arena.allocate(JAVA_INT);
            check((int) TrinoGpuLibrary.OP_IS_FINISHED.invokeExact(op, out));
            return out.get(JAVA_INT, 0) != 0;
        }
        catch (Throwable e) {
            throw propagate(e);
        }
    }

    @Override
    public void close()
    {
        try {
            TrinoGpuLibrary.OP_CLOSE.invokeExact(op);
            memoryContext.setBytes(0);
        }
        catch (Throwable e) {
            throw propagate(e);
        }
    }

    protected void check(int status)
    {
        if (status != 0) {
            throw failure(status, ctx);
        }
    }

    /** tgpu_status -> the exception the Java operator would have thrown (include/trino_gpu.h: tgpu_status) */
    static RuntimeException failure(int status, MemorySegment ctx)
    {
        String message = TrinoGpuLibrary.lastError(ctx);
        return switch (status) {
            case -3 -> new TrinoException(GENERIC_INSUFFICIENT_RESOURCES, message);
            case -4 -> new TrinoException(NUMERIC_VALUE_OUT_OF_RANGE, message);
            case -5 -> new TrinoException(DIVISION_BY_ZERO, message);
            case -8 -> new TrinoException(INVALID_CAST_ARGUMENT, message);
            case -9 -> new TrinoException(INVALID_FUNCTION_ARGUMENT, message);   // "Concatenated string is too large"
            case -6 -> new TrinoException(NOT_SUPPORTED, message);   // shapes the planner-side check (GpuSupport) should have kept on the Java operator
            case -1 -> new IllegalArgumentException(message);
            case -7 -> new IllegalStateException(message);
            default -> new TrinoException(GENERIC_INTERNAL_ERROR, message);   // -2 device failure
        };
    }

    private static RuntimeException propagate(Throwable e)
    {
        if (e instanceof RuntimeException runtimeException) {
            return runtimeException;
        }
        return new RuntimeException(e);
    }
}
