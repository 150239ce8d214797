#!/usr/bin/env python
"""Secondary operator micro-benchmarks on device-resident synthetic columns (not the headline bench):
FilterAndProject (Q1 program), BIGINT high-cardinality GROUP BY + sum, PagePartitioner.  Prints one JSON line each."""
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402

from q1 import q1_program  # noqa: E402
from trino_b200 import abi  # noqa: E402
from trino_b200 import operators as ops  # noqa: E402

PEAK = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"] if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else 3350.0   # H100 SXM data sheet HBM3 bandwidth


def timed(ctx, fn, reps=5, warm=2):
    for _ in range(warm):
        fn()
    ctx.timer_start()
    for _ in range(reps):
        fn()
    return ctx.timer_stop_ms() / reps


def main():
    ctx = ops.Context(0)
    lib = ctx.lib
    n = int(float(sys.argv[1])) if len(sys.argv) > 1 else 300_000_000
    # ---- FilterAndProject, Q1 program
    spec = [(abi.INT32, 4), (abi.INT8, 1), (abi.INT8, 1), (abi.FLOAT64, 8), (abi.FLOAT64, 8), (abi.FLOAT64, 8), (abi.FLOAT64, 8)]
    ptrs = [ctx.malloc(n * sz) for _, sz in spec]
    ctx.check(lib.tgpu_synth_lineitem_q1(ctx.h, n, 0, 0x7C01, *[C.c_void_p(p) for p in ptrs]))
    page = ops.DevicePage([ops.DeviceColumn(t, p, n) for (t, _), p in zip(spec, ptrs)], n)
    fp = ops.FilterAndProjectOperatorFactory(ctx, q1_program()).create_operator()
    rows_out = [0]

    def run_fp():
        fp.add_input(page)
        o = fp.get_output_device()
        rows_out[0] = o.rows
        o.release()
    ms = timed(ctx, run_fp)
    sel = rows_out[0] / n
    alg = 38 + sel * (2 + 5 * 8)      # read all input columns once, write 2 key bytes + 5 doubles per selected row
    print(json.dumps({"op": "FilterAndProject(Q1 program)", "rows": n, "ms": ms, "rows_per_s": n / ms * 1e3, "selectivity": sel,
                      "algorithmic_bytes_per_row": alg, "frac_of_measured_peak": alg * n / ms * 1e3 / 1e9 / PEAK}))
    fp.close()
    for p in ptrs:
        ctx.free(p)
    # ---- BIGINT GROUP BY (high cardinality) + sum(double)
    m = n // 2
    groups = 10_000_000
    d_keys = ctx.malloc(m * 8)
    ctx.check(lib.tgpu_synth_orders_keys(ctx.h, groups, 0, min(groups, m), 0x55, 1, C.c_void_p(d_keys)))   # first `groups` rows: a permutation
    if m > groups:   # remaining rows: shuffled keys again (every key seen several times)
        for lo in range(groups, m, groups):
            cnt = min(groups, m - lo)
            ctx.check(lib.tgpu_synth_orders_keys(ctx.h, groups, 0, cnt, 0x77 + lo, 1, C.c_void_p(d_keys + lo * 8)))
    d_val = ctx.malloc(m * 8)
    ctx.check(lib.tgpu_synth_lineitem_keys(ctx.h, m, 0, m, 1, 0, C.c_void_p(d_val)))   # any int64 payload
    gpage = ops.DevicePage([ops.DeviceColumn(abi.INT64, d_keys, m), ops.DeviceColumn(abi.INT64, d_val, m)], m)
    f = ops.HashAggregationOperatorFactory(ctx, [0], abi.STEP_SINGLE, [ops.Aggregator(abi.AGG_SUM, 1), ops.Aggregator(abi.AGG_COUNT_STAR)], expected_groups=groups)
    gcount = [0]

    def run_agg():
        op = f.create_operator()
        op.add_input(gpage)
        gcount[0] = op.group_count()
        op.close()
    ms = timed(ctx, run_agg, reps=3, warm=1)
    print(json.dumps({"op": "HashAggregation(BIGINT key, sum+count)", "rows": m, "groups": gcount[0], "ms": ms, "rows_per_s": m / ms * 1e3,
                      "algorithmic_bytes_per_row": 36, "frac_of_measured_peak": 36 * m / ms * 1e3 / 1e9 / PEAK}))
    # ---- PagePartitioner: 8 partitions, rows of key + payload (W = 16)
    part = ops.PartitionedOutputOperatorFactory(ctx, [0], 8).create_operator()

    def run_part():
        part.add_input(gpage)
        while True:
            o = part.get_output_device()
            if o is None:
                break
            o.release()
    ms = timed(ctx, run_part, reps=3, warm=1)
    print(json.dumps({"op": "PartitionedOutput(8 partitions, W=16)", "rows": m, "ms": ms, "rows_per_s": m / ms * 1e3,
                      "algorithmic_bytes_per_row": 36, "frac_of_measured_peak": 36 * m / ms * 1e3 / 1e9 / PEAK}))
    part.close()
    ctx.close()


if __name__ == "__main__":
    main()
