"""TPC-H Q6 through the GPU AggregationOperator over device-resident synthetic lineitem, with an A/B against the same query through
HashAggregationOperatorFactory (the keyed small-group path) keyed on an all-zero INT8 column.  Prints one JSON line.

    python tools/bench_q6.py [--sf 100] [--steps 5] [--warmup 2] [--ab 3]

Bytes per row: the 28 B/row model reads shipdate (4) + quantity, extendedprice, discount (8 each) for every row.  The sector model
counts what the kernel reads with deferred loads: 20 B/row for the filter columns plus 8 B x the fraction of 4-row groups with a
selected row for extendedprice (counted on the SF1 rows of the same generator).  Under the 28 B/row model the fraction of the data-sheet
bandwidth can exceed 1.0: the kernel does not read all of those bytes."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

SEED = 0x7C01
HBM_GBS = 3350.0          # H100 SXM5 80 GB data sheet (HBM3)


def device_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    name, power = [x.strip() for x in r.stdout.strip().split(",")[:2]] if r.returncode == 0 and "," in r.stdout else ("?", "?")
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sf", type=float, default=100)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--ab", type=int, default=3)
    args = ap.parse_args()
    import oracle_lib as o
    from q6 import q6_factory, q6_filter, q6_oracle, q6_selected
    from q1 import q1_host_page
    from trino_b200 import abi
    from trino_b200 import operators as ops

    ctx = ops.Context(0)
    # correctness at SF1 against the oracle, and the fraction of 4-row groups with a selected row
    cols1 = o.synth_lineitem_q1(6_000_000, 0, SEED)
    got = ops.drive(q6_factory(ctx).create_operator(), [q1_host_page(cols1)])[0].rows()[0]
    rev, cnt = q6_oracle(cols1)
    assert got[1] == cnt and abs(got[0] - rev) <= 1e-6 * abs(rev), (got, rev, cnt)
    sel = q6_selected(cols1)
    groups = sel[: len(sel) // 4 * 4].reshape(-1, 4).any(axis=1)
    group_frac = float(groups.mean())

    n = int(6_000_000 * args.sf)
    spec = [(abi.INT32, 4), (abi.INT8, 1), (abi.INT8, 1), (abi.FLOAT64, 8), (abi.FLOAT64, 8), (abi.FLOAT64, 8), (abi.FLOAT64, 8)]
    ptrs = [ctx.malloc(n * sz) for _, sz in spec]
    ctx.check(ctx.lib.tgpu_synth_lineitem_q1(ctx.h, n, 0, SEED, *[C.c_void_p(p) for p in ptrs]))
    zero = ctx.to_device(np.zeros(n, dtype=np.int8))
    dcols = [ops.DeviceColumn(t, p, n) for (t, _), p in zip(spec, ptrs)]
    page = ops.DevicePage(dcols, n)
    keyed_page = ops.DevicePage(dcols + [ops.DeviceColumn(abi.INT8, zero, n)], n)
    global_f = q6_factory(ctx)
    # the same query on the keyed operator: projections (zero key, extendedprice * discount)
    D = abi.V_DOUBLE
    keyed_prog = ops.PageProcessorProgram(q6_filter(), [7, ops.Call(abi.EX_MUL, ops.Col(4, D), ops.Col(5, D))])
    keyed_f = ops.HashAggregationOperatorFactory(ctx, [0], abi.STEP_SINGLE, [ops.Aggregator(abi.AGG_SUM, 1), ops.Aggregator(abi.AGG_COUNT_STAR)],
                                                 expected_groups=1, pre=keyed_prog)

    def run(factory, pg):
        op = factory.create_operator()
        op.add_input(pg)
        op.finish()
        out = op.get_output()
        op.close()
        return out.rows()[0]

    def measure(factory, pg, reps):
        kms = 0.0
        ctx.timer_start()
        for _ in range(reps):
            r = run(factory, pg)
            kms += ctx.last_kernel_ms()
        return ctx.timer_stop_ms() / reps, kms / reps, r

    for _ in range(args.warmup):
        g_row = run(global_f, page)
        k_row = run(keyed_f, keyed_page)
    step_ms, kernel_ms, g_row = measure(global_f, page, max(5, args.steps))
    ab = {"global": [], "keyed": []}
    for _ in range(max(3, args.ab)):
        ab["global"].append(measure(global_f, page, 3)[:2])
        ab["keyed"].append(measure(keyed_f, keyed_page, 3)[:2])
    k_row = run(keyed_f, keyed_page)
    assert g_row[1] == k_row[2] and abs(g_row[0] - k_row[1]) <= 1e-9 * abs(k_row[1]), (g_row, k_row)
    name, power = device_info()
    bytes28 = 28.0 * n
    bytes_sector = (20.0 + 8.0 * group_frac) * n
    med = lambda xs, i: float(np.median([x[i] for x in xs]))
    out = {
        "metric": "q6_input_rows_per_sec", "value": n / (step_ms * 1e-3), "unit": "rows/s", "rows": n, "sf": args.sf,
        "step_ms": step_ms, "kernel_ms": kernel_ms, "kernel": "tg_agg_global_jit",
        "hbm_frac_28B_model": bytes28 / (kernel_ms * 1e-3) / 1e9 / HBM_GBS,
        "hbm_frac_sector_model": bytes_sector / (kernel_ms * 1e-3) / 1e9 / HBM_GBS,
        "sector_model_bytes_per_row": 20.0 + 8.0 * group_frac, "groups_of_4_with_a_selected_row": group_frac,
        "note": "fractions of the data-sheet HBM bandwidth (3350 GB/s); the 28 B/row model can exceed 1.0 because deferred loads skip "
                "extendedprice sectors whose 4 rows all fail the filter; group fraction counted on SF1 rows of the same generator",
        "ab_median_ms": {"global_step": med(ab["global"], 0), "global_kernel": med(ab["global"], 1),
                         "keyed_step": med(ab["keyed"], 0), "keyed_kernel": med(ab["keyed"], 1)},
        "ab_runs_ms": ab, "result": {"revenue": g_row[0], "count": g_row[1]}, "sf1_oracle_check": "ok",
        "device": name, "power_limit": power,
    }
    print(json.dumps(out))
    for p in ptrs + [zero]:
        ctx.free(p)
    ctx.close()


if __name__ == "__main__":
    main()
