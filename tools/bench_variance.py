"""stddev_samp(l_quantity) and var_pop(l_extendedprice) over device-resident lineitem-shaped pages (2^24 rows each), against the same plan
with avg in place of each variance function, run alternately in one session, in three workloads: AggregationOperator (no keys), a
Q1-shaped group-by over 4 TINYINT keys (path S) and a BIGINT key with 10 M groups (the multipass path G).  Per repeat (--repeats, each
the median of --steps steps after --warmup, CUDA events around the whole step): ms of both plans, rows/s, and the fraction of 3.35 TB/s
under the byte model: each plan reads its two 8-byte columns once (16 bytes per row) plus the key column; the state is not counted.
The card name and power limit are read in the same run.

  python tools/bench_variance.py [--rows 600000000] [--steps 5] [--warmup 2] [--repeats 3]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from trino_b200 import abi                       # noqa: E402
from trino_b200 import operators as ops          # noqa: E402

PAGE_ROWS = 1 << 24
PEAK = 3.35e12


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True)
    name, power = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=600_000_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev)
    g.manual_seed(1)
    n = args.rows
    qty = torch.randint(1, 51, (n,), device=dev, generator=g).double()
    price = (torch.randint(90_000, 10_500_000, (n,), device=dev, generator=g).double() / 100)
    ctx = ops.Context(0)
    pages = []
    for b in range(0, n, PAGE_ROWS):
        m = min(PAGE_ROWS, n - b)
        pages.append(ops.DevicePage([ops.DeviceColumn(abi.FLOAT64, t[b:b + m].data_ptr(), m) for t in (qty, price)], m))
    flag = torch.randint(0, 4, (n,), device=dev, generator=g).to(torch.int8)             # Q1's 4 (returnflag, linestatus) groups
    big = torch.randint(0, 10_000_000, (n,), device=dev, generator=g)                        # 10 M BIGINT groups
    for k, b in enumerate(range(0, n, PAGE_ROWS)):
        m = min(PAGE_ROWS, n - b)
        pages[k].extra = {"flag": ops.DeviceColumn(abi.INT8, flag[b:b + m].data_ptr(), m), "big": ops.DeviceColumn(abi.INT64, big[b:b + m].data_ptr(), m)}
    A = ops.Aggregator
    plans = {"variance": [A(abi.AGG_STDDEV_SAMP, 1), A(abi.AGG_VAR_POP, 2)], "avg": [A(abi.AGG_AVG, 1), A(abi.AGG_AVG, 2)]}
    glob = {k: [A(a.function, a.input_channel - 1) for a in v] for k, v in plans.items()}
    workloads = {
        "global": ([pg for pg in pages], {k: ops.AggregationOperatorFactory(ctx, abi.STEP_SINGLE, v, input_types=[abi.FLOAT64, abi.FLOAT64])
                                          for k, v in glob.items()}),
        "q1_path_s": ([ops.DevicePage([pg.extra["flag"]] + pg.columns, pg.rows) for pg in pages],
                      {k: ops.HashAggregationOperatorFactory(ctx, [0], abi.STEP_SINGLE, v, 16) for k, v in plans.items()}),
        "bigint_10m_multipass": ([ops.DevicePage([pg.extra["big"]] + pg.columns, pg.rows) for pg in pages],
                                 {k: ops.HashAggregationOperatorFactory(ctx, [0], abi.STEP_SINGLE, v, 10_000_000) for k, v in plans.items()}),
    }
    # byte model: 16 bytes of arguments per row, plus the key (1 or 8 bytes) on the keyed workloads
    bytes_per_row = {"global": 16, "q1_path_s": 17, "bigint_10m_multipass": 24}

    def step(fac, pgs):
        op = fac.create_operator()
        for p in pgs:
            op.add_input(p)
            while op.get_output() is not None:
                pass
        op.finish()
        while not op.is_finished():
            op.get_output()
        op.close()

    def timed(fac, pgs):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        s.record()
        step(fac, pgs)
        e.record()
        torch.cuda.synchronize()
        return s.elapsed_time(e)

    name, power = card()
    res = {"card": name, "power_limit": power, "rows": n, "page_rows": PAGE_ROWS, "steps": args.steps, "warmup": args.warmup, "workloads": {}}
    for wname, (pgs, facs) in workloads.items():
        for _ in range(args.warmup):
            for f in facs.values():
                step(f, pgs)
        reps = []
        for _ in range(args.repeats):
            times = {k: [] for k in facs}
            for _ in range(args.steps):
                for k, f in facs.items():          # alternated step by step
                    times[k].append(timed(f, pgs))
            rep = {}
            for k, t in times.items():
                ms = sorted(t)[len(t) // 2]
                rep[k] = {"ms": round(ms, 3), "rows_per_s": n / (ms / 1e3), "frac_peak": n * bytes_per_row[wname] / (ms / 1e3) / PEAK}
            reps.append(rep)
        res["workloads"][wname] = reps
    print(json.dumps(res))
    ctx.close()


if __name__ == "__main__":
    main()
