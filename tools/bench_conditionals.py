"""Conditional expressions over device-resident lineitem-shaped pages (2^24 rows each), each against the same program with the conditional
replaced by its THEN branch, run alternately in one session.

  (1) Q14's CASE as a FilterAndProject (no filter): CASE WHEN p_type LIKE 'PROMO%' THEN l_extendedprice * (1 - l_discount) ELSE 0 END,
      decimal(26,4) over decimal(12,2) columns; the THEN program projects l_extendedprice * (1 - l_discount)
  (2) Q12's CASE: FilterAndProject [key, CASE WHEN o_orderpriority IN ('1-URGENT', '2-HIGH') THEN 1 ELSE 0 END] -> HashAggregationOperator
      sum by an 8-value key; the THEN program projects the constant 1
  (3) sum(IF(l_discount > 0.05, l_extendedprice, 0.0)) in DOUBLE through AggregationOperator's fused pre-stage (tg_agg_global_jit); the
      THEN program sums l_extendedprice

The columns come from the generators of bench_decimal_project.py (decimal(12,2) as INT64 unscaled values, and their DOUBLE copies) and
bench_varchar_filter.py (device UTF8 pages gathered from a string pool).  Each workload reports, per repeat (--repeats, each the median
of --steps steps after --warmup, CUDA events around the whole step), the ms of both programs, rows/s, and a byte model (bytes each
program must read and write, below) as a fraction of 3.35 TB/s.  The card name and power limit are read in the same run.

  python tools/bench_conditionals.py [--rows 600000000] [--steps 5] [--warmup 2] [--repeats 3]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench_decimal_project as bdp              # noqa: E402
import bench_varchar_filter as bvf               # noqa: E402
from trino_b200 import abi                       # noqa: E402
from trino_b200 import operators as ops          # noqa: E402

PAGE_ROWS = bdp.PAGE_ROWS
PEAK = bdp.PEAK
B, D, S, DEC, BOOL = abi.V_BIGINT, abi.V_DOUBLE, abi.V_VARCHAR, abi.V_DECIMAL, abi.V_BOOLEAN
T = bdp.T
P_TYPES = [f"{a} {b} {c}".encode() for a in ("STANDARD", "SMALL", "MEDIUM", "LARGE", "ECONOMY", "PROMO")
           for b in ("ANODIZED", "BURNISHED", "PLATED", "POLISHED", "BRUSHED") for c in ("TIN", "NICKEL", "BRASS", "STEEL", "COPPER")]
PRIORITIES = [b"1-URGENT", b"2-HIGH", b"3-MEDIUM", b"4-NOT SPECIFIED", b"5-LOW"]


def string_pages(pool, n, dev, seed):
    g = torch.Generator(device=dev)
    g.manual_seed(seed)
    ids = torch.randint(0, len(pool), (n,), device=dev, generator=g)
    pages = bvf.utf8_pages(pool, ids, dev)
    mean_len = float(np.mean([len(p) for p in pool]))
    return pages, mean_len


def device_pages(n, cols):
    """cols: list of (tensor, type) or a list of utf8 pages (one entry per page) for a VARCHAR channel"""
    out = []
    for k, b in enumerate(range(0, n, PAGE_ROWS)):
        dc = []
        for c in cols:
            if isinstance(c, list):
                dc.append(bvf.col_utf8(c[k]))
            else:
                t, ty = c
                dc.append(ops.DeviceColumn(ty, t[b:b + PAGE_ROWS].data_ptr(), min(PAGE_ROWS, n - b), None))
        out.append(ops.DevicePage(dc, min(PAGE_ROWS, n - b)))
    return out


def step_global(ctx, make_op, pgs):
    op = make_op()
    ctx.synchronize()
    ctx.timer_start()
    for p in pgs:
        op.add_input(p)
    op.finish()
    outs = []
    while True:
        o = op.get_output()
        if o is None:
            break
        outs.append(o)
    ms = ctx.timer_stop_ms()
    op.close()
    return ms, outs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=600_000_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_conditionals.py measures on the GPU and found none")
    name, power = bdp.card()
    ctx = ops.Context(0)
    dev = torch.device("cuda:0")
    n = args.rows
    c = bdp.columns(n, dev, 20)
    for k in ("ship", "flag", "status", "qty", "tax", "qty_d", "tax_d"):
        del c[k]
    key = torch.randint(0, 8, (n,), device=dev, dtype=torch.int8)
    ptype, ptype_len = string_pages(P_TYPES, n, dev, 21)
    prio, prio_len = string_pages(PRIORITIES, n, dev, 22)
    torch.cuda.synchronize()
    res = {"card": name, "power_limit": power, "rows": n, "page_rows": PAGE_ROWS, "steps": args.steps, "warmup": args.warmup,
           "repeats": args.repeats}
    print(json.dumps(res), flush=True)

    def fp(prog, pgs, chain=None):
        return lambda: bdp.step(ctx, lambda: ops.FilterAndProjectOperatorFactory(ctx, prog).create_operator(), pgs, chain=chain)

    def report(key_, runs, bytes_cond, bytes_then):
        out = {"cond_ms": [], "then_ms": [], "cond_rows_per_s": [], "cond_of_peak": [], "then_of_peak": []}
        for (tc, _), (tt, _) in runs:
            out["cond_ms"].append(round(tc, 3))
            out["then_ms"].append(round(tt, 3))
            out["cond_rows_per_s"].append(n / tc * 1e3)
            out["cond_of_peak"].append(round(bytes_cond / tc * 1e3 / PEAK, 3))
            out["then_of_peak"].append(round(bytes_then / tt * 1e3 / PEAK, 3))
        out["cond_bytes"], out["then_bytes"] = bytes_cond, bytes_then
        res[key_] = out
        print(key_, json.dumps(out), flush=True)

    # (1) Q14's CASE: channels 0 p_type, 1 extendedprice, 2 discount
    pg14 = device_pages(n, [ptype, (c["ep"], abi.INT64), (c["disc"], abi.INT64)])
    ep, disc = ops.Col(1, DEC, T), ops.Col(2, DEC, T)
    rev = ops.Call(abi.EX_MUL, ep, ops.Call(abi.EX_SUB, ops.Const(1, DEC, (1, 0)), disc))
    q14 = ops.Case([(ops.Call(abi.EX_LIKE, ops.Col(0, S), pattern="PROMO%"), rev)], ops.Const(0, DEC, rev.dtype))
    runs = [bdp.alternate(ctx, fp(ops.PageProcessorProgram(None, [q14]), pg14), fp(ops.PageProcessorProgram(None, [rev]), pg14),
                          args.steps, args.warmup) for _ in range(args.repeats)]
    # bytes: p_type offsets (4) and bytes, extendedprice and discount (16) read; the decimal(26,4) cell (16) and its null byte written
    report("q14_case_project", runs, int(n * (4 + ptype_len + 16 + 17)), int(n * (16 + 17)))
    del pg14

    # (2) Q12's CASE -> HashAggregationOperator: channels 0 key, 1 o_orderpriority
    pg12 = device_pages(n, [(key, abi.INT8), prio])
    urgent = ops.Call(abi.EX_IN, ops.Col(1, S), in_list=["1-URGENT", "2-HIGH"])
    q12 = ops.Case([(urgent, ops.Const(1, B))], ops.Const(0, B))
    agg = lambda: ops.HashAggregationOperatorFactory(ctx, [0], abi.STEP_SINGLE, [ops.Aggregator(abi.AGG_SUM, 1)], 16).create_operator()
    runs = [bdp.alternate(ctx, fp(ops.PageProcessorProgram(None, [0, q12]), pg12, chain=agg),
                          fp(ops.PageProcessorProgram(None, [0, ops.Const(1, B)]), pg12, chain=agg), args.steps, args.warmup)
            for _ in range(args.repeats)]
    # bytes: FilterAndProject reads key (1), priority offsets (4) and bytes, writes key, value and null bytes (1 + 8 + 2); the
    # aggregation reads those 11 again
    report("q12_case_project_hash_agg", runs, int(n * (1 + 4 + prio_len + 11 + 11)), int(n * (1 + 11 + 11)))
    del pg12

    # (3) sum(IF(l_discount > 0.05, l_extendedprice, 0.0)) in the global pre-stage: channels 0 extendedprice, 1 discount (DOUBLE)
    pg3 = device_pages(n, [(c["ep_d"], abi.FLOAT64), (c["disc_d"], abi.FLOAT64)])
    cond = ops.If(ops.Call(abi.EX_GT, ops.Col(1, D), ops.Const(0.05, D)), ops.Col(0, D), ops.Const(0.0, D))
    types = [abi.FLOAT64, abi.FLOAT64]

    def glob(e):
        pre = ops.PageProcessorProgram(None, [e])
        return lambda: step_global(ctx, lambda: ops.AggregationOperatorFactory(ctx, abi.STEP_SINGLE, [ops.Aggregator(abi.AGG_SUM, 0)], pre=pre,
                                                                               input_types=types).create_operator(), pg3)
    runs = [bdp.alternate(ctx, glob(cond), glob(ops.Col(0, D)), args.steps, args.warmup) for _ in range(args.repeats)]
    # bytes: extendedprice and discount read (16); the THEN program reads extendedprice only (8)
    report("sum_if_global_pre_stage", runs, n * 16, n * 8)
    print(json.dumps(res))
    ctx.close()


if __name__ == "__main__":
    main()
