"""DECIMAL FilterAndProject over device-resident lineitem pages (2^24 rows each), against the same programs over DOUBLE columns.

  (a) Q1's FilterAndProject: l_shipdate <= cutoff; returnflag, linestatus, quantity, extendedprice, extendedprice * (1 - discount)
      (decimal(26,4)), extendedprice * (1 - discount) * (1 + tax) (decimal(38,6)), discount.  The DOUBLE program is bench.py's q1_program().
  (b) Q6: the Q6 filter, projecting extendedprice * discount (decimal(25,4))
  (c) the division path: extendedprice / quantity (decimal(27,15): a 128-bit dividend)
  (d) decimal Q1 end to end: FilterAndProject -> HashAggregation (decimal sum and avg) per step; the fused DOUBLE Q1 for context

Every decimal column is decimal(12,2) as TPC-H's DECIMAL mapping gives it (INT64 unscaled values).  Each workload alternates a DOUBLE
step and a DECIMAL step, warm-up first, and reports the median of --steps steps (CUDA events), rows/s, a byte model from the code below
(bytes each program must read and write) and the achieved bytes/s as a fraction of 3.35 TB/s.  The card name and power limit are read in
the same run.

  python tools/bench_decimal_project.py [--rows 600000000] [--steps 5] [--warmup 2]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import q1                                        # noqa: E402
from trino_b200 import abi                       # noqa: E402
from trino_b200 import operators as ops          # noqa: E402

PAGE_ROWS = 1 << 24
PEAK = 3.35e12
B, D, DEC = abi.V_BIGINT, abi.V_DOUBLE, abi.V_DECIMAL
T = (12, 2)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=20).stdout
        name, power = [x.strip() for x in q.splitlines()[0].split(",")]
        return name, power
    except Exception:      # noqa: BLE001 - the table still names the card
        return torch.cuda.get_device_name(0), "unknown"


def columns(n, dev, seed):
    """lineitem columns on the device: shipdate INT32, returnflag / linestatus INT8, then quantity, extendedprice, discount, tax as
    decimal(12,2) unscaled INT64 and as DOUBLE"""
    g = torch.Generator(device=dev)
    g.manual_seed(seed)
    c = {
        "ship": torch.randint(8036, 10561, (n,), device=dev, dtype=torch.int32, generator=g),
        "flag": torch.randint(0, 3, (n,), device=dev, dtype=torch.int8, generator=g),
        "status": torch.randint(0, 2, (n,), device=dev, dtype=torch.int8, generator=g),
        "qty": torch.randint(100, 5001, (n,), device=dev, dtype=torch.int64, generator=g),
        "ep": torch.randint(90_000, 10_500_000, (n,), device=dev, dtype=torch.int64, generator=g),
        "disc": torch.randint(0, 11, (n,), device=dev, dtype=torch.int64, generator=g),
        "tax": torch.randint(0, 9, (n,), device=dev, dtype=torch.int64, generator=g),
    }
    for k in ("qty", "ep", "disc", "tax"):
        c[k + "_d"] = c[k].to(torch.float64) / 100.0
    return c


def pages(c, names, types):
    out = []
    n = c["ship"].numel()
    for b in range(0, n, PAGE_ROWS):
        cols = []
        for nm, ty in zip(names, types):
            t = c[nm][b:b + PAGE_ROWS]
            cols.append(ops.DeviceColumn(ty, t.data_ptr(), t.numel(), None))
        out.append(ops.DevicePage(cols, min(PAGE_ROWS, n - b)))
    return out


def step(ctx, make_op, pgs, chain=None):
    """one step: every page through the operator (and `chain`, fed the device outputs); ms (CUDA events) and the rows it produced"""
    op = make_op()
    nxt = chain() if chain else None
    outs = []
    ctx.synchronize()
    ctx.timer_start()
    for p in pgs:
        op.add_input(p)
        o = op.get_output_device()
        if o is not None:
            if nxt:          # the aggregation has consumed the page: free it now, as a driver would
                nxt.add_input(o)
                outs.append(o.rows)
                o.release()
            else:
                outs.append(o)
    if nxt:
        nxt.finish()
        while nxt.get_output() is not None:
            pass
    ms = ctx.timer_stop_ms()
    rows = sum(o if isinstance(o, int) else o.rows for o in outs)
    for o in outs:
        if not isinstance(o, int):
            o.release()
    op.close()
    if nxt:
        nxt.close()
    return ms, rows


def alternate(ctx, a, b, steps, warmup):
    """(median ms, rows) of workload a and of workload b, run alternately"""
    ta, tb, ra, rb = [], [], 0, 0
    for s in range(warmup + steps):
        ms_a, ra = a()
        ms_b, rb = b()
        if s >= warmup:
            ta.append(ms_a)
            tb.append(ms_b)
    return (float(np.median(ta)), ra), (float(np.median(tb)), rb)


# ---- programs (channels: 0 ship, 1 flag, 2 status, 3 qty, 4 ep, 5 disc, 6 tax) and their byte models --------------------------------
def q1_decimal():
    one = ops.Const(1, DEC, (1, 0))
    ep, disc, tax = ops.Col(4, DEC, T), ops.Col(5, DEC, T), ops.Col(6, DEC, T)
    dp = ops.Call(abi.EX_MUL, ep, ops.Call(abi.EX_SUB, one, disc))
    charge = ops.Call(abi.EX_MUL, dp, ops.Call(abi.EX_ADD, one, tax))
    return ops.PageProcessorProgram(ops.Call(abi.EX_LE, ops.Col(0, B), ops.Const(q1.CUTOFF, B)), [1, 2, 3, 4, dp, charge, 5])


def q1_bytes(n, m, wide):
    """filter pass: ship (4) read, a flag byte written and read back; projection of m rows: flag, status, qty, ep, disc, tax read
    (1 + 1 + 4 x 8), flag, status, qty, ep, disc written (1 + 1 + 3 x 8) and the two computed columns (8 or 16 each) with their null-map
    bytes (1 each)"""
    computed = 2 * (16 if wide else 8) + 2
    return n * (4 + 2) + m * (34 + 26 + computed)


def q6(decimal):
    if decimal:
        ship, qty, ep, disc = ops.Col(0, B), ops.Col(3, DEC, T), ops.Col(4, DEC, T), ops.Col(5, DEC, T)
        c = lambda v: ops.Const(v, DEC, T)
    else:
        ship, qty, ep, disc = ops.Col(0, B), ops.Col(3, D), ops.Col(4, D), ops.Col(5, D)
        c = lambda v: ops.Const(v / 100.0, D)
    flt = ops.Call(abi.EX_AND, ops.Call(abi.EX_BETWEEN, ship, ops.Const(8766, B), ops.Const(9130, B)),
                   ops.Call(abi.EX_AND, ops.Call(abi.EX_BETWEEN, disc, c(5), c(7)), ops.Call(abi.EX_LT, qty, c(2400))))
    return ops.PageProcessorProgram(flt, [ops.Call(abi.EX_MUL, ep, disc)])


def q6_bytes(n, m, wide):
    """filter: ship, disc, qty read (4 + 8 + 8), a flag byte written and read; projection: ep, disc read, the product and its null map"""
    return n * (20 + 2) + m * (16 + (16 if wide else 8) + 1)


def div(decimal):
    if decimal:
        e = ops.Call(abi.EX_DIV, ops.Col(4, DEC, T), ops.Col(3, DEC, T))
        assert e.dtype == (27, 15)
    else:
        e = ops.Call(abi.EX_DIV, ops.Col(4, D), ops.Col(3, D))
    return ops.PageProcessorProgram(None, [e])


def div_bytes(n, wide):
    return n * (16 + (16 if wide else 8) + 1)


def q1_aggs_decimal():
    A = ops.Aggregator
    return [A(abi.AGG_SUM_DECIMAL, 2), A(abi.AGG_SUM_DECIMAL, 3), A(abi.AGG_SUM_DECIMAL, 4), A(abi.AGG_SUM_DECIMAL, 5),
            A(abi.AGG_AVG_DECIMAL, 2), A(abi.AGG_AVG_DECIMAL, 3), A(abi.AGG_AVG_DECIMAL, 6), A(abi.AGG_COUNT_STAR)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=600_000_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    name, power = card()
    ctx = ops.Context(0)
    dev = torch.device("cuda:0")
    n = args.rows
    c = columns(n, dev, 20)
    fixed = ["ship", "flag", "status"]
    ft = [abi.INT32, abi.INT8, abi.INT8]
    dec_pages = pages(c, fixed + ["qty", "ep", "disc", "tax"], ft + [abi.INT64] * 4)
    dbl_pages = pages(c, fixed + ["qty_d", "ep_d", "disc_d", "tax_d"], ft + [abi.FLOAT64] * 4)
    res = {"card": name, "power_limit": power, "rows": n, "page_rows": PAGE_ROWS, "steps": args.steps, "warmup": args.warmup}

    def fp(prog, pgs):
        return lambda: step(ctx, lambda: ops.FilterAndProjectOperatorFactory(ctx, prog).create_operator(), pgs)

    def report(key, dbl, dec, bytes_dbl, bytes_dec):
        (td, rd), (tx, rx) = dbl, dec
        bd, bx = bytes_dbl(rd), bytes_dec(rx)
        res[key] = {"double_ms": td, "decimal_ms": tx, "rows_out": rx, "rows_per_s_decimal": n / tx * 1e3,
                    "double_bytes": bd, "decimal_bytes": bx, "double_bytes_per_s": bd / td * 1e3, "decimal_bytes_per_s": bx / tx * 1e3,
                    "double_of_peak": bd / td * 1e3 / PEAK, "decimal_of_peak": bx / tx * 1e3 / PEAK,
                    "decimal_vs_double_bytes_per_s": (bx / tx) / (bd / td)}
        print(key, json.dumps(res[key]), flush=True)

    dbl, dec = alternate(ctx, fp(q1.q1_program(), dbl_pages), fp(q1_decimal(), dec_pages), args.steps, args.warmup)
    report("a_q1_project", dbl, dec, lambda m: q1_bytes(n, m, False), lambda m: q1_bytes(n, m, True))
    dbl, dec = alternate(ctx, fp(q6(False), dbl_pages), fp(q6(True), dec_pages), args.steps, args.warmup)
    report("b_q6_project", dbl, dec, lambda m: q6_bytes(n, m, False), lambda m: q6_bytes(n, m, True))
    dbl, dec = alternate(ctx, fp(div(False), dbl_pages), fp(div(True), dec_pages), args.steps, args.warmup)
    report("c_division", dbl, dec, lambda m: div_bytes(n, False), lambda m: div_bytes(n, True))
    # (d): decimal Q1 as FilterAndProject -> HashAggregation; the fused DOUBLE Q1 (one operator) for context
    fused = lambda: step_fused(ctx, dbl_pages)
    e2e = lambda: step(ctx, lambda: ops.FilterAndProjectOperatorFactory(ctx, q1_decimal()).create_operator(), dec_pages,
                       chain=lambda: ops.HashAggregationOperatorFactory(ctx, [0, 1], abi.STEP_SINGLE, q1_aggs_decimal(), 16).create_operator())
    (tf, _), (te, _) = alternate(ctx, fused, e2e, args.steps, args.warmup)
    res["d_q1_end_to_end"] = {"fused_double_q1_ms": tf, "decimal_q1_ms": te, "decimal_rows_per_s": n / te * 1e3}
    print("d_q1_end_to_end", json.dumps(res["d_q1_end_to_end"]), flush=True)
    print(json.dumps(res))
    ctx.close()


def step_fused(ctx, pgs):
    """one step of the fused DOUBLE Q1 (filter + project + GROUP BY in one operator)"""
    op = q1.q1_factory(ctx, fused=True).create_operator()
    ctx.synchronize()
    ctx.timer_start()
    for p in pgs:
        op.add_input(p)
    op.finish()
    while op.get_output() is not None:
        pass
    ms = ctx.timer_stop_ms()
    op.close()
    return ms, 0


if __name__ == "__main__":
    main()
