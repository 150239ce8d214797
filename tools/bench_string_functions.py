"""String functions in FilterAndProject over device-resident pages at SF100 scale.

  (a) 150 M customer rows, synthetic c_phone 'CC-XXX-XXX-XXXX':  substring(c_phone, 1, 2) IN (Q22's seven codes), projecting
      substring(c_phone, 1, 2) and c_acctbal (Q22's customer scan)
  (b) 150 M orders rows, o_comment of 19-78 bytes:                 substr(o_comment, 1, 20), no filter
  (c) the same o_comment column:                                   trim(o_comment) WHERE length(o_comment) BETWEEN 40 AND 60
  (c') the same filter with o_comment passed through:              the existing gather (tg_utf8_copy_kernel), for the same output bytes
  (d) o_orderpriority || '-' || o_clerk, no filter
Strings are gathered on the device from seeded pools, so the expected rows and bytes are exact (tests/string_function_reference.py over
each pool entry, weighted by how often it was drawn).  Pages hold 2^24 rows.  Reports, per workload: the median step time (CUDA events,
after warm-up), the time of each kernel in one profiled step (torch.profiler), the byte model per row and its fraction of 3.35 TB/s, with
the card name and power limit read in the same run.

  python tools/bench_string_functions.py [--rows 150000000] [--steps 5] [--warmup 2]
"""
import argparse
import json
import os
import sys
from collections import defaultdict

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, HERE)

import string_function_reference as sref                                       # noqa: E402
from bench_varchar_filter import PEAK, card, col_fixed, col_utf8, comment_pool, utf8_pages     # noqa: E402
from trino_b200 import abi                                                       # noqa: E402
from trino_b200 import operators as ops                                          # noqa: E402

S, B = abi.V_VARCHAR, abi.V_BIGINT
Q22_CODES = ["13", "31", "23", "29", "30", "18", "17"]
PRIORITIES = [b"1-URGENT", b"2-HIGH", b"3-MEDIUM", b"4-NOT SPECIFIED", b"5-LOW"]


def step(ctx, prog, pages):
    """one step: every page through one operator; (ms, output rows, output bytes of VARCHAR column 0)"""
    op = ops.FilterAndProjectOperatorFactory(ctx, prog).create_operator()
    outs = []
    ctx.synchronize()
    ctx.timer_start()
    for p in pages:
        op.add_input(p)
        o = op.get_output_device()
        if o is not None:
            outs.append(o)
    ms = ctx.timer_stop_ms()
    rows = sum(o.rows for o in outs)
    nbytes = 0
    for o in outs:
        c = o.column(0)
        if c.type == abi.UTF8 and o.rows:
            off = ctx.to_host(c.offsets + 4 * o.rows, np.int32, 1)
            nbytes += int(off[0])
        o.release()
    op.close()
    return ms, rows, nbytes


def run(ctx, prog, pages, steps, warmup):
    times, rows, nbytes = [], 0, 0
    for s in range(warmup + steps):
        ms, rows, nbytes = step(ctx, prog, pages)
        if s >= warmup:
            times.append(ms)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        step(ctx, prog, pages)
    kernels = defaultdict(float)
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and "memcpy" not in e.name.lower() and "memset" not in e.name.lower():
            kernels[e.name.replace("(anonymous namespace)::", "").split("(")[0].split("<")[0][:48]] += e.device_time_total / 1000.0
    return float(np.median(times)), rows, nbytes, {k: round(v, 3) for k, v in sorted(kernels.items(), key=lambda kv: -kv[1])[:6]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=150_000_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=42)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    ctx = ops.Context(0)
    g = torch.Generator(device=dev).manual_seed(args.seed)
    rng = np.random.default_rng(args.seed)
    name, power = card()
    n = args.rows
    page_rows = 1 << 24
    bounds = [(b, min(n, b + page_rows)) for b in range(0, n, page_rows)]

    def report(tag, ms, rows, nbytes, kernels, bytes_per_row, want_rows, want_bytes):
        assert rows == want_rows, f"{tag}: {rows} rows, the reference says {want_rows}"
        assert nbytes == want_bytes, f"{tag}: {nbytes} output bytes, the reference says {want_bytes}"
        r = {"workload": tag, "median_ms": round(ms, 3), "rows_per_s": n / (ms * 1e-3), "bytes_per_row": round(bytes_per_row, 2),
             "fraction_of_3.35TBps": round(n * bytes_per_row / (ms * 1e-3) / PEAK, 3), "rows_out": rows, "bytes_out": nbytes,
             "kernels_ms": kernels, "card": name, "power_limit": power}
        print(json.dumps(r), flush=True)

    # ---- (a) customer: c_phone, c_acctbal
    phone_pool = [f"{c}-{a}-{b}-{d}".encode() for c, a, b, d in zip(rng.integers(10, 35, 8192), rng.integers(100, 1000, 8192),
                                                                     rng.integers(100, 1000, 8192), rng.integers(1000, 10000, 8192))]
    pid = torch.randint(0, len(phone_pool), (n,), generator=g, device=dev)
    pcount = torch.bincount(pid, minlength=len(phone_pool)).tolist()
    ppages = utf8_pages(phone_pool, pid, dev)
    bal = torch.randint(-99999, 999999, (n,), generator=g, device=dev, dtype=torch.int64)
    pages = [ops.DevicePage([col_utf8(ppages[k]), col_fixed(bal[b:e], abi.INT64)], e - b) for k, (b, e) in enumerate(bounds)]
    key = ops.Call(abi.EX_SUBSTR, ops.Col(0, S), ops.Const(1, B), ops.Const(2, B))
    prog = ops.PageProcessorProgram(ops.Call(abi.EX_IN, key, in_list=Q22_CODES), [key, 1])
    hit = [c for c, s in zip(pcount, phone_pool) if sref.substring(s, 1, 2).decode() in Q22_CODES]
    want = sum(hit)
    pbytes = sum(int(p[0][-1]) for p in ppages) / n
    ms, rows, nb, k = run(ctx, prog, pages, args.steps, args.warmup)
    sel = want / n
    # filter: offsets + phone bytes read, flags; projection: selected rows' phone re-read + key descriptors + acctbal in/out + key out
    report("a_q22_substr_in", ms, rows, nb, k, 4 + pbytes + 2 + sel * (4 + pbytes + 8 + 16 + 8 + 1 + 4 + 2 + 8), want, 2 * want)
    del pages, ppages, bal, pid
    torch.cuda.empty_cache()

    # ---- orders: o_comment, o_orderpriority, o_clerk
    pool = comment_pool(args.seed)
    cid = torch.randint(0, len(pool), (n,), generator=g, device=dev)
    ccount = torch.bincount(cid, minlength=len(pool)).tolist()
    cpages = utf8_pages(pool, cid, dev)
    clerks = [b"Clerk#%09d" % i for i in range(1, 1001)]
    kid = torch.randint(0, len(clerks), (n,), generator=g, device=dev)
    kcount = torch.bincount(kid, minlength=len(clerks)).tolist()
    qid = torch.randint(0, len(PRIORITIES), (n,), generator=g, device=dev)
    qcount = torch.bincount(qid, minlength=len(PRIORITIES)).tolist()
    kpages, qpages = utf8_pages(clerks, kid, dev), utf8_pages(PRIORITIES, qid, dev)
    pages = [ops.DevicePage([col_utf8(cpages[i]), col_utf8(qpages[i]), col_utf8(kpages[i])], e - b) for i, (b, e) in enumerate(bounds)]
    cb = sum(c * len(s) for c, s in zip(ccount, pool)) / n
    C0 = ops.Col(0, S)

    out_b = sum(c * len(sref.substring(s, 1, 20)) for c, s in zip(ccount, pool))
    prog = ops.PageProcessorProgram(None, [ops.Call(abi.EX_SUBSTR, C0, ops.Const(1, B), ops.Const(20, B))])
    ms, rows, nb, k = run(ctx, prog, pages, args.steps, args.warmup)
    # offsets + the first <= 20 bytes of each comment read (sequential), descriptors written and read, offsets + bytes written
    report("b_substr_20", ms, rows, nb, k, 4 + out_b / n + 8 + 1 + 8 + 8 + 8 + 4 + out_b / n, n, out_b)

    keep = [40 <= sref.length(s) <= 60 for s in pool]
    want = sum(c for c, kp in zip(ccount, keep) if kp)
    out_c = sum(c * len(sref.trim(s)) for c, s, kp in zip(ccount, pool, keep) if kp)
    out_p = sum(c * len(s) for c, s, kp in zip(ccount, pool, keep) if kp)
    filt = ops.Call(abi.EX_BETWEEN, ops.Call(abi.EX_LENGTH, C0), ops.Const(40, B), ops.Const(60, B))
    sel = want / n
    # filter: offsets + bytes read, flags; output rows: offsets + bytes read again, descriptors (or positions) written and read, offsets +
    # bytes written
    for tag, proj, out in (("c_trim_length_between", ops.Call(abi.EX_TRIM, C0), out_c), ("c_passthrough_gather", 0, out_p)):
        prog = ops.PageProcessorProgram(filt, [proj])
        ms, rows, nb, k = run(ctx, prog, pages, args.steps, args.warmup)
        report(tag, ms, rows, nb, k, 4 + cb + 1 + sel * (4 + 8 + 1 + 8 + 8 + 8 + 4) + (out_p + out) / n, want, out)

    out_d = n * 1 + sum(c * len(s) for c, s in zip(qcount, PRIORITIES)) + sum(c * len(s) for c, s in zip(kcount, clerks))
    prog = ops.PageProcessorProgram(None, [ops.concat(ops.Col(1, S), ops.Const("-", S), ops.Col(2, S))])
    ms, rows, nb, k = run(ctx, prog, pages, args.steps, args.warmup)
    # both columns' offsets and bytes read, three descriptors written and read, offsets + bytes written
    report("d_concat_priority_clerk", ms, rows, nb, k, 8 + 2 * out_d / n + 24 + 1 + 24 + 8 + 8 + 4, n, out_d)
    ctx.close()


if __name__ == "__main__":
    main()
