"""VARCHAR predicates in FilterAndProject over device-resident pages at SF100 scale.

  (a) 600 M lineitem rows, the 7 TPC-H ship modes:            l_shipmode IN ('MAIL', 'SHIP'), projecting l_orderkey
  (b) 600 M lineitem rows, ship modes x 4 ship instructions:  l_shipmode IN ('AIR', 'AIR REG') AND l_shipinstruct = 'DELIVER IN PERSON'
  (c) 150 M orders rows, o_comment of 19-78 bytes:            o_comment NOT LIKE '%special%requests%'   (FJS middle)
  (d) the same o_comment column:                              o_comment NOT LIKE '%special%re_uests%'   (`_` after `%`: the NFA)
For (a) and (b) the same filter over INT8 code columns through the numeric IN / = is timed alternately in the same run.

Strings are gathered on the device from seeded pools, so the expected row counts are exact: each pool entry's verdict comes from the
Python reference (tests/like_reference.py) and is weighted by how often the entry was drawn.  Pages hold 2^24 rows (int32 offsets).
Reports, per workload: the median step time (CUDA events, after warm-up), rows/s, the byte model (4 B offsets + string bytes + fixed-width
bytes read + bytes written, per row) and its fraction of 3.35 TB/s, with the card name and power limit read in the same run.

  python tools/bench_varchar_filter.py [--rows 600000000] [--steps 5] [--warmup 2]
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

import like_reference as lr                      # noqa: E402
from trino_b200 import abi                       # noqa: E402
from trino_b200 import operators as ops          # noqa: E402

PAGE_ROWS = 1 << 24
PEAK = 3.35e12
SHIPMODES = [b"REG AIR", b"AIR", b"RAIL", b"SHIP", b"TRUCK", b"MAIL", b"FOB"]
INSTRUCTIONS = [b"DELIVER IN PERSON", b"COLLECT COD", b"NONE", b"TAKE BACK RETURN"]
S, B = abi.V_VARCHAR, abi.V_BIGINT


def comment_pool(seed, size=4096, special_fraction=0.1):
    rng = np.random.default_rng(seed)
    words = [b"furiously", b"quickly", b"carefully", b"final", b"pending", b"deposits", b"accounts", b"packages", b"ideas", b"slyly",
             b"regular", b"express", b"blithely", b"ironic", b"bold", b"even", b"haggle", b"sleep", b"wake", b"among"]
    pool = []
    for i in range(size):
        target = int(rng.integers(19, 79))
        parts = []
        if rng.random() < special_fraction:
            parts = [b"special", words[int(rng.integers(len(words)))], b"requests"]
        while len(b" ".join(parts)) < target:
            parts.insert(int(rng.integers(len(parts) + 1)), words[int(rng.integers(len(words)))])
        pool.append(b" ".join(parts)[:target].ljust(19, b"x"))
    return pool


def utf8_pages(pool, ids, dev):
    """device UTF8 columns (one per page) of pool[ids]: (offsets, bytes, rows) per page, gathered on the device"""
    flat = torch.tensor(np.frombuffer(b"".join(pool), np.uint8).copy(), device=dev)
    lens = torch.tensor([len(p) for p in pool], device=dev, dtype=torch.int64)
    starts = torch.cumsum(lens, 0) - lens
    pages = []
    for b in range(0, ids.numel(), PAGE_ROWS):
        pid = ids[b:b + PAGE_ROWS]
        ln = lens[pid]
        off = torch.zeros(pid.numel() + 1, dtype=torch.int64, device=dev)
        torch.cumsum(ln, 0, out=off[1:])
        total = int(off[-1])
        row = torch.repeat_interleave(torch.arange(pid.numel(), device=dev), ln, output_size=total)
        within = torch.arange(total, device=dev) - off[:-1][row]
        data = flat[starts[pid][row] + within].contiguous()
        pages.append((off.to(torch.int32).contiguous(), data if total else torch.zeros(16, dtype=torch.uint8, device=dev), pid.numel()))
        del row, within
    return pages


def col_utf8(page):
    off, data, n = page
    return ops.DeviceColumn(abi.UTF8, data.data_ptr(), n, None, off.data_ptr())


def col_fixed(t, type_):
    return ops.DeviceColumn(type_, t.data_ptr(), t.numel(), None)


def run(ctx, prog, pages, steps, warmup):
    """median ms of one step (every page through one operator), and the rows it selected"""
    times, rows = [], 0
    for s in range(warmup + steps):
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
        for o in outs:
            o.release()
        op.close()
        if s >= warmup:
            times.append(ms)
    return float(np.median(times)), rows


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=20).stdout
        name, power = [x.strip() for x in q.splitlines()[0].split(",")]
        return name, power
    except Exception:      # noqa: BLE001 - the table still names the card
        return torch.cuda.get_device_name(0), "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=600_000_000)
    ap.add_argument("--orders", type=int, default=150_000_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=42)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    ctx = ops.Context(0)
    g = torch.Generator(device=dev).manual_seed(args.seed)
    name, power = card()
    results = []

    def report(tag, ms, rows, n, bytes_per_row, want):
        assert rows == want, f"{tag}: {rows} rows selected, the reference says {want}"
        gbs = n * bytes_per_row / (ms * 1e-3)
        r = {"workload": tag, "median_ms": round(ms, 3), "rows_per_s": n / (ms * 1e-3), "bytes_per_row": round(bytes_per_row, 2),
             "fraction_of_3.35TBps": round(gbs / PEAK, 3), "selected": rows, "card": name, "power_limit": power}
        results.append(r)
        print(json.dumps(r), flush=True)

    # ---- lineitem: ship mode, ship instruction, orderkey
    n = args.rows
    mode = torch.randint(0, len(SHIPMODES), (n,), generator=g, device=dev)
    instr = torch.randint(0, len(INSTRUCTIONS), (n,), generator=g, device=dev)
    mode_pages, instr_pages = utf8_pages(SHIPMODES, mode, dev), utf8_pages(INSTRUCTIONS, instr, dev)
    orderkey = torch.arange(n, dtype=torch.int64, device=dev)
    mode8, instr8 = mode.to(torch.int8), instr.to(torch.int8)
    mode_count = torch.bincount(mode, minlength=len(SHIPMODES)).tolist()
    pair_count = torch.bincount(mode * 4 + instr, minlength=len(SHIPMODES) * 4).tolist()
    str_pages, code_pages = [], []
    for k, b in enumerate(range(0, n, PAGE_ROWS)):
        e = min(n, b + PAGE_ROWS)
        str_pages.append(ops.DevicePage([col_utf8(mode_pages[k]), col_utf8(instr_pages[k]), col_fixed(orderkey[b:e], abi.INT64)], e - b))
        code_pages.append(ops.DevicePage([col_fixed(mode8[b:e], abi.INT8), col_fixed(instr8[b:e], abi.INT8), col_fixed(orderkey[b:e], abi.INT64)], e - b))
    mode_bytes = sum(int(p[0][-1]) for p in mode_pages) / n
    instr_bytes = sum(int(p[0][-1]) for p in instr_pages) / n

    want_a = mode_count[SHIPMODES.index(b"MAIL")] + mode_count[SHIPMODES.index(b"SHIP")]
    a_str = ops.PageProcessorProgram(ops.Call(abi.EX_IN, ops.Col(0, S), in_list=["MAIL", "SHIP"]), [2])
    a_int = ops.PageProcessorProgram(ops.Call(abi.EX_IN, ops.Col(0, B), in_list=[SHIPMODES.index(b"MAIL"), SHIPMODES.index(b"SHIP")]), [2])
    modes_b = [SHIPMODES.index(b"AIR"), SHIPMODES.index(b"REG AIR")]
    want_b = sum(pair_count[m * 4 + 0] for m in modes_b)
    b_str = ops.PageProcessorProgram(ops.Call(abi.EX_AND, ops.Call(abi.EX_IN, ops.Col(0, S), in_list=["AIR", "REG AIR"]),
                                              ops.Call(abi.EX_EQ, ops.Col(1, S), ops.Const("DELIVER IN PERSON", S))), [2])
    b_int = ops.PageProcessorProgram(ops.Call(abi.EX_AND, ops.Call(abi.EX_IN, ops.Col(0, B), in_list=modes_b),
                                              ops.Call(abi.EX_EQ, ops.Col(1, B), ops.Const(0, B))), [2])
    sel_a, sel_b = want_a / n, want_b / n
    # byte model: filter inputs read once by the filter pass + flags written / read + the selected rows' key read and written
    for rep in range(2):       # alternate the string and the code forms in the same run
        ms, rows = run(ctx, a_str, str_pages, args.steps, args.warmup)
        report(f"a_shipmode_in_varchar#{rep}", ms, rows, n, 4 + mode_bytes + 2 + 16 * sel_a, want_a)
        ms, rows = run(ctx, a_int, code_pages, args.steps, args.warmup)
        report(f"a_shipmode_in_int8#{rep}", ms, rows, n, 1 + 2 + 16 * sel_a, want_a)
        ms, rows = run(ctx, b_str, str_pages, args.steps, args.warmup)
        report(f"b_q19_conjunct_varchar#{rep}", ms, rows, n, 8 + mode_bytes + instr_bytes + 2 + 16 * sel_b, want_b)
        ms, rows = run(ctx, b_int, code_pages, args.steps, args.warmup)
        report(f"b_q19_conjunct_int8#{rep}", ms, rows, n, 2 + 2 + 16 * sel_b, want_b)
    del str_pages, code_pages, mode_pages, instr_pages, orderkey, mode8, instr8, mode, instr
    torch.cuda.empty_cache()

    # ---- orders: o_comment
    m = args.orders
    pool = comment_pool(args.seed)
    cid = torch.randint(0, len(pool), (m,), generator=g, device=dev)
    counts = torch.bincount(cid, minlength=len(pool)).tolist()
    cpages = utf8_pages(pool, cid, dev)
    okey = torch.arange(m, dtype=torch.int64, device=dev)
    pages = [ops.DevicePage([col_utf8(cpages[k]), col_fixed(okey[b:min(m, b + PAGE_ROWS)], abi.INT64)], min(m, b + PAGE_ROWS) - b)
             for k, b in enumerate(range(0, m, PAGE_ROWS))]
    cbytes = sum(int(p[0][-1]) for p in cpages) / m
    for tag, pattern in (("c_not_like_fjs", "%special%requests%"), ("d_not_like_nfa", "%special%re_uests%")):
        matcher = lr.Matcher(pattern)
        want = sum(c for c, s in zip(counts, pool) if not matcher.match(s))
        prog = ops.PageProcessorProgram(ops.Call(abi.EX_NOT, ops.Call(abi.EX_LIKE, ops.Col(0, S), pattern=pattern)), [1])
        ms, rows = run(ctx, prog, pages, args.steps, args.warmup)
        report(f"{tag} ({matcher.kind})", ms, rows, m, 4 + cbytes + 2 + 16 * want / m, want)
    ctx.close()


if __name__ == "__main__":
    main()
