"""LookupJoinOperator with a join filter function over device-resident synthetic TPC-H lineitem / orders keys.  Prints one JSON line.

    python tools/bench_join_filter.py [--sf 100] [--sf-dup 25] [--steps 3] [--warmup 1] [--page-rows 16777216]

Two shapes, each timed against the same join without the filter on the general probe path (TGPU_JOIN_GENERAL_PATH=1 is set for the
whole run; a filtered lookup never takes the fused path), alternating filtered / unfiltered steps:
  (a) unique build: orders (o_orderkey, o_orderdate) probed by lineitem (l_orderkey, l_shipdate), INNER, filter
      l_shipdate - o_orderdate BETWEEN 0 AND 121 - no position links, one filter evaluation per matched probe row;
  (b) duplicate build: lineitem (l_orderkey, l_shipdate), about 4 rows per key, probed by orders (o_orderkey, o_orderdate), INNER,
      filter o_orderdate + 90 < l_shipdate - position links: candidate pairs, one evaluation per pair.  SF25 by default: the filtered
      and the unfiltered lookup over the same build side are held at once, and two over SF100 lineitem do not fit 80 GB.
Keys come from the library's synthetic generators; the dates are drawn on the device by torch from a fixed seed.  A step probes the
whole probe side in pages of --page-rows rows and drains every output page on the device.  The output row count of the filtered join
is checked against a count computed with torch (sort + searchsorted) on the same device columns.

Byte model (a lower bound of the traffic, stated per row): each probe row reads its key (8 B), one 16-byte table slot and its filter
column (4 B) and writes / reads back its join position (4 + 4 B); each candidate reads the build filter column (4 B) and each output row
writes a probe and a build output column (8 + 4 B) and their two gather indices (4 + 4 B).  `hbm_frac` is that volume over the step time
divided by the H100 SXM5 data-sheet bandwidth, 3.35 TB/s."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

os.environ["TGPU_JOIN_GENERAL_PATH"] = "1"
HBM_BPS = 3.35e12
SEED_ORDERS, SEED_LINEITEM, SEED_DATES = 0x7C02, 0x7C01, 0x7C0D


def device_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    if r.returncode != 0 or "," not in r.stdout:
        return "?", "?"
    name, power = [x.strip() for x in r.stdout.strip().split(",")[:2]]
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sf", type=float, default=100, help="scale factor of shape (a)")
    # two lookups over one build side live at once (filtered and unfiltered); at SF100 a 600 M-row lineitem build twice does not fit 80 GB
    ap.add_argument("--sf-dup", type=float, default=25, help="scale factor of shape (b)")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--page-rows", type=int, default=1 << 24)
    args = ap.parse_args()
    import torch

    from trino_b200 import abi
    from trino_b200 import operators as ops

    ctx = ops.Context(0)
    lib = ctx.lib
    gen = torch.Generator(device="cuda:0")
    gen.manual_seed(SEED_DATES)
    B = abi.V_BIGINT

    def tables(sf):
        n_orders = int(1_500_000 * sf)
        n_lines = lib.tgpu_synth_lineitem_rows(n_orders)
        okeys = torch.empty(n_orders, dtype=torch.int64, device="cuda:0")
        lkeys = torch.empty(n_lines, dtype=torch.int64, device="cuda:0")
        ctx.check(lib.tgpu_synth_orders_keys(ctx.h, n_orders, 0, n_orders, SEED_ORDERS, 1, C.c_void_p(okeys.data_ptr())))
        ctx.check(lib.tgpu_synth_lineitem_keys(ctx.h, n_orders, 0, n_lines, SEED_LINEITEM, 0, C.c_void_p(lkeys.data_ptr())))
        ctx.synchronize()
        odate = torch.randint(0, 2406, (n_orders,), dtype=torch.int32, device="cuda:0", generator=gen)
        lship = torch.randint(0, 2527, (n_lines,), dtype=torch.int32, device="cuda:0", generator=gen)
        torch.cuda.synchronize()
        return okeys, odate, lkeys, lship

    def dpage(key, val, first=0, count=None):
        count = key.numel() - first if count is None else count
        return ops.DevicePage([ops.DeviceColumn(abi.INT64, key.data_ptr() + first * 8, count),
                               ops.DeviceColumn(abi.INT32, val.data_ptr() + first * 4, count)], count)

    def torch_count(bkey, bval, pkey, pval, pred, unique_side):
        """output rows of the filtered INNER join: for every (build row, probe row) with equal keys, pred(build value, probe value).
        unique_side: the side whose keys are unique ("build" or "probe"); the other side's rows each meet at most one row"""
        if unique_side == "probe":
            order = torch.argsort(pkey)
            sk = pkey[order]
            at = torch.searchsorted(sk, bkey).clamp(max=sk.numel() - 1)
            hit = sk[at] == bkey
            return int((hit & pred(bval, pval[order][at])).sum())
        order = torch.argsort(bkey)
        sk = bkey[order]
        at = torch.searchsorted(sk, pkey).clamp(max=sk.numel() - 1)
        hit = sk[at] == pkey
        return int((hit & pred(bval[order][at], pval)).sum())

    def run_shape(name, bkey, bval, pkey, pval, filt, pred, unique_side, sf):
        nb = 2
        build_page = dpage(bkey, bval)
        n_probe = pkey.numel()
        pages = [dpage(pkey, pval, f, min(args.page_rows, n_probe - f)) for f in range(0, n_probe, args.page_rows)]
        lookups = {}
        for label, f in (("filtered", filt), ("unfiltered", None)):
            bridge = ops.JoinBridge()
            b = ops.HashBuilderOperatorFactory(ctx, bridge, [0], [1], bkey.numel(), filter=f, num_build_channels=nb).create_operator()
            b.add_input(build_page)
            b.finish()
            ctx.synchronize()
            lookups[label] = (bridge, b)
        has_links = lookups["filtered"][0].lookup_source.has_position_links()

        def step(label):
            bridge = lookups[label][0]
            op = ops.LookupJoinOperatorFactory(ctx, bridge, abi.JOIN_INNER, False, [0], [0]).create_operator()
            rows = 0
            for pg in pages:
                op.add_input(pg)
                while True:
                    out = op.get_output_device()
                    if out is None:
                        break
                    rows += out.rows
                    out.release()
            op.finish()
            op.close()
            return rows

        for _ in range(args.warmup):
            step("filtered")
            step("unfiltered")
        times = {"filtered": [], "unfiltered": []}
        rows = {}
        for _ in range(args.steps):
            for label in ("filtered", "unfiltered"):
                ctx.synchronize()
                ctx.timer_start()
                rows[label] = step(label)
                times[label].append(ctx.timer_stop_ms())
        want = torch_count(bkey, bval, pkey, pval, pred, unique_side)
        assert rows["filtered"] == want, (name, rows["filtered"], want)
        candidates = rows["unfiltered"]
        ms = sorted(times["filtered"])[len(times["filtered"]) // 2]
        ms_plain = sorted(times["unfiltered"])[len(times["unfiltered"]) // 2]
        model_bytes = n_probe * (8 + 16 + 4 + 8) + candidates * 4 + rows["filtered"] * (12 + 8)
        for bridge, b in lookups.values():
            b.close()
            bridge.lookup_source.close()
        return {
            "shape": name, "sf": sf, "build_rows": bkey.numel(), "probe_rows": n_probe, "position_links": has_links,
            "candidates": candidates, "output_rows": rows["filtered"], "torch_count": want, "count_check": "ok",
            "step_ms": ms, "probe_rows_per_sec": n_probe / (ms * 1e-3), "step_ms_all": times["filtered"],
            "unfiltered_general_path_step_ms": ms_plain, "unfiltered_step_ms_all": times["unfiltered"],
            "filter_over_unfiltered": ms / ms_plain,
            "model_bytes": model_bytes, "hbm_frac": model_bytes / (ms * 1e-3) / HBM_BPS,
        }

    results = []
    okeys, odate, lkeys, lship = tables(args.sf)
    # (a) probe lineitem channels (2, 3) = (l_orderkey, l_shipdate); build (0, 1) = (o_orderkey, o_orderdate)
    filt_a = ops.Call(abi.EX_BETWEEN, ops.Call(abi.EX_SUB, ops.Col(3, B), ops.Col(1, B)), ops.Const(0, B), ops.Const(121, B))
    results.append(run_shape("a: unique build, l_shipdate - o_orderdate BETWEEN 0 AND 121", okeys, odate, lkeys, lship, filt_a,
                             lambda b, p: ((p - b) >= 0) & ((p - b) <= 121), "build", args.sf))
    if args.sf_dup != args.sf:
        del okeys, odate, lkeys, lship
        torch.cuda.empty_cache()
        okeys, odate, lkeys, lship = tables(args.sf_dup)
    # (b) build lineitem (0, 1) = (l_orderkey, l_shipdate); probe orders (2, 3) = (o_orderkey, o_orderdate)
    filt_b = ops.Call(abi.EX_LT, ops.Call(abi.EX_ADD, ops.Col(3, B), ops.Const(90, B)), ops.Col(1, B))
    results.append(run_shape("b: duplicate build, o_orderdate + 90 < l_shipdate", lkeys, lship, okeys, odate, filt_b,
                             lambda b, p: (p + 90) < b, "probe", args.sf_dup))
    name, power = device_info()
    print(json.dumps({"metric": "join_filter_probe_rows_per_sec", "device": name, "power_limit": power, "page_rows": args.page_rows,
                      "steps": args.steps, "hbm_bytes_per_sec": HBM_BPS, "shapes": results}))
    ctx.close()


if __name__ == "__main__":
    main()
