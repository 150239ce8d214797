"""DRAM traffic of the fused join probe on the bench workload, against a device-to-device copy of the same volume.

    python tools/probe_traffic.py [--sf 100] [--reps 10] [--model packed4|packed8|keyed|positions]

Builds the bench's lineitem JOIN orders (BIGINT key, one 8-byte payload column, key-ordered probe page), times one
LookupJoinOperator page with the CUDA events the library records around its kernels (tgpu_ctx_last_kernel_ms), and prints the
bytes the probe moves per page, computed from the shapes:

    packed4   : probe keys 8 B/row + 4-byte packed slots {krel, cell}, each 32-byte table line read once + payload written
                8 B/row + the match bitmap, 1 bit/row (what the bench's build picks)
    packed8   : the same with 8-byte packed slots, 64 bytes per line
    keyed     : the same with 16-byte keyed slots {key, cell}, 128 bytes per line
    positions : probe keys 8 B/row + 16-byte slots {key, head, pad}, each line read once + slot-ordered payload, 64 B per line
                + payload written 8 B/row + the int32 join position of every row, 4 B/row

The table lines a key-ordered page reads are those of the order-preserving layout between the smallest and the largest build
key.  A torch copy_ of (reads + writes) / 2 bytes moves the same volume; the kernel's effective GB/s is reported against the
copy's measured GB/s, not against a data-sheet figure.  Also prints the lookup's device memory (tgpu_lookup_memory_bytes), which
shows the slot width the build picked.  Prints one JSON line.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SEED_LINEITEM, SEED_ORDERS = 0x7C01, 0x7C02      # bench.py's generator seeds
LINE_BYTES = {"packed4": 32, "packed8": 64, "keyed": 128}      # a table line of 8 slots


def table_geometry(rows, kmin, kmax):
    """capacity and line shift of the dense order-preserving layout that the build picks for TPC-H order keys (join.cu build_table)"""
    lf = 0.25 if rows <= (1 << 16) else 0.5 if rows <= (1 << 20) else 0.75
    need = int(rows / lf) + 1
    cap = 8
    while cap < need:
        cap <<= 1
    lines = cap >> 3
    span = kmax - kmin
    shift = 0
    while (span >> shift) >= lines:
        shift += 1
    return cap, shift


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sf", type=float, default=100.0)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--model", default="packed4", choices=list(LINE_BYTES) + ["positions"],
                    help="byte model: the keyed table in 4-, 8- or 16-byte slots + match bitmap, or 16-byte slots + slot-ordered payload + int32 positions")
    args = ap.parse_args()

    import torch
    from trino_b200 import abi
    from trino_b200 import operators as ops

    ctx = ops.Context(0)
    lib = ctx.lib
    n_orders = int(1_500_000 * args.sf)
    n = lib.tgpu_synth_lineitem_rows(n_orders)
    d_okeys = ctx.malloc(n_orders * 8)
    ctx.check(lib.tgpu_synth_orders_keys(ctx.h, n_orders, 0, n_orders, SEED_ORDERS, 1, C.c_void_p(d_okeys)))
    d_lkeys = ctx.malloc(n * 8)
    ctx.check(lib.tgpu_synth_lineitem_keys(ctx.h, n_orders, 0, n, SEED_LINEITEM, 0, C.c_void_p(d_lkeys)))

    def project(ptr, rows, expr):
        op = ops.FilterAndProjectOperatorFactory(ctx, ops.PageProcessorProgram(None, [expr])).create_operator()
        op.add_input(ops.DevicePage([ops.DeviceColumn(abi.INT64, ptr, rows)], rows))
        out = op.get_output_device()
        op.close()
        return out

    price = project(d_lkeys, n, ops.Call(abi.EX_MUL, ops.Call(abi.EX_CAST_BIGINT_TO_DOUBLE, ops.Col(0, abi.V_BIGINT)), ops.Const(0.5, abi.V_DOUBLE)))
    date = project(d_okeys, n_orders, ops.Call(abi.EX_MOD, ops.Col(0, abi.V_BIGINT), ops.Const(2557, abi.V_BIGINT)))
    bridge = ops.JoinBridge()
    builder = ops.HashBuilderOperatorFactory(ctx, bridge, [0], [1], n_orders).create_operator()
    builder.add_input(ops.DevicePage([ops.DeviceColumn(abi.INT64, d_okeys, n_orders), date.column(0)], n_orders))
    builder.finish()
    lookup_bytes = bridge.lookup_source.get_in_memory_size_in_bytes()
    probe_op = ops.LookupJoinOperatorFactory(ctx, bridge, abi.JOIN_INNER, False, [0], [0, 1]).create_operator()
    probe = ops.DevicePage([ops.DeviceColumn(abi.INT64, d_lkeys, n), price.column(0)], n)

    kms = []
    for i in range(2 + args.reps):
        probe_op.add_input(probe)
        if i >= 2:
            kms.append(ctx.last_kernel_ms())
        out = probe_op.get_output_device()
        assert out is not None and out.rows == n
        out.release()
    kernel_ms = min(kms)

    # byte model from the shapes
    host_keys = ctx.to_host(d_okeys, np.int64, n_orders)
    kmin, kmax = int(host_keys.min()), int(host_keys.max())
    cap, shift = table_geometry(n_orders, kmin, kmax)
    lines = ((kmax - kmin) >> shift) + 1
    streams = {"probe_keys": 8 * n}
    if args.model in LINE_BYTES:
        streams["keyed_slots"] = LINE_BYTES[args.model] * lines
        streams["payload_written"] = 8 * n
        streams["match_bitmap"] = (n + 31) // 32 * 4
        reads = streams["probe_keys"] + streams["keyed_slots"]
    else:
        streams["slots"] = 128 * lines
        streams["payload_by_slot"] = 64 * lines
        streams["payload_written"] = 8 * n
        streams["positions"] = 4 * n
        reads = streams["probe_keys"] + streams["slots"] + streams["payload_by_slot"]
    total = sum(streams.values())
    writes = total - reads

    # copy yardstick: reads and writes the same volume
    half = total // 2 // 8
    src = torch.empty(half, dtype=torch.int64, device="cuda:0").fill_(1)
    dst = torch.empty_like(src)
    for _ in range(3):
        dst.copy_(src)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    cms = []
    for _ in range(args.reps):
        ev0.record()
        dst.copy_(src)
        ev1.record()
        ev1.synchronize()
        cms.append(ev0.elapsed_time(ev1))
    copy_ms = min(cms)
    copy_gbs = 2 * half * 8 / (copy_ms * 1e-3) / 1e9
    kernel_gbs = total / (kernel_ms * 1e-3) / 1e9
    print(json.dumps({"tool": "probe_traffic", "gpu": gpu_info(), "model": args.model, "sf": args.sf, "probe_rows": n, "build_rows": n_orders,
                      "table_capacity": cap, "table_lines_read": lines,
                      "lookup_memory_bytes": lookup_bytes, "bytes": streams, "bytes_total": total, "bytes_read": reads,
                      "bytes_written": writes, "kernel_ms_min": kernel_ms, "kernel_ms_all": kms, "kernel_gb_per_s": kernel_gbs,
                      "copy_ms_min": copy_ms, "copy_gb_per_s": copy_gbs, "kernel_over_copy": kernel_gbs / copy_gbs,
                      "rows_per_s": n / (kernel_ms * 1e-3)}))
    probe_op.close()
    builder.close()
    bridge.lookup_source.close()
    ctx.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
