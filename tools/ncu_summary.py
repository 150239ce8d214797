#!/usr/bin/env python
"""Turn `.ncu-rep` captures into markdown tables (reads them with `ncu -i … --page raw --csv`).
usage: tools/ncu_summary.py <rep> [<rep> …]   -> markdown on stdout"""
import csv
import io
import subprocess
import sys

METRICS = [
    ("kernel duration", "gpu__time_duration.sum"),
    ("grid", "launch__grid_size"),
    ("block", "launch__block_size"),
    ("registers/thread", "launch__registers_per_thread"),
    ("static smem/block", "launch__shared_mem_per_block_static"),
    ("dynamic smem/block", "launch__shared_mem_per_block_dynamic"),
    ("CTAs/SM limit: registers", "launch__occupancy_limit_registers"),
    ("CTAs/SM limit: shared memory", "launch__occupancy_limit_shared_mem"),
    ("waves per SM", "launch__waves_per_multiprocessor"),
    ("achieved occupancy (% of max warps)", "sm__warps_active.avg.pct_of_peak_sustained_active"),
    ("DRAM bytes read", "dram__bytes_read.sum"),
    ("DRAM bytes written", "dram__bytes_write.sum"),
    ("DRAM throughput (% of peak)", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed"),
    ("L2 sector hit rate", "lts__t_sector_hit_rate.pct"),
    ("L1 sector hit rate", "l1tex__t_sector_hit_rate.pct"),
    ("warp instructions executed", "smsp__inst_executed.sum"),
    ("SM throughput (% of peak)", "sm__throughput.avg.pct_of_peak_sustained_elapsed"),
    ("issue slots busy", "smsp__issue_active.avg.pct_of_peak_sustained_active"),
    ("stall: long scoreboard (warps per issue)", "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio"),
    ("stall: short scoreboard", "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio"),
    ("stall: barrier", "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio"),
    ("stall: LG throttle", "smsp__average_warps_issue_stalled_lg_throttle_per_issue_active.ratio"),
    ("stall: MIO throttle", "smsp__average_warps_issue_stalled_mio_throttle_per_issue_active.ratio"),
    ("stall: wait", "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio"),
    ("smem bank conflicts", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum"),
    ("tensor pipe active", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active"),
]


def summarise(rep):
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    header, units = rows[0], rows[1]
    out = []
    for r in rows[2:]:
        rec = dict(zip(header, r))
        unit = dict(zip(header, units))
        out.append("### `%s`\n\ncapture: `%s`\n\n| metric | value |\n|---|---|" % (rec.get("Kernel Name", "?"), rep))
        for label, m in METRICS:
            if m in rec:
                out.append("| %s (`%s`) | %s %s |" % (label, m, rec[m], unit.get(m, "")))
        try:
            rd, wr = float(rec["dram__bytes_read.sum"]), float(rec["dram__bytes_write.sum"])
            scale = {"Gbyte": 1e9, "Mbyte": 1e6, "Kbyte": 1e3, "byte": 1.0}
            tb = rd * scale.get(unit["dram__bytes_read.sum"], 1.0) + wr * scale.get(unit["dram__bytes_write.sum"], 1.0)
            dur = float(rec["gpu__time_duration.sum"]) * {"ms": 1e-3, "us": 1e-6, "ns": 1e-9, "s": 1.0}.get(unit["gpu__time_duration.sum"], 1e-9)
            out.append("\nDRAM traffic per launch: **%.3f GB**; %.0f GB/s under the profiler (cold caches, serialised)." % (tb / 1e9, tb / 1e9 / dur))
        except (KeyError, ValueError):
            pass
        out.append("")
    return "\n".join(out)


if __name__ == "__main__":
    for rep in sys.argv[1:]:
        print(summarise(rep))
