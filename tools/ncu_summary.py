#!/usr/bin/env python
"""Summarise an .ncu-rep (read with `ncu -i ... --page raw --csv`) into the handful of numbers the
roofline discussion needs.  Usage: python tools/ncu_summary.py prof.ncu-rep"""
import csv
import subprocess
import sys

KEYS = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram__bytes_read.sum.per_second",
    "lts__t_sector_hit_rate.pct", "lts__t_sectors_srcunit_tex.sum", "lts__t_sectors_srcunit_tex.avg.pct_of_peak_sustained_elapsed",
    "lts__throughput.avg.pct_of_peak_sustained_elapsed", "l1tex__throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__pipe_tensor_cycles_active_realtime.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__inst_executed_pipe_fma.sum", "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active",
    "sm__pipe_fmaheavy_cycles_active.avg.pct_of_peak_sustained_active", "sm__inst_executed.avg.per_cycle_elapsed",
    "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread", "launch__grid_size",
    "launch__block_size", "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem",
    "smsp__warp_issue_stalled_long_scoreboard_per_warp_active.pct", "smsp__warp_issue_stalled_lg_throttle_per_warp_active.pct",
    "smsp__warp_issue_stalled_math_pipe_throttle_per_warp_active.pct", "smsp__warp_issue_stalled_short_scoreboard_per_warp_active.pct",
    "smsp__warp_issue_stalled_barrier_per_warp_active.pct", "smsp__warp_issue_stalled_mio_throttle_per_warp_active.pct",
    "smsp__warp_issue_stalled_wait_per_warp_active.pct", "smsp__issue_active.avg.pct_of_peak_sustained_active",
    "sm__cycles_elapsed.avg", "sm__cycles_active.avg",
]


def main(path):
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    hdr, units = rows[0], rows[1]
    for r in rows[2:]:
        name = r[hdr.index("Kernel Name")] if "Kernel Name" in hdr else "?"
        print(f"# kernel: {name}")
        for h, u, v in zip(hdr, units, r):
            short = h.split("TriageCompute.")[-1]
            if short in KEYS or h in KEYS:
                print(f"{short:90s} {v} {u}")


if __name__ == "__main__":
    main(sys.argv[1])
