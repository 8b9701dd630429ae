#!/usr/bin/env python
"""Summarise one kernel of an .ncu-rep into JSON.

usage: ncu_summary.py <report.ncu-rep> <kernel-name-substring> <note> > <name>_summary.json
Reads `ncu -i … --page raw --csv`; keeps the time, DRAM, instruction and pipe metrics of the kernel.
"""
import csv, io, json, subprocess, sys

KEEP = (
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "smsp__inst_executed.sum",
    "smsp__inst_executed.avg.per_cycle_active", "sm__warps_active.avg.pct_of_peak_sustained_active",
    "launch__grid_size", "launch__block_size", "launch__registers_per_thread", "launch__shared_mem_per_block_dynamic",
    "launch__occupancy_limit_blocks", "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem",
    "launch__occupancy_limit_warps", "lts__t_sector_hit_rate.pct", "l1tex__t_sector_hit_rate.pct",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed", "gpu__compute_memory_throughput.avg.pct_of_peak_sustained_elapsed",
    "dram__throughput.avg.pct_of_peak_sustained_elapsed",
    "smsp__thread_inst_executed_per_inst_executed.ratio",
)
STALL = "smsp__average_warps_issue_stalled_"


def main():
    rep, kern, note = sys.argv[1], sys.argv[2], sys.argv[3]
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    head, units = rows[0], rows[1]
    ki = head.index("Kernel Name")
    for r in rows[2:]:
        if kern in r[ki]:
            break
    else:
        sys.exit("kernel not in report")
    m = {}
    for h, u, v in zip(head, units, r):
        if h in KEEP or (h.startswith(STALL) and h.endswith("_per_warp_active.pct") is False and h.endswith(".ratio")):
            m[h] = [v, u]
    json.dump({"report": rep.split("/")[-1], "kernel": r[ki], "note": note, "metrics": m}, sys.stdout, indent=1)
    print()


if __name__ == "__main__":
    main()
