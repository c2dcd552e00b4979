#!/usr/bin/env python
"""Summarise `ncu --set full` reports into a small CSV:  python tools/ncu_summary.py out.csv rep1.ncu-rep rep2.ncu-rep ...
One row per (report, metric) for the metrics the roofline discussion uses."""
import csv
import subprocess
import sys

WANT = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "dram__throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed", "smsp__issue_active.avg.pct", "smsp__inst_executed.sum",
        "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
        "launch__shared_mem_per_block_dynamic", "launch__shared_mem_per_block_static", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
        "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio", "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio", "smsp__average_warps_issue_stalled_mio_throttle_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio", "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio", "smsp__average_warps_issue_stalled_branch_resolving_per_issue_active.ratio"]


def main():
    out = sys.argv[1]
    rows = [["report", "kernel", "metric", "unit", "value"]]
    for rep in sys.argv[2:]:
        txt = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
        r = list(csv.reader(txt.splitlines()))
        if len(r) < 3:
            continue
        hdr, units, vals = r[0], r[1], r[2]
        kname = vals[hdr.index("Kernel Name")] if "Kernel Name" in hdr else "?"
        for w in WANT:
            if w in hdr:
                i = hdr.index(w)
                rows.append([rep.split("/")[-1], kname[:90], w, units[i], vals[i]])
    with open(out, "w", newline="") as f:
        csv.writer(f).writerows(rows)
    print("wrote", out, len(rows) - 1, "rows")


if __name__ == "__main__":
    main()
