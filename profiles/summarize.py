#!/usr/bin/env python
"""Summarise an .ncu-rep (ncu need not run on a GPU machine to read it) into a small text file.
usage: python profiles/summarize.py x.ncu-rep x.summary.txt"""
import csv
import io
import subprocess
import sys

KEYS = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "dram__throughput.avg.pct_of_peak_sustained_elapsed",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "l1tex__throughput.avg.pct_of_peak_sustained_active", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
    "launch__grid_size", "launch__block_size", "launch__registers_per_thread", "launch__shared_mem_per_block_dynamic",
    "launch__shared_mem_per_block_static", "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem",
    "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__issue_active.avg.pct_of_peak_sustained_active",
    "smsp__inst_executed.sum", "l1tex__t_sectors_pipe_lsu_mem_global_op_ld.sum", "l1tex__t_sectors_pipe_lsu_mem_global_op_st.sum",
    "l1tex__t_sectors_pipe_lsu_mem_global_op_red.sum", "l1tex__t_sectors_pipe_lsu_mem_global_op_atom.sum",
    "lts__t_sectors_op_red.sum", "lts__t_sectors_op_atom.sum", "lts__t_sectors_op_read.sum", "lts__t_sectors_op_write.sum",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
]
STALL = "smsp__average_warps_issue_stalled_"


def main():
    rep, out = sys.argv[1], sys.argv[2]
    txt = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(txt)))
    hdr, units = rows[0], rows[1]
    lines = ["# summary of %s (ncu --set full --clock-control none)" % rep]
    for r in rows[2:]:
        d = dict(zip(hdr, r))
        lines.append("## kernel: %s  grid=%s block=%s" % (d.get("Kernel Name"), d.get("Grid Size"), d.get("Block Size")))
        for i, h in enumerate(hdr):
            if h in KEYS:
                lines.append("%-70s %-16s %s" % (h, units[i], r[i]))
        st = [(float(r[i]), h[len(STALL):].replace("_per_issue_active.ratio", "")) for i, h in enumerate(hdr)
              if h.startswith(STALL) and h.endswith("_per_issue_active.ratio") and r[i] not in ("", "n/a")]
        lines.append("stall reasons (warps per issue-active cycle): " + ", ".join("%s=%.2f" % (n, v) for v, n in sorted(st, reverse=True)[:8]))
    open(out, "w").write("\n".join(lines) + "\n")
    print("\n".join(lines))


if __name__ == "__main__":
    main()
