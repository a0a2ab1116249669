#!/usr/bin/env python
"""Turn an .ncu-rep (ncu --set full) into the transposed per-kernel CSV.

usage: tools/ncu_summary.py <capture>.ncu-rep <tag>_ncu_frame_kernels.csv [--first]
One column per captured launch (or, with --first, the first launch of each kernel name), one row per metric of
interest.  Also prints dram bytes per launch of every kernel."""
import csv
import io
import subprocess
import sys

KEEP = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
    "dram__throughput.avg.pct_of_peak_sustained_elapsed", "lts__t_sector_hit_rate.pct", "l1tex__t_sector_hit_rate.pct",
    "lts__t_sectors_op_red.sum", "lts__t_sectors_op_atom.sum", "lts__t_bytes.sum",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed", "smsp__issue_active.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active",
    "smsp__inst_executed.sum", "smsp__thread_inst_executed_per_inst_executed.ratio",
    "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread", "launch__occupancy_limit_registers",
    "launch__occupancy_limit_shared_mem", "launch__grid_size", "launch__block_size", "launch__shared_mem_per_block_dynamic",
    "launch__shared_mem_per_block_static", "smsp__warp_issue_stalled_long_scoreboard_per_warp_active.pct",
    "smsp__warp_issue_stalled_short_scoreboard_per_warp_active.pct", "smsp__warp_issue_stalled_wait_per_warp_active.pct",
    "smsp__warp_issue_stalled_barrier_per_warp_active.pct", "smsp__warp_issue_stalled_math_pipe_throttle_per_warp_active.pct",
    "smsp__warp_issue_stalled_lg_throttle_per_warp_active.pct", "smsp__warp_issue_stalled_not_selected_per_warp_active.pct",
    "smsp__warp_issue_stalled_branch_resolving_per_warp_active.pct", "smsp__warp_issue_stalled_dispatch_stall_per_warp_active.pct",
    "smsp__warp_issue_stalled_mio_throttle_per_warp_active.pct", "smsp__warp_issue_stalled_no_instruction_per_warp_active.pct",
    "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "smsp__inst_executed_op_shared_ld.sum",
]


def main():
    rep, out = sys.argv[1], sys.argv[2]
    first = "--first" in sys.argv
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units, data = rows[0], rows[1], rows[2:]
    ki = hdr.index("Kernel Name")
    cols, seen = [], set()
    for r in data:
        name = r[ki].split("(")[0]
        if first and name in seen:
            continue
        seen.add(name)
        cols.append(r)
    with open(out, "w") as f:
        f.write("# ncu --set full --clock-control none --import-source on; numbers under ncu are not bench values\n")
        f.write("# raw report: %s (not committed)\n" % rep)
        w = csv.writer(f)
        w.writerow(["metric", "unit"] + [r[ki].split("(")[0] for r in cols])
        for m in KEEP:
            if m in hdr:
                j = hdr.index(m)
                w.writerow([m, units[j]] + [r[j] for r in cols])
    jr, jw = hdr.index("dram__bytes_read.sum"), hdr.index("dram__bytes_write.sum")
    for r in cols:
        def tobytes(v, u):
            v = float(v.replace(",", ""))
            return v * {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(u, 1)
        print(r[ki].split("(")[0], "dram bytes/launch =", tobytes(r[jr], units[jr]) + tobytes(r[jw], units[jw]))


if __name__ == "__main__":
    main()
