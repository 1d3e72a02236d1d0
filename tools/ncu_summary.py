"""tools/ncu_summary.py -- condense an .ncu-rep (ncu --set full) into the few numbers DESIGN.md cites.
usage: python tools/ncu_summary.py prof.ncu-rep summary.md"""
import csv
import io
import subprocess
import sys

KEYS = [
    "gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
    "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem", "launch__waves_per_multiprocessor",
    "sm__warps_active.avg.pct_of_peak_sustained_active", "dram__bytes_read.sum", "dram__bytes_write.sum",
    "dram__bytes_read.sum.per_second", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "smsp__inst_executed.sum", "smsp__issue_active.avg.per_cycle_active", "smsp__cycles_active.avg",
    "sm__cycles_elapsed.avg", "sm__cycles_elapsed.avg.per_second",
    "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active",
    "sm__pipe_fmaheavy_cycles_active.avg.pct_of_peak_sustained_elapsed",
    "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_tma.avg.pct_of_peak_sustained_active",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "smsp__warps_eligible.avg.per_cycle_active",
    "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_dispatch_stall_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_no_instruction_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
    "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
]


def main():
    rep, out = sys.argv[1], sys.argv[2]
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units = rows[0], rows[1]
    lines = [f"# ncu summary of `{rep.split('/')[-1]}`\n", "Captured with `ncu --set full --clock-control none --import-source on` (see the command in DESIGN.md).\n"]
    for r in rows[2:]:
        d = dict(zip(hdr, r))
        lines.append(f"\n## {d.get('Kernel Name', '?')}  (grid {d.get('Grid Size')}, block {d.get('Block Size')})\n")
        lines.append("| metric | value | unit |\n|---|---|---|")
        for k in KEYS:
            if k in d:
                lines.append(f"| `{k}` | {d[k]} | {units[hdr.index(k)]} |")
    open(out, "w").write("\n".join(lines) + "\n")
    print("wrote", out)


if __name__ == "__main__":
    main()
