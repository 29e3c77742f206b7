#!/usr/bin/env python3
"""Summarise an .ncu-rep (ncu --set full) into a small text file: key throughput, occupancy, DRAM traffic,
issue statistics and the top stall reasons.  Usage: tools/ncu_summary.py in.ncu-rep out.txt [note...]"""
import csv, subprocess, sys, io
KEYS = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed", "smsp__inst_executed.sum", "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "sm__inst_executed.sum.per_cycle_elapsed", "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread",
        "launch__grid_size", "launch__block_size", "launch__shared_mem_per_block_static", "launch__occupancy_limit_shared_mem",
        "launch__occupancy_limit_registers", "launch__waves_per_multiprocessor", "sm__cycles_elapsed.avg", "sm__cycles_elapsed.avg.per_second",
        "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "lts__t_sector_hit_rate.pct", "l1tex__t_sector_hit_rate.pct",
        "sm__pipe_alu_cycles_active.avg.pct_of_peak_sustained_active", "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active", "smsp__thread_inst_executed_per_inst_executed.ratio"]
def main():
    rep, out = sys.argv[1], sys.argv[2]; note = " ".join(sys.argv[3:])
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units = rows[0], rows[1]
    with open(out, "w") as f:
        f.write(f"# ncu --set full summary of {rep.split('/')[-1]}\n# {note}\n")
        for row in rows[2:]:
            name = row[hdr.index("Kernel Name")] if "Kernel Name" in hdr else "?"
            f.write(f"\nkernel: {name}\n")
            for i, h in enumerate(hdr):
                if h in KEYS: f.write(f"  {h:75s} {row[i]:>18s} {units[i]}\n")
            stalls = [(float(row[i]), h) for i, h in enumerate(hdr) if h.startswith("smsp__average_warp") and "issue_stalled" in h and h.endswith("_per_issue_active.ratio") and row[i]]
            if not stalls:
                stalls = [(float(row[i]), h) for i, h in enumerate(hdr) if "warp_issue_stalled" in h and h.endswith(".pct") and row[i]]
            for v, h in sorted(stalls, reverse=True)[:8]: f.write(f"  stall {h:69s} {v:18.3f}\n")
if __name__ == "__main__":
    main()
