"""Condense an .ncu-rep (ncu --set full) into the handful of numbers DESIGN.md / bench.py quote.
usage: python tools/ncu_summary.py x.ncu-rep > x.txt"""
import csv
import subprocess
import sys

WANT = [
    "gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
    "launch__shared_mem_per_block_dynamic", "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem",
    "sm__warps_active.avg.pct_of_peak_sustained_active", "dram__bytes_read.sum", "dram__bytes_write.sum",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active",
    "smsp__issue_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum", "sm__cycles_elapsed.avg",
    "smsp__warps_active.avg.per_cycle_active", "smsp__warps_eligible.avg.per_cycle_active",
    "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "l1tex__t_sector_hit_rate.pct", "lts__t_sector_hit_rate.pct",
]


def main(path):
    raw = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(raw.splitlines()))
    hdr, units = rows[0], rows[1]
    idx = {h: i for i, h in enumerate(hdr)}
    print(f"# {path}")
    for r in rows[2:]:
        print(f"\n## {r[idx['Kernel Name']]}   (launch id {r[idx['ID']]})")
        for w in WANT:
            if w in idx:
                print(f"{w:72s} {r[idx[w]]:>16s} {units[idx[w]]}")
        stalls = []
        for h, i in idx.items():
            if h.startswith("smsp__pcsamp_warps_issue_stalled_") and not h.endswith("_not_issued"):
                try:
                    stalls.append((float(r[i]), h.replace("smsp__pcsamp_warps_issue_stalled_", "")))
                except ValueError:
                    pass
        tot = sum(v for v, _ in stalls) or 1.0
        print("warp-state samples (share): " + ", ".join(f"{n} {100 * v / tot:.1f}%" for v, n in sorted(stalls, reverse=True)[:7]))


if __name__ == "__main__":
    main(sys.argv[1])
