#!/usr/bin/env python3
"""Turns an .ncu-rep into a small markdown table (no GPU needed), e.g. under the local, git-ignored profiles/:
    python tools/ncu_summary.py validate_out/val_prof.ncu-rep > profiles/ncu_<what>.md
"""
import csv
import subprocess
import sys

METRICS = [
    ("gpu__time_duration.sum", "time"),
    ("dram__bytes_read.sum", "dram read"),
    ("dram__bytes_write.sum", "dram write"),
    ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram %"),
    ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm %"),
    ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue active %"),
    ("smsp__inst_executed.sum", "warp insts"),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "warps active %"),
    ("launch__registers_per_thread", "regs"),
    ("launch__grid_size", "grid"),
    ("launch__block_size", "block"),
    ("launch__shared_mem_per_block_dynamic", "dyn smem"),
    ("launch__occupancy_limit_registers", "occ lim regs"),
    ("launch__occupancy_limit_shared_mem", "occ lim smem"),
    ("l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "smem bank conflicts"),
]


def main():
    rep = sys.argv[1]
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
    rows = list(csv.reader(out.splitlines()))
    hdr, units, data = rows[0], rows[1], rows[2:]
    ix = {h: i for i, h in enumerate(hdr)}
    cols = [(m, n) for m, n in METRICS if m in ix]
    print(f"ncu --set full --clock-control none, report `{rep.split('/')[-1]}` (per-launch values; times are cold-cache and serialised)\n")
    print("| kernel | " + " | ".join(n for _, n in cols) + " |")
    print("|---|" + "---|" * len(cols))
    for r in data:
        name = r[ix["Kernel Name"]].split("(")[0].replace("hapb200::", "").replace("void ", "")
        cells = []
        for m, _ in cols:
            v, u = r[ix[m]], units[ix[m]]
            try:
                v = f"{float(v):.4g}"
            except ValueError:
                pass
            cells.append(f"{v} {u}".strip())
        print(f"| `{name}` | " + " | ".join(cells) + " |")


if __name__ == "__main__":
    main()
