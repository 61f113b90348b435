#!/usr/bin/env python
"""Print the per-kernel table of the raw ncu exports (prof_out/<prefix>_<kernel>.csv, written by tools/ncu_export.sh).
usage: ncu_summary.py <prefix>     e.g. r1_ncu_full_v10"""
import csv, glob, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
prefix = sys.argv[1]
cols = [("grid x block", None), ("regs", "launch__registers_per_thread"), ("time", "gpu__time_duration.sum"), ("DRAM read", "dram__bytes_read.sum"),
        ("DRAM write", "dram__bytes_write.sum"), ("DRAM % of peak", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed"), ("L2 hit", "lts__t_sector_hit_rate.pct"),
        ("warp inst", "smsp__inst_executed.sum"), ("issue-active", "smsp__issue_active.avg.pct_of_peak_sustained_active"),
        ("warps active", "sm__warps_active.avg.pct_of_peak_sustained_active"), ("lanes/inst", "smsp__thread_inst_executed_per_inst_executed.ratio"),
        ("top stall (warps per issue)", None)]
print("| kernel | " + " | ".join(c[0] for c in cols) + " |")
print("|---|" + "---|" * len(cols))
for f in sorted(glob.glob(os.path.join(ROOT, "prof_out", prefix + "_*.csv"))):
    rows = list(csv.reader(open(f)))
    H, U, V = rows[0], rows[1], rows[2]
    def g(n, unit=True):
        if n not in H:
            return "n/a"
        i = H.index(n)
        try:
            x = float(V[i]); v = f"{x:.3g}" if abs(x) < 1e5 else f"{x:.3e}"
        except ValueError:
            v = V[i]
        return (v + " " + U[i]).strip() if unit else v
    out = []
    for name, metric in cols:
        if name == "grid x block":
            out.append(f"{g('launch__grid_size', False)} x {g('launch__block_size', False)}")
        elif name.startswith("top stall"):
            st = sorted(((float(V[i]), n.split("issue_stalled_")[1].split("_per_")[0]) for i, n in enumerate(H)
                         if n.startswith("smsp__average_warps_issue_stalled") and n.endswith("_per_issue_active.ratio")), reverse=True)
            out.append(", ".join(f"{n} {v:.2f}" for v, n in st[:3]))
        else:
            out.append(g(metric))
    print(f"| `{os.path.basename(f)[len(prefix) + 1:-4]}` | " + " | ".join(out) + " |")
