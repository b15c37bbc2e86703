"""Summary of one ncu --set full capture as JSON.

    python tools/ncu_summary.py <report.ncu-rep> > <name>_summary.json
"""
import csv
import io
import json
import subprocess
import sys


def main():
    out = subprocess.run(["ncu", "-i", sys.argv[1], "--page", "raw", "--csv"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    head, units, vals = rows[0], rows[1], rows[2]
    col = {h: (vals[i], units[i]) for i, h in enumerate(head)}
    keep = ["Kernel Name", "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
            "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum", "launch__registers_per_thread",
            "launch__grid_size", "launch__block_size", "launch__shared_mem_per_block_dynamic", "l1tex__t_sector_hit_rate.pct",
            "lts__t_sector_hit_rate.pct", "smsp__issue_active.avg.pct"]
    res = {}
    for k in keep:
        if k in col:
            res[k] = col[k][0]
            if col[k][1]:
                res[k + " [unit]"] = col[k][1]
    stalls = {}
    for h, (v, _) in col.items():
        if h.startswith("smsp__average_warps_issue_stalled_") and h.endswith("_per_issue_active.ratio"):
            stalls[h[len("smsp__average_warps_issue_stalled_"):-len("_per_issue_active.ratio")]] = round(float(v), 6)
    res["stall_cycles_per_issue"] = dict(sorted(stalls.items()))
    json.dump(res, sys.stdout, indent=1)
    print()


main()
