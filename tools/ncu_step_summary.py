"""Summarise an `ncu --csv --metrics ...` log of one policy step per kernel: launches, total time, DRAM bytes, achieved GB/s,
time-weighted tensor-pipe / issue activity.  Usage: python tools/ncu_step_summary.py kernel_metrics_step.csv [hbm_peak_gbs]"""
import csv
import re
import sys
from collections import defaultdict

path = sys.argv[1]
peak = float(sys.argv[2]) if len(sys.argv) > 2 else 6564.2
lines = open(path, newline="").read().splitlines()
start = next(i for i, l in enumerate(lines) if l.startswith('"ID"'))
rows = list(csv.DictReader(lines[start:]))
per = defaultdict(dict)  # launch id -> metric -> value
name = {}
grid = {}
for r in rows:
    i = int(r["ID"])
    name[i] = r["Kernel Name"]
    grid[i] = (r["Grid Size"], r["Block Size"])
    try:
        per[i][r["Metric Name"]] = float(r["Metric Value"].replace(",", ""))
    except ValueError:
        pass


def short(n):
    n = re.sub(r"^void ", "", n)
    n = re.sub(r"\(.*$", "", n)
    return n[:110]


agg = defaultdict(lambda: [0, 0.0, 0.0, 0.0, 0.0])  # launches, ns, bytes, tensor*ns, issue*ns
for i, m in per.items():
    a = agg[short(name[i])]
    t = m.get("gpu__time_duration.sum", 0.0)
    a[0] += 1
    a[1] += t
    a[2] += m.get("dram__bytes_read.sum", 0.0) + m.get("dram__bytes_write.sum", 0.0)
    a[3] += t * m.get("sm__pipe_tensor_subpipe_hmma_cycles_active.avg.pct_of_peak_sustained_active", 0.0)
    a[4] += t * m.get("smsp__issue_active.avg.pct_of_peak_sustained_active", 0.0)
tot = sum(a[1] for a in agg.values())
totb = sum(a[2] for a in agg.values())
print(f"total {tot / 1e6:.2f} ms over {sum(a[0] for a in agg.values())} launches, DRAM {totb / 1e9:.1f} GB "
      f"({totb / tot:.0f} GB/s average = {100 * totb / tot / peak:.1f}% of the {peak:.0f} GB/s copy peak)")
for k, a in sorted(agg.items(), key=lambda kv: -kv[1][1]):
    n, t, b, tp, ip = a
    print(f"  {t / 1e6:7.3f} ms x{n:4d}  {100 * t / tot:5.1f}%  dram {b / 1e9:7.3f} GB {b / t:6.0f} GB/s ({100 * b / t / peak:4.1f}%)  "
          f"tensor {tp / t:5.1f}%  issue {ip / t:5.1f}%  {k}")
