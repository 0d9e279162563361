#!/usr/bin/env python
"""Summarise an `ncu --metrics gpu__time_duration.sum --csv --log-file X.csv <cmd>` launch list: per kernel name the
launch count, average duration and share of the total kernel time (cold-cache, serialised: compare SHARES).
usage: python scripts/launch_summary.py launches.csv "header line" > launch_list_summary.txt"""
import csv
import sys
from collections import defaultdict

rows = []
with open(sys.argv[1], newline="") as f:
    lines = [ln for ln in f if not ln.startswith("==")]
rd = csv.reader(lines)
hdr = next(rd)
ix = {h: i for i, h in enumerate(hdr)}
kn, mv, mu = ix["Kernel Name"], ix["Metric Value"], ix["Metric Unit"]
agg = defaultdict(lambda: [0, 0.0])
for r in rd:
    if len(r) <= mv or r[ix["Metric Name"]] != "gpu__time_duration.sum":
        continue
    v = float(r[mv].replace(",", ""))
    u = r[mu]
    us = v / 1000.0 if u in ("nsecond", "ns") else (v if u in ("usecond", "us") else v * 1000.0 if u in ("msecond", "ms") else v)
    a = agg[r[kn]]
    a[0] += 1; a[1] += us
tot = sum(a[1] for a in agg.values())
n = sum(a[0] for a in agg.values())
if len(sys.argv) > 2:
    print(sys.argv[2])
print(f"{n} launches, {tot / 1000.0:.2f} ms kernel time (cold-cache, serialised under the profiler: SHARES, not absolute times).")
for name, (c, t) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
    print(f"  {100 * t / tot:5.1f}%  n={c:4d}  avg {t / c:8.1f} us  {name[:110]}")
