#!/usr/bin/env python3
"""Markdown table of ONE MSM's launches from an `ncu --metrics gpu__time_duration.sum --csv` launch list of bench.py:
the launches between the last two k_msm_decompose, with each kernel's share of their sum.

   python tools/launch_list.py launches.csv > launches_<what>.md"""
import csv
import re
import sys


def main():
    rows = [r for r in csv.reader(open(sys.argv[1], newline="")) if r]
    hdr = next(i for i, r in enumerate(rows) if "Kernel Name" in r)
    names = rows[hdr]
    kn, gs, bs, mv, mu = (names.index(x) for x in ("Kernel Name", "Grid Size", "Block Size", "Metric Value", "Metric Unit"))
    launches = []
    for r in rows[hdr + 1:]:
        if len(r) <= mv:
            continue
        v = float(r[mv].replace(",", ""))
        us = v / 1e3 if r[mu] in ("ns", "nsecond") else (v * 1e3 if r[mu] in ("ms", "msecond") else v)
        short = re.sub(r"^void ", "", r[kn])
        short = re.sub(r"<.*", "", short).replace("gb200::", "")
        short = re.sub(r"^cub::\w+::", "cub::", short)
        launches.append((short, r[gs], r[bs], us))
    idx = [i for i, l in enumerate(launches) if l[0] == "k_msm_decompose"]
    if len(idx) < 2:
        sys.exit("fewer than two k_msm_decompose launches in the list")
    one = launches[idx[-2]:idx[-1]]
    total = sum(l[3] for l in one)
    print("| kernel | grid | block | us | share |\n|---|---|---|---:|---:|")
    for k, g, b, us in one:
        print(f"| {k} | {g} | {b} | {us:.1f} | {100 * us / total:.1f}% |")
    print(f"| **total** | | | {total:.1f} | 100% |")


if __name__ == "__main__":
    main()
