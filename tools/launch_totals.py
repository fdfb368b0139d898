#!/usr/bin/env python3
"""Per-kernel totals of an `ncu --metrics gpu__time_duration.sum --csv` launch list, from the launch that matches
`--from <kernel substring>` (its LAST-BUT-k occurrence, default: first) to the end: count, total ms, share.

   python tools/launch_totals.py launches_plonk.csv --from k_plonk_ratio --nth -1"""
import argparse
import csv
import re
from collections import OrderedDict


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("csv")
    ap.add_argument("--from", dest="frm", default=None)
    ap.add_argument("--nth", type=int, default=0, help="which occurrence of --from starts the window (negative: from the end)")
    ap.add_argument("--back", type=int, default=0, help="start this many launches before the match")
    args = ap.parse_args()
    rows = [r for r in csv.reader(open(args.csv, newline="")) if r]
    hdr = next(i for i, r in enumerate(rows) if "Kernel Name" in r)
    names = rows[hdr]
    kn, mv, mu = (names.index(x) for x in ("Kernel Name", "Metric Value", "Metric Unit"))
    launches = []
    for r in rows[hdr + 1:]:
        if len(r) <= mv:
            continue
        v = float(r[mv].replace(",", ""))
        ms = v / 1e6 if r[mu] in ("ns", "nsecond") else (v / 1e3 if r[mu] in ("us", "usecond") else v)
        short = re.sub(r"^void ", "", r[kn])
        short = re.sub(r"<.*", "", short).replace("gb200::", "")
        short = re.sub(r"\(.*", "", short)
        short = re.sub(r"^cub::\w+::", "cub::", short)
        launches.append((short, ms))
    start = 0
    if args.frm:
        idx = [i for i, l in enumerate(launches) if args.frm in l[0]]
        if not idx:
            raise SystemExit("no launch matches " + args.frm)
        start = max(0, idx[args.nth] - args.back)
    win = launches[start:]
    tot = OrderedDict()
    for k, ms in win:
        c, t = tot.get(k, (0, 0.0))
        tot[k] = (c + 1, t + ms)
    total = sum(t for _, t in tot.values())
    print(f"{len(win)} launches from #{start} of {len(launches)}, {total:.2f} ms in kernels\n")
    print("| kernel | launches | ms | share |\n|---|---:|---:|---:|")
    for k, (c, t) in sorted(tot.items(), key=lambda kv: -kv[1][1]):
        print(f"| {k} | {c} | {t:.3f} | {100 * t / total:.1f}% |")


if __name__ == "__main__":
    main()
