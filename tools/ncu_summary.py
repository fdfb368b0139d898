#!/usr/bin/env python3
"""Markdown summary of one `ncu --set full` capture, read back on the CPU box:

   ncu -i prof.ncu-rep --page raw --csv > /tmp/prof.csv
   python tools/ncu_summary.py /tmp/prof.csv [kernel-substring] > ncu_<kernel>_summary.md

The CSV of `--page raw` has one row per profiled launch and one column per metric (first rows: names, then units).
Only the metrics that matter on this path are kept: duration, the pipes (IMAD.WIDE issues on fmaheavy), issue rate,
occupancy, local-memory traffic and DRAM bytes (-> `roofline.traffic` of bench.py).  A formatter, nothing else."""
import csv
import sys

WANT = [
    ("gpu__time_duration.sum", "kernel time"),
    ("launch__grid_size", "grid"), ("launch__block_size", "block"), ("launch__registers_per_thread", "registers / thread"),
    ("launch__occupancy_limit_registers", "occupancy limit (registers), blocks/SM"),
    ("launch__occupancy_limit_shared_mem", "occupancy limit (shared memory), blocks/SM"),
    ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "SM throughput, % of peak"),
    ("sm__pipe_fmaheavy_cycles_active.avg.pct_of_peak_sustained_elapsed", "pipe fmaheavy (IMAD.WIDE), % of peak"),
    ("sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_elapsed", "pipe fma, % of peak"),
    ("sm__pipe_alu_cycles_active.avg.pct_of_peak_sustained_elapsed", "pipe alu, % of peak"),
    ("sm__pipe_fp64_cycles_active.avg.pct_of_peak_sustained_elapsed", "pipe fp64, % of peak"),
    ("smsp__issue_active.avg.per_cycle_active", "issue active, inst/cycle/SMSP"),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "warps active, % of peak"),
    ("smsp__inst_executed_op_local_ld.sum", "local loads (instructions)"), ("smsp__inst_executed_op_local_st.sum", "local stores (instructions)"),
    ("smsp__inst_executed_op_shared_ld.sum", "shared loads (instructions)"), ("smsp__inst_executed_op_shared_st.sum", "shared stores (instructions)"),
    ("l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "shared-memory bank conflicts"),
    ("lts__t_sector_hit_rate.pct", "L2 sector hit rate, %"),
    ("dram__bytes_read.sum", "DRAM bytes read"), ("dram__bytes_write.sum", "DRAM bytes written"),
    ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "DRAM throughput, % of peak"),
]
STALLS = "smsp__average_warps_issue_stalled_"


def main():
    path = sys.argv[1]
    pick = sys.argv[2] if len(sys.argv) > 2 else ""
    rows = list(csv.reader(open(path, newline="")))
    hdr = next(i for i, r in enumerate(rows) if "Kernel Name" in r)
    names, units = rows[hdr], rows[hdr + 1]
    col = {n: i for i, n in enumerate(names)}
    launches = [r for r in rows[hdr + 2:] if len(r) == len(names) and pick in r[col["Kernel Name"]]]
    if not launches:
        sys.exit("no launch matches " + repr(pick))
    for r in launches:
        print(f"## {r[col['Kernel Name']][:120]}\n")
        print("| metric | value | unit |\n|---|---|---|")
        for key, label in WANT:
            if key in col and r[col[key]] != "":
                print(f"| {label} (`{key}`) | {r[col[key]]} | {units[col[key]]} |")
        rd, wr = col.get("dram__bytes_read.sum"), col.get("dram__bytes_write.sum")
        if rd is not None and wr is not None:
            def b(i):
                v = float(r[i].replace(",", ""))
                u = units[i].lower()
                return v * {"byte": 1, "kbyte": 1e3, "mbyte": 1e6, "gbyte": 1e9}.get(u, 1)
            print(f"| **traffic (read + write)** | {(b(rd) + b(wr)) / 1e9:.4f} | GB |")
        st = sorted(((float(r[i].replace(",", "")), n) for n, i in col.items()
                     if n.startswith(STALLS) and n.endswith("_per_warp_active.pct") is False and r[i] not in ("", "n/a")
                     and n.endswith(".ratio")), reverse=True)[:6]
        if st:
            print("\nTop stall reasons (warps per issue): " + ", ".join(f"{n[len(STALLS):].split('.')[0]} {v:.2f}" for v, n in st))
        print()


if __name__ == "__main__":
    main()
