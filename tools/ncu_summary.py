#!/usr/bin/env python3
"""Per-kernel summary of an `ncu --set full` report exported with `ncu -i X.ncu-rep --page raw --csv`: one line per launch with
duration, DRAM bytes and fraction of peak, pipe activity, occupancy, registers.
    python tools/ncu_summary.py perf_out/raw.csv > perf_out/ncu_<what>_summary.txt"""
import csv
import sys

COLS = [("gpu__time_duration.sum", "time"), ("dram__bytes_read.sum", "dram_rd"), ("dram__bytes_write.sum", "dram_wr"),
        ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram%"), ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm%"),
        ("sm__pipe_fmaheavy_cycles_active.avg.pct_of_peak_sustained_active", "fmaheavy%"),
        ("sm__pipe_alu_cycles_active.avg.pct_of_peak_sustained_active", "alu%"),
        ("sm__warps_active.avg.pct_of_peak_sustained_active", "warps%"), ("lts__t_sector_hit_rate.pct", "l2hit%"),
        ("launch__registers_per_thread", "regs"), ("launch__grid_size", "grid"), ("launch__block_size", "block"),
        ("launch__shared_mem_per_block_dynamic", "smem_dyn")]


def main(path):
    rows = list(csv.reader(open(path)))
    hdr, units = rows[0], rows[1]
    kn = hdr.index("Kernel Name")
    print(f"# source: {path} (ncu --set full --clock-control none; per-launch values, cold caches, serialised)")
    for r in rows[2:]:
        if len(r) <= kn:
            continue
        name = r[kn]
        short = name[:name.index("(")] if "(" in name else name
        parts = []
        for m, label in COLS:
            if m in hdr and r[hdr.index(m)] not in ("", "n/a"):
                parts.append(f"{label}={r[hdr.index(m)]}{units[hdr.index(m)] if units[hdr.index(m)] not in ('', '%') else ''}")
        print(short[-110:], "|", "  ".join(parts))


if __name__ == "__main__":
    main(sys.argv[1])
