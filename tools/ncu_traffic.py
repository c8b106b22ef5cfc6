#!/usr/bin/env python3
"""Extracts the per-launch DRAM traffic and the headline counters of one kernel from an `ncu --set full` report:
    ncu -i perf_out/pair0.ncu-rep --page raw --csv > perf_out/raw.csv
    python tools/ncu_traffic.py perf_out/raw.csv MsmAffinePairBody 20 perf_out/pair0_traffic.json"""
import csv
import json
import sys

WANT = ["dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__time_duration.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread", "sm__inst_executed_pipe_fmaheavy.sum",
        "sm__pipe_fmaheavy_cycles_active.avg.pct_of_peak_sustained_active", "sm__pipe_alu_cycles_active.avg.pct_of_peak_sustained_active",
        "lts__t_sector_hit_rate.pct", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active"]
UNIT = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "Tbyte": 1e12, "ns": 1, "us": 1e3, "ms": 1e6, "s": 1e9}


def main(path, pattern, log_deg, out):
    rows = list(csv.reader(open(path)))
    hdr, units = rows[0], rows[1]
    kn = hdr.index("Kernel Name")
    sel = [r for r in rows[2:] if len(r) > kn and pattern in r[kn]]
    if not sel:
        raise SystemExit(f"no launch of a kernel matching {pattern!r} in {path}")
    res = {"kernel": sel[0][kn], "launches_in_capture": len(sel), "log_deg": int(log_deg), "source": f"ncu --set full capture, {path}"}
    for m in WANT:
        if m not in hdr:
            continue
        i = hdr.index(m)
        vals = [float(r[i].replace(",", "")) * UNIT.get(units[i], 1) for r in sel if r[i] not in ("", "n/a")]
        if vals:
            res[m] = sum(vals) / len(vals)
    res["dram_bytes_read"] = int(res.get("dram__bytes_read.sum", 0))
    res["dram_bytes_write"] = int(res.get("dram__bytes_write.sum", 0))
    json.dump(res, open(out, "w"), indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main(*sys.argv[1:5])
