#!/usr/bin/env python3
"""Device timing of the G2 MSM (<E::G2 as VariableBaseMSM>::msm_bigint) at 2^16 / 2^18 / 2^20 terms and of
MultilinearPC::open at nv = 20, on BLS12-381 and BN254.  Bases and scalars are resident in HBM (DEVICE_PTRS scalars); every
call is synchronous, so a host clock around it measures the whole call, host tail included.  Each configuration is warmed up
once and then timed `--reps` times; the JSON lines give the median and the spread (min, max).  The open is split into the
fold chain (profile stage 16) and the rest (the nv G2 MSMs and their host tails) from a separate profiled run.
Prints the card's name and power limit first.
Run on the GPU box:  python tests/perf/mlpc_bench.py > perf_out/mlpc_bench.jsonl"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import pkgload  # noqa: E402

pc = pkgload.load()
from oracle import pyref  # noqa: E402
from tests import g2_cases as gc  # noqa: E402
from tests import util  # noqa: E402


def timed(fn, reps):
    fn()
    out = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t0) * 1e3)
    return out


def stats(ms):
    return {"ms_median": round(statistics.median(ms), 3), "ms_min": round(min(ms), 3), "ms_max": round(max(ms), 3), "runs": len(ms)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--max-log", type=int, default=20)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"card": card.stdout.strip()}), flush=True)
    eng = pc.Engine(0)
    for cname in gc.PAIRING:
        C = pyref.Curve(cname)
        gid = gc.group(pc, cname)
        h_xy, _ = gc.to_limbs(cname, [gc.generator(cname)])
        nmax = 1 << a.max_log
        bases = eng.g2_fixed_base_mul(gid, h_xy[0], util.rand_fr_fast(cname, nmax, 1))
        srs = eng.srs_register(gid, bases)
        sc = torch.from_numpy(util.rand_fr_fast(cname, nmax, 2).view("int64")).cuda()
        for lg in (16, 18, 20):
            if lg > a.max_log:
                continue
            ms = timed(lambda: eng.msm(srs, sc.data_ptr(), n=1 << lg, flags=pc.DEVICE_PTRS | pc.SCALARS_MONT), a.reps)
            g = eng.msm_last_geometry()
            print(json.dumps({"kernel": f"G2 MSM {cname} 2^{lg}, device-resident scalars", **stats(ms),
                              "path": g["path"], "c": g["c"], "W": g["W"]}), flush=True)
        srs.release()
        nv = a.max_log
        levels = [eng.g2_fixed_base_mul(gid, h_xy[0], util.rand_fr_fast(cname, 1 << (nv - i), 10 + i)) for i in range(nv)]
        key = eng.mlpc_register(C.id, levels)
        ev = torch.from_numpy(util.rand_fr_fast(cname, 1 << nv, 3).view("int64")).cuda()
        pt = util.rand_fr_fast(cname, nv, 4)
        ms = timed(lambda: eng.mlpc_open(key, ev.data_ptr(), pt, n=1 << nv, flags=pc.DEVICE_PTRS), a.reps)
        eng.profile_enable(True)
        eng.mlpc_open(key, ev.data_ptr(), pt, n=1 << nv, flags=pc.DEVICE_PTRS)
        fold = eng.profile_get(16)[0]
        stages = {s: round(eng.profile_get(s)[0], 3) for s in range(7)}
        eng.profile_enable(False)
        print(json.dumps({"kernel": f"MultilinearPC open {cname} nv = {nv} ({(1 << nv) - 1} G2 terms over {nv} MSMs)", **stats(ms),
                          "profiled_fold_ms": round(fold, 3), "profiled_msm_stage_ms": stages}), flush=True)
        key.release()
    eng.close()


if __name__ == "__main__":
    main()
