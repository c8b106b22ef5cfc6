"""HyraxPC on one H100 (BN254): commit, open (with the fr_axpy finish) and check of 1 and 64 proofs at nv = 12 ... 22 -- the
reference's hyrax_times sizes and cfg4 (nv = 22) -- with profile stage 19's device time, and pcgpu_fr_row_mul at the cfg4 shape
(2^11 rows x (2^11 + 1) columns, device-resident) against the 3.35 TB/s HBM3 bound.

    python tests/perf/hyrax_pc_bench.py [--nv 12,14,...] [--reps 5] [--row-mul-only] [--lib path/to/libpcgpu.so]

--row-mul-only --lib <library> times only the row product through another build of the library (the parent commit's, for the
before / after figure).  Prints one JSON line per measurement.  Needs a GPU; there is no fallback.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet, HBM3


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def timed(f, reps):
    f()                                     # warm-up: module load, arena growth, comb tables
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        f()                                 # every entry point returns after its stream drained
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def row_mul(eng, reps):
    """pcgpu_fr_row_mul at the cfg4 shape with device-resident operands"""
    from poly_commit_b200.binding import BN254, DEVICE_PTRS
    from tests import util
    rows, cols = 2048, 2049
    v, m = eng.buffer(rows), eng.buffer(rows * cols)
    out = eng.buffer(cols)
    v.write(util.rand_fr_fast("bn254", rows, 1))
    m.write(util.rand_fr_fast("bn254", rows * cols, 2))
    call = lambda: eng._ck(eng.lib.pcgpu_fr_row_mul(eng.ctx, BN254, v.ptr(), m.ptr(), rows, cols, out.ptr(), DEVICE_PTRS))
    nbytes = (rows * cols + rows + cols) * 32
    ms = timed(call, reps)                  # whole-call wall clock: the host side of the call and every launch
    # device time: CUDA events around the call on the stream the library runs on (its launches and its one small copy)
    import torch
    s = torch.cuda.Stream()
    eng.set_stream(s.cuda_stream)
    dev = []
    with torch.cuda.stream(s):
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            call()
            e1.record()
            e1.synchronize()
            dev.append(e0.elapsed_time(e1))
    eng.set_stream(None)
    dms = float(np.median(dev))
    return {"what": "fr_row_mul", "rows": rows, "cols": cols, "call_ms": round(ms, 4), "device_ms": round(dms, 4),
            "device_GB_per_s": round(nbytes / (dms * 1e-3) / 1e9, 1), "share_of_hbm": round(nbytes / (dms * 1e-3) / HBM_BYTES_PER_S, 3)}


def scheme(eng, nv, reps):
    from poly_commit_b200 import hyrax
    from tests import util
    cname = "bn254"
    dim = 1 << (nv // 2)
    xy = util.random_points(cname, dim + 1, 5)
    ck = hyrax.CommitterKey(eng, 1, xy[:dim], xy[dim])
    ev, rnd = util.rand_fr_fast(cname, dim * dim, 6), util.rand_fr_fast(cname, dim, 7)
    point, blinds = util.rand_fr_fast(cname, nv, 8), util.rand_fr_fast(cname, dim + 3, 9)
    ch = util.rand_fr_fast(cname, 1, 10)
    res = {"nv": nv, "dim": dim}
    state = {}

    def commit():
        if "st" in state:
            state["st"].release()
        state["rows"], state["inf"], state["st"] = hyrax.commit_resident(ck, ev, rnd)
    res["commit_ms"] = round(timed(commit, reps), 3)

    def open_():
        state["proofs"] = hyrax.open(ck, [state["st"]], point, blinds, lambda j, *pts: ch[0])
    res["open_ms"] = round(timed(open_, reps), 3)
    eng.profile_enable(True)
    open_()
    ms19, _ = eng.profile_get(19)
    eng.profile_enable(False)
    res["open_stage19_ms"] = round(ms19, 3)
    for count in (1, 64):
        rc = [(state["rows"], state["inf"])] * count
        pr = state["proofs"] * count
        chs = np.tile(ch, (count, 1))
        ok = []
        res[f"check{count}_ms"] = round(timed(lambda: ok.append(hyrax.check(ck, rc, point, pr, chs)), reps), 3)
        assert all(ok[-1])
    state["st"].release()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nv", default="12,14,16,18,20,22")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--row-mul-only", action="store_true")
    ap.add_argument("--lib", default=None)
    a = ap.parse_args()
    import pkgload
    pc = pkgload.load()
    eng = pc.Engine(0, lib_path=a.lib)
    c = card()
    r = row_mul(eng, max(a.reps, 20))
    print(json.dumps(dict(r, lib=a.lib or "this tree", card=c)), flush=True)
    if a.row_mul_only:
        return
    for nv in (int(x) for x in a.nv.split(",")):
        print(json.dumps(dict(scheme(eng, nv, a.reps), card=c)), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
