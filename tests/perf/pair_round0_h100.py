#!/usr/bin/env python3
"""Round 0 of the MSM's batched-affine pair rounds on one H100, in one process:

  gather-rate probe   plain torch indexing into a 2 GB int64 tensor: 15.7 M random 128-byte rows (16 words) against 15.7 M
                      random 64-byte rows (8 words), the row count and record size of one 2^20-term BLS12-381 MSM over the
                      window-folded tables (c = 17, 15 groups).  Each repetition times both sizes back to back with CUDA
                      events; a sequential copy of the same output bytes is timed beside them, since indexing also writes
                      its result.  This is the rate of torch's indexing kernel, which pays per row, not of the HBM: on an
                      H100 it moves ~1.7e9 rows/s at either width, while round 0 itself sustains over 1e10 random 64-byte
                      accesses/s.  So equal times for both widths do not show that the HBM charges per access.
  per-stage times     one 2^20 + 1-term BLS12-381 MSM on a folded SRS, the library's CUDA-event stage profile per repetition:
                      stage 12 is round 0, stage 11 all pair rounds, stages 0-5 the rest of the pipeline.

Prints one JSON line per part, with the card name, power limit and maximum SM clock read in the same run.
  python tests/perf/pair_round0_h100.py [--reps 20] [--root DIR] > perf_out/pair_round0.jsonl
--root loads the package from another checkout of the project (built in place), for a before / after comparison."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

STAGES = {0: "digits", 1: "scan", 2: "scatter", 3: "tasks", 4: "accumulate", 5: "reduce", 11: "pair_rounds", 12: "pair_round0"}
ROWS = 15 * (1 << 20)          # table records one 2^20-term MSM touches: 2^20 bases x 15 windows
TABLE_BYTES = 1 << 31


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else f"nvidia-smi failed: {q.stderr.strip()}"


def spread(xs):
    xs = sorted(xs)
    return {"median": round(float(np.median(xs)), 4), "min": round(xs[0], 4), "max": round(xs[-1], 4), "n": len(xs)}


def gather_probe(reps):
    table = torch.empty(TABLE_BYTES // 8, dtype=torch.int64, device="cuda").random_()
    g = torch.Generator(device="cuda").manual_seed(5)
    views = {128: table.view(-1, 16), 64: table.view(-1, 8)}
    idx = {b: torch.randint(0, v.shape[0], (ROWS,), device="cuda", generator=g) for b, v in views.items()}
    out = {b: torch.empty((ROWS, v.shape[1]), dtype=torch.int64, device="cuda") for b, v in views.items()}
    seq = {b: table[:out[b].numel()].view_as(out[b]) for b in views}

    def run(b, kind):
        if kind == "gather":
            torch.index_select(views[b], 0, idx[b], out=out[b])
        else:
            out[b].copy_(seq[b])

    kinds = [(b, k) for b in (128, 64) for k in ("gather", "copy")]
    for b, k in kinds:
        run(b, k)
    times = {bk: [] for bk in kinds}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2 * len(kinds))]
    for _ in range(reps):
        for i, (b, k) in enumerate(kinds):
            ev[2 * i].record()
            run(b, k)
            ev[2 * i + 1].record()
        torch.cuda.synchronize()
        for i, bk in enumerate(kinds):
            times[bk].append(ev[2 * i].elapsed_time(ev[2 * i + 1]))
    res = {}
    for (b, k), ts in times.items():
        s = spread(ts)
        sec = s["median"] * 1e-3
        s["accesses_per_s"] = ROWS / sec
        s["read_bytes_per_s"] = ROWS * b / sec
        res[f"{k}_{b}B"] = s
    res["ratio_gather_128_over_64"] = round(res["gather_128B"]["median"] / res["gather_64B"]["median"], 3)
    del table, out, seq
    torch.cuda.empty_cache()
    return res


def msm_stages(root, reps):
    sys.path.insert(0, root)
    import pkgload
    pc = pkgload.load()
    from poly_commit_b200 import params
    cid = pc.BLS12_381
    n = (1 << 20) + 1
    eng = pc.Engine(0)
    ks = torch.from_numpy(params.random_fr(cid, n, 1001).view(np.int64)).cuda()
    d_bases = torch.empty((n, 12), dtype=torch.int64, device="cuda")
    eng.fixed_base_mul(cid, params.g1_generator(cid), ks.data_ptr(), n=n, flags=pc.DEVICE_PTRS, out=d_bases.data_ptr())
    d_sc = torch.from_numpy(params.random_fr(cid, n, 77).view(np.int64)).cuda()
    srs = eng.srs_register(cid, d_bases.data_ptr(), n=n, flags=pc.DEVICE_PTRS | pc.SRS_PRECOMPUTE)
    fl = pc.SCALARS_MONT | pc.DEVICE_PTRS
    ref = eng.msm(srs, d_sc.data_ptr(), n=n, flags=fl)
    for _ in range(3):
        eng.msm(srs, d_sc.data_ptr(), n=n, flags=fl)
    geom = eng.msm_last_geometry()
    per = {name: [] for name in STAGES.values()}
    total = []
    same = True
    for _ in range(reps):
        eng.profile_enable(True)
        got = eng.msm(srs, d_sc.data_ptr(), n=n, flags=fl)
        for s, name in STAGES.items():
            per[name].append(eng.profile_get(s)[0])
        eng.profile_enable(False)
        total.append(sum(per[STAGES[s]][-1] for s in (0, 1, 2, 11, 3, 4, 5)))
        same = same and bool((got[0] == ref[0]).all() and got[1] == ref[1])
    eng.close()
    return {"root": os.path.abspath(root), "geometry": {k: geom[k] for k in ("c", "W", "G", "R", "T") if k in geom},
            "same_result_every_rep": same, "result_x_word0": int(ref[0].reshape(-1)[0]),
            "device_stages_ms": round(float(np.median(total)), 4), "stages_ms": {k: spread(v) for k, v in per.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
    ap.add_argument("--skip-probe", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this script measures the GPU")
    c = card()
    if not args.skip_probe:
        print(json.dumps({"what": "gather rate", "card": c, "rows": ROWS, "table_bytes": TABLE_BYTES, **gather_probe(args.reps)}),
              flush=True)
    print(json.dumps({"what": "msm 2^20+1 bls12_381 folded", "card": c, **msm_stages(args.root, args.reps)}), flush=True)


if __name__ == "__main__":
    main()
