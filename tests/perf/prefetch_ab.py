#!/usr/bin/env python3
"""One-knob A/B of the pair-round kernels on one H100 (AB_KNOB names the environment variable; written for the software-prefetch
experiment, PCGPU_PAIR_PREFETCH = distance in slots, +16 = into L1 -- measured slower and removed):
single-MSM stage timings (CUDA events of the library's profiler) and the batch commit+open entry point, every variant checked
against the first.  python tests/perf/prefetch_ab.py [log_n] [values...] > perf_out/prefetch_ab.jsonl"""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import numpy as np
import torch

import pkgload

pc = pkgload.load()
from poly_commit_b200 import params  # noqa: E402


def main():
    logn = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    values = sys.argv[2:] or ["0", "1", "2", "3", "4", "17", "18"]
    knob = os.environ.get("AB_KNOB", "PCGPU_PAIR_PREFETCH")
    cid = pc.BLS12_381
    n = (1 << logn) + 1
    eng = pc.Engine(0)
    ks = torch.from_numpy(params.random_fr(cid, n, 1001).view(np.int64)).cuda()
    d_bases = torch.empty((n, 12), dtype=torch.int64, device="cuda")
    eng.fixed_base_mul(cid, params.g1_generator(cid), ks.data_ptr(), n=n, flags=pc.DEVICE_PTRS, out=d_bases.data_ptr())
    d_sc = torch.from_numpy(params.random_fr(cid, n, 77).view(np.int64)).cuda()
    z = params.random_fr(cid, 1, 4)[0]
    fl = pc.SCALARS_MONT | pc.DEVICE_PTRS
    srs = eng.srs_register(cid, d_bases.data_ptr(), n=n, flags=pc.DEVICE_PTRS | pc.SRS_PRECOMPUTE)
    ref = None
    for v in values:
        os.environ[knob] = v
        got = eng.msm(srs, d_sc.data_ptr(), n=n, flags=fl)
        if ref is None:
            ref = got
        ok = bool((got[0] == ref[0]).all() and got[1] == ref[1])
        for _ in range(2):
            eng.msm(srs, d_sc.data_ptr(), n=n, flags=fl)
        eng.profile_enable(True)
        reps = 6
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(reps):
            eng.msm(srs, d_sc.data_ptr(), n=n, flags=fl)
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) / reps * 1e3
        st = {"pair_rounds": round(eng.profile_get(11)[0] / reps, 4), "pair_round0": round(eng.profile_get(12)[0] / reps, 4),
              "accumulate": round(eng.profile_get(4)[0] / reps, 4)}
        eng.profile_enable(False)

        def t(fn, reps=3):
            fn(); torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(reps):
                fn()
            torch.cuda.synchronize()
            return (time.perf_counter() - t0) / reps * 1e3
        batch = t(lambda: eng.kzg_commit_open_batch(srs, [(d_sc.data_ptr(), n)] * 8, z, flags=pc.DEVICE_PTRS)) / 8
        print(json.dumps({"what": f"msm 2^{logn}", knob: v, "ok": ok, "ms_per_msm": round(ms, 4), "stages_ms": st,
                          "commit_open_batch8_ms_per_poly": round(batch, 3)}), flush=True)


if __name__ == "__main__":
    main()
