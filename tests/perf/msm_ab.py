#!/usr/bin/env python3
"""A/B timings of the MSM pipeline's tuning knobs on one H100 (device-resident inputs, CUDA-event stage timings from the
library's profiler, wall clock around synchronous calls), every variant checked against the first one:
  window bits of the folded tables (PCGPU_SRS_C: 16 -> 16 windows, 17 -> 15 windows),
  pair-round kernel (PCGPU_PAIR_MODE: 0 one-shot, 1 chunked persistent) and its chunk length (PCGPU_PAIR_K),
  one call (kzg_commit_open) against commit followed by open, and the batch entry point.
  python tests/perf/msm_ab.py [log_n] > perf_out/msm_ab.jsonl"""
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

STAGES = ["digits", "scan", "scatter", "tasks", "accumulate", "reduce", "host", "division"]


def main():
    logn = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    cid = pc.BLS12_381
    n = (1 << logn) + 1
    eng = pc.Engine(0)
    ks = torch.from_numpy(params.random_fr(cid, n, 1001).view(np.int64)).cuda()
    d_bases = torch.empty((n, 12), dtype=torch.int64, device="cuda")
    eng.fixed_base_mul(cid, params.g1_generator(cid), ks.data_ptr(), n=n, flags=pc.DEVICE_PTRS, out=d_bases.data_ptr())
    d_sc = torch.from_numpy(params.random_fr(cid, n, 77).view(np.int64)).cuda()
    z = params.random_fr(cid, 1, 4)[0]
    fl = pc.SCALARS_MONT | pc.DEVICE_PTRS
    ref = None
    variants = [dict(PCGPU_SRS_C="16", PCGPU_PAIR_MODE="0"), dict(PCGPU_SRS_C="17", PCGPU_PAIR_MODE="0"),
                dict(PCGPU_SRS_C="17", PCGPU_PAIR_MODE="0", PCGPU_MSM_AFFINE_ROUNDS="4")]
    knobs = ("PCGPU_SRS_C", "PCGPU_PAIR_MODE", "PCGPU_PAIR_K", "PCGPU_MSM_AFFINE_ROUNDS")
    srs_cache = {}
    for v in variants:
        for k in knobs:
            os.environ.pop(k, None)
        os.environ.update(v)
        c = v["PCGPU_SRS_C"]
        if c not in srs_cache:
            srs_cache[c] = eng.srs_register(cid, d_bases.data_ptr(), n=n, flags=pc.DEVICE_PTRS | pc.SRS_PRECOMPUTE)
        srs = srs_cache[c]
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
        st = {name: round(eng.profile_get(s)[0] / reps, 4) for s, name in enumerate(STAGES)}
        st["pair_rounds"] = round(eng.profile_get(11)[0] / reps, 4)
        st["pair_round0"] = round(eng.profile_get(12)[0] / reps, 4)
        eng.profile_enable(False)
        print(json.dumps({"what": f"msm 2^{logn}", **v, "ok": ok, "ms_per_msm": round(ms, 4), "stages_ms": st}), flush=True)
    # one call vs two calls vs batch, with the best table / kernel setting left in the environment by the last variant above
    for k in knobs:
        os.environ.pop(k, None)
    srs = eng.srs_register(cid, d_bases.data_ptr(), n=n, flags=pc.DEVICE_PTRS | pc.SRS_PRECOMPUTE)
    c0 = eng.kzg_commit(srs, d_sc.data_ptr(), n=n, flags=pc.DEVICE_PTRS)
    w0 = eng.kzg_open(srs, d_sc.data_ptr(), z, n=n, flags=pc.DEVICE_PTRS)
    (c1, _), (w1, _) = eng.kzg_commit_open(srs, d_sc.data_ptr(), z, n=n, flags=pc.DEVICE_PTRS)
    okf = bool((c0[0] == c1).all() and (w0[0] == w1).all())

    def t(fn, reps=8):
        fn(); torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / reps * 1e3

    two = t(lambda: (eng.kzg_commit(srs, d_sc.data_ptr(), n=n, flags=pc.DEVICE_PTRS), eng.kzg_open(srs, d_sc.data_ptr(), z, n=n, flags=pc.DEVICE_PTRS)))
    one = t(lambda: eng.kzg_commit_open(srs, d_sc.data_ptr(), z, n=n, flags=pc.DEVICE_PTRS))
    batch = t(lambda: eng.kzg_commit_open_batch(srs, [(d_sc.data_ptr(), n)] * 8, z, flags=pc.DEVICE_PTRS), reps=3) / 8
    h = d_sc.cpu().numpy().view(np.uint64)
    hp = torch.from_numpy(h.view(np.int64)).pin_memory().numpy().view(np.uint64)
    one_host = t(lambda: eng.kzg_commit_open(srs, hp, z, n=n))
    batch_host = t(lambda: eng.kzg_commit_open_batch(srs, [hp] * 8, z), reps=3) / 8
    print(json.dumps({"what": f"commit+open 2^{logn}, ms per polynomial", "ok": okf, "commit_then_open": round(two, 3),
                      "commit_open_one_call": round(one, 3), "commit_open_batch8": round(batch, 3),
                      "commit_open_one_call_host_buffers": round(one_host, 3), "commit_open_batch8_host_buffers": round(batch_host, 3)}), flush=True)


if __name__ == "__main__":
    main()
