#!/usr/bin/env python3
"""Prepared against plain pairings on the device: pcgpu_multi_pairing and pcgpu_multi_pairing_prepared on the same points,
alternating in one run, at k = 2 (KZG10::check), 3 and 5 (SonicKZG10's check with no and with two degree bounds) and 21
(MultilinearPC::check at nv = 20) pairs per equation, for count = 1, 256 and 16384 equations per call, on BLS12-381 and BN254.
Points are honest group elements (fixed-base multiples of the generators), resident in HBM (DEVICE_PTRS); the prepared path
pairs the same G1 points with the same G2 points, prepared once.  Every call is synchronous, so a host clock around it
measures the whole call.  Each configuration is warmed up once per path and then timed `--reps` times with the two paths
alternating; the JSON lines give the median and the spread (min, max), and the stage-17 device time (CUDA events around the
Miller and final-exponentiation kernels) from the same calls.  Then pcgpu_g2_prepare of a 4-point Sonic verifier key and of
4096 points, and SonicKZG10 check / batch_check at degree 2^--sonic-log (hiding, one degree bound).  Prints the card's name
and power limit first.  (tests/perf/pairing_bench.py times the plain path alone.)
Run on the GPU box:  python tests/perf/pairing_bench.py > perf_out/pairing_prepared_bench.jsonl"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import pkgload  # noqa: E402

pc = pkgload.load()
from oracle import orc, pyref  # noqa: E402
from tests import g2_cases as gc  # noqa: E402
from tests import util  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--counts", default="1,256,16384")
    ap.add_argument("--ks", default="2,3,5,21")
    ap.add_argument("--sonic-log", type=int, default=20)
    a = ap.parse_args()
    counts = [int(c) for c in a.counts.split(",")]
    ks = [int(k) for k in a.ks.split(",")]
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"card": card.stdout.strip()}), flush=True)
    eng = pc.Engine(0)
    for cname in gc.PAIRING:
        C = pyref.Curve(cname)
        npts = 4096                                   # distinct points, tiled to the largest shape
        h_xy, _ = gc.to_limbs(cname, [gc.generator(cname)])
        g1 = eng.fixed_base_mul(C.id, orc.g1_generator(C.id), util.rand_fr(cname, npts, 1, mont=False))
        g2 = eng.g2_fixed_base_mul(gc.group(pc, cname), h_xy[0], util.rand_fr(cname, npts, 2, mont=False))
        pairs = max(counts) * max(ks)
        reps = -(-pairs // npts)
        d1 = torch.from_numpy(np.tile(g1, (reps, 1))[:pairs].reshape(-1).view(np.int64)).cuda()
        d2 = torch.from_numpy(np.tile(g2, (reps, 1))[:pairs].reshape(-1).view(np.int64)).cuda()
        prep = eng.g2_prepare(C.id, g2)
        q_index = np.tile(np.arange(npts, dtype=np.uint32), reps)[:pairs]
        for k in ks:
            for count in counts:
                calls = {
                    "plain": lambda: eng.multi_pairing(C.id, d1.data_ptr(), d2.data_ptr(), k, flags=pc.DEVICE_PTRS, count=count),
                    "prepared": lambda: eng.multi_pairing_prepared(C.id, d1.data_ptr(), prep, q_index[:k * count], k,
                                                                   flags=pc.DEVICE_PTRS, count=count)}
                ms, dev = {p: [] for p in calls}, {p: [0.0, 0] for p in calls}
                for call in calls.values():
                    call()
                for _ in range(a.reps):
                    for path, call in calls.items():
                        eng.profile_enable(True)
                        torch.cuda.synchronize()
                        t0 = time.perf_counter()
                        call()
                        ms[path].append((time.perf_counter() - t0) * 1e3)
                        d_ms, n = eng.profile_get(17)
                        eng.profile_enable(False)
                        dev[path][0] += d_ms
                        dev[path][1] += n
                for path in calls:
                    med = statistics.median(ms[path])
                    print(json.dumps({"curve": cname, "path": path, "k": k, "count": count, "ms_median": round(med, 3),
                                      "ms_min": round(min(ms[path]), 3), "ms_max": round(max(ms[path]), 3), "runs": len(ms[path]),
                                      "stage17_ms_per_call": round(dev[path][0] / max(dev[path][1], 1), 3),
                                      "equations_per_s": round(count / (med * 1e-3), 1)}), flush=True)
        prep.release()
        for n in (4, npts):
            eng.g2_prepare(C.id, g2[:n]).release()                 # warm-up
            t0 = time.perf_counter()
            eng.g2_prepare(C.id, g2[:n]).release()
            print(json.dumps({"curve": cname, "g2_prepare_points": n, "ms": round((time.perf_counter() - t0) * 1e3, 3)}), flush=True)
        sonic(eng, cname, a.sonic_log)
    eng.close()


def sonic(eng, cname, lg):
    """SonicKZG10 check and batch_check (two points) at degree 2^lg with hiding and one degree bound, keys from a known beta"""
    from poly_commit_b200 import sonic_pc
    from tests.test_sonic_pc import SonicKeys
    n, C = 1 << lg, pyref.Curve(cname)
    t0 = time.perf_counter()
    keys = SonicKeys(eng, pc, cname, n, n, 3, [n // 2], seed=5)
    t_keys = time.perf_counter() - t0
    polys = [(util.rand_fr_fast(cname, n, 6), None), (util.rand_fr_fast(cname, n // 2, 7), n // 2)]
    rands = [util.rand_fr(cname, 4, 8, mont=True), util.rand_fr(cname, 3, 9, mont=True)]
    x, y = util.rand_fr(cname, 2, 10, mont=True)
    comms, vals, proof, chals = keys.prove(polys, rands, x, 11)
    query_set = [("a", ("x", x)), ("b", ("x", x)), ("b", ("y", y))]
    ch = list(util.rand_fr(cname, 3, 12, mont=True))
    pd = dict(zip("ab", polys))
    proofs = sonic_pc.batch_open(keys.ck, pd, query_set, ch, dict(zip("ab", rands)))
    pts = dict(x=x, y=y)
    evals = {(lb, pl): keys.value(pd[lb][0], pts[pl]) for lb, (pl, _) in query_set}
    rnd = np.stack([util.fr_const(cname, 1), util.rand_fr(cname, 1, 13, mont=True)[0]])
    runs = {"check": lambda: sonic_pc.check(eng, C.id, keys.vk, comms, x, vals, proof, chals),
            "batch_check": lambda: sonic_pc.batch_check(eng, C.id, keys.vk, dict(zip("ab", comms)), query_set, evals, proofs, ch, rnd)}
    for name, f in runs.items():
        assert f()
        ms = []
        for _ in range(3):
            t0 = time.perf_counter()
            assert f()
            ms.append((time.perf_counter() - t0) * 1e3)
        print(json.dumps({"curve": cname, "sonic": name, "degree": n, "ms_median": round(statistics.median(ms), 3),
                          "ms_min": round(min(ms), 3), "ms_max": round(max(ms), 3), "key_setup_s": round(t_keys, 1)}), flush=True)


if __name__ == "__main__":
    main()
