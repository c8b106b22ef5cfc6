#!/usr/bin/env python3
"""Device timing of pcgpu_multi_pairing: equations per second at k = 2 (KZG10::check), 3 (SonicKZG10's check) and 21
(MultilinearPC::check at nv = 20) pairs per equation, for count = 1, 256 and 16384 equations per call, on BLS12-381 and BN254.
Points are honest group elements (fixed-base multiples of the generators), resident in HBM (DEVICE_PTRS); every call is
synchronous, so a host clock around it measures the whole call.  Each configuration is warmed up once and then timed `--reps`
times; the JSON lines give the median and the spread (min, max), and the stage-17 device time (CUDA events around the Miller
and final-exponentiation kernels) from the same calls.  Prints the card's name and power limit first.
Run on the GPU box:  python tests/perf/pairing_bench.py > perf_out/pairing_bench.jsonl"""
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
    ap.add_argument("--ks", default="2,3,21")
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
        for k in ks:
            for count in counts:
                def call():
                    eng.multi_pairing(C.id, d1.data_ptr(), d2.data_ptr(), k, flags=pc.DEVICE_PTRS, count=count)
                call()
                eng.profile_enable(True)
                ms = []
                for _ in range(a.reps):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    call()
                    ms.append((time.perf_counter() - t0) * 1e3)
                dev_ms, n = eng.profile_get(17)
                eng.profile_enable(False)
                med = statistics.median(ms)
                print(json.dumps({"curve": cname, "k": k, "count": count, "ms_median": round(med, 3), "ms_min": round(min(ms), 3),
                                  "ms_max": round(max(ms), 3), "runs": len(ms), "stage17_ms_per_call": round(dev_ms / max(n, 1), 3),
                                  "equations_per_s": round(count / (med * 1e-3), 1)}), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
