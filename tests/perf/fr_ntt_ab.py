#!/usr/bin/env python3
"""Quick timings of the Fr-vector kernels and the NTT (CUDA events, device-resident) under tuning knobs:
  python tests/perf/fr_ntt_ab.py [KNOB=v1,v2,...] > perf_out/fr_ntt_ab.jsonl      e.g. PCGPU_NTT_OCC=3,4"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import numpy as np
import torch

import pkgload

pc = pkgload.load()
from oracle import pyref  # noqa: E402
from tests import util  # noqa: E402


def timeit(fn, reps=20, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int64)).cuda()


def main():
    knob, values = None, [None]
    if len(sys.argv) > 1 and "=" in sys.argv[1]:
        knob, vs = sys.argv[1].split("=")
        values = vs.split(",")
    eng = pc.Engine(0)
    eng.set_stream(torch.cuda.current_stream().cuda_stream)
    cname = "bls12_381"
    C = pyref.Curve(cname)
    n = 1 << 22
    x, y = dev(util.rand_fr_fast(cname, n, 1)), dev(util.rand_fr_fast(cname, n, 2))
    q = torch.empty_like(x)
    z = util.rand_fr(cname, 1, 4, mont=True)[0]
    F = pc.DEVICE_PTRS
    for v in values:
        if knob:
            os.environ[knob] = v
        rec = {"knob": knob, "value": v}
        for ln in (16, 20, 22):
            m = 1 << ln
            rec[f"div_linear_2p{ln}_ms"] = round(timeit(lambda: eng.fr_div_linear(C.id, x.data_ptr(), z, n=m, flags=F, q=q.data_ptr())), 4)
            rec[f"inner_product_2p{ln}_ms"] = round(timeit(lambda: eng.fr_inner_product(C.id, x.data_ptr(), y.data_ptr(), n=m, flags=F)), 4)
        for ln in (10, 16, 20, 22):
            m = 1 << ln
            rec[f"ntt_2p{ln}_ms"] = round(timeit(lambda: eng.ntt(C.id, x.data_ptr(), ln, n_in=m, flags=F, out=q.data_ptr())), 4)
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
