#!/usr/bin/env python3
"""SRS ingestion timing on one GPU: pcgpu_g1_deserialize / pcgpu_g1_serialize at 2^20 points (BLS12-381, BN254, Pallas),
host buffers (copies inside the timed region) and device pointers (kernel + status read only).
  python tests/perf/wire_bench.py > perf_out/wire_bench.json"""
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
from oracle import orc, pyref  # noqa: E402
from tests import util  # noqa: E402


def timed(fn, reps=3):
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps


def main():
    eng = pc.Engine(0)
    logn = int(os.environ.get("WIRE_LOGN", "20"))
    n = 1 << logn
    res = {"n": n}
    for cname in ("bls12_381", "bn254", "pallas"):
        C = pyref.Curve(cname)
        beta = util.rand_fr(cname, 1, 1001, mont=True)[0]
        pows = orc.fr_powers_canonical(C.id, beta, n)
        g = eng.fixed_base_mul(C.id, orc.g1_generator(C.id), pows)
        row = {}
        for compressed in (True, False):
            tag = "compressed" if compressed else "uncompressed"
            blob = eng.g1_serialize(C.id, g, None, compressed)
            back, inf = eng.g1_deserialize(C.id, blob, n, compressed, True)
            assert (back == g).all() and not inf.any()
            row[f"serialize_{tag}_ms"] = round(timed(lambda: eng.g1_serialize(C.id, g, None, compressed)) * 1e3, 2)
            for validate in (True, False):
                dt = timed(lambda: eng.g1_deserialize(C.id, blob, n, compressed, validate))
                row[f"deserialize_{tag}_{'validate' if validate else 'novalidate'}_ms"] = round(dt * 1e3, 2)
            # device-resident: bytes, points and infinity flags stay in HBM
            d_blob = torch.from_numpy(blob).cuda()
            d_xy = torch.empty((n, g.shape[1]), dtype=torch.int64, device="cuda")
            d_inf = torch.empty(n, dtype=torch.uint8, device="cuda")
            torch.cuda.synchronize()
            import ctypes
            bad, reason = ctypes.c_size_t(0), ctypes.c_int(0)
            flags = (pc.binding.WIRE_COMPRESSED if compressed else 0) | pc.binding.DEVICE_PTRS

            def dev_call():
                rc = eng.lib.pcgpu_g1_deserialize(eng.ctx, C.id, ctypes.c_void_p(d_blob.data_ptr()), n, flags,
                                                  ctypes.c_void_p(d_xy.data_ptr()), ctypes.c_void_p(d_inf.data_ptr()),
                                                  ctypes.byref(bad), ctypes.byref(reason))
                assert rc == 0
            dt = timed(dev_call)
            assert (d_xy.cpu().numpy().view(np.uint64) == g).all()
            row[f"deserialize_{tag}_validate_device_ms"] = round(dt * 1e3, 2)
            row[f"deserialize_{tag}_validate_device_points_per_s"] = round(n / dt)
        res[cname] = row
    print(json.dumps(res))


if __name__ == "__main__":
    main()
