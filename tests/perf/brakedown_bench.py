#!/usr/bin/env python3
"""Device timing of the Brakedown commit of a 2^22-variable multilinear polynomial (BN254 Fr, default BrakedownPCParams,
Blake2s columns, SHA-256 tree), inputs and outputs resident in HBM, CUDA events on the launching stream, 3 warm-ups.
The split between the sparse encode and the hashes + tree comes from profile stages 15 and 14.  Prints the card's name and
power limit, then one JSON line in the format of kernel_bench.py.
Run on the GPU box:  python tests/perf/brakedown_bench.py > perf_out/brakedown_bench.jsonl"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import pkgload  # noqa: E402

pc = pkgload.load()
from oracle import pyref  # noqa: E402
from tests import brakedown_ref, util  # noqa: E402


def peak():
    try:
        return float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
    except Exception:
        return 3350.0   # H100 SXM data sheet (HBM3)


def timeit(fn, reps=10, warm=3):
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


def main():
    from poly_commit_b200 import linear_codes
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"card": card.stdout.strip()}), flush=True)
    eng = pc.Engine(0)
    eng.set_stream(torch.cuda.current_stream().cuda_stream)
    cn = "bn254"
    C = pyref.Curve(cn)
    p = linear_codes.brakedown_params(C.id, 1 << 22, brakedown_ref.u64_source(7))
    code = linear_codes.brakedown_register(eng, p)
    n, m, N = p["n"], p["m"], p["m_ext"]
    P = 1 << (N - 1).bit_length()
    mat = torch.from_numpy(util.rand_fr_fast(cn, n * m, 9).view("int64")).cuda()
    ext = torch.empty((n, N, 4), dtype=torch.int64, device="cuda")
    leaves = torch.empty((N, 32), dtype=torch.uint8, device="cuda")
    nodes = torch.empty((P - 1, 32), dtype=torch.uint8, device="cuda")
    fused = lambda: eng.brakedown_commit(code, mat.data_ptr(), n_rows=n, n_cols=m, flags=pc.DEVICE_PTRS, out_ext=ext.data_ptr(),
                                         out_leaves=leaves.data_ptr(), out_nodes=nodes.data_ptr())
    reps = 10
    ms = timeit(fused, reps=reps)
    eng.profile_enable(True)
    for _ in range(reps):
        fused()
    enc, hashes = eng.profile_get(15)[0] / reps, eng.profile_get(14)[0] / reps
    eng.profile_enable(False)
    nnz = sum(int(x[0][-1]) for x in p["a_mats"] + p["b_mats"])
    algo_bytes = 32 * n * m + 32 * nnz + 2 * 32 * n * N + 32 * N
    gbs = algo_bytes / 1e9 / (ms / 1e3)
    print(json.dumps({"kernel": f"brakedown commit 2^22 vars, BN254 ({n} x {m} -> x {N}, {len(p['a_dims'])} levels): sparse encode + "
                                f"Blake2s columns + SHA-256 tree",
                      "ms": round(ms, 4), "algorithmic_bytes": algo_bytes, "achieved_GBps": round(gbs, 1), "hbm_peak_GBps": peak(),
                      "frac_of_measured_hbm": round(gbs / peak(), 4), "encode_ms": round(enc, 4), "hashes_tree_ms": round(hashes, 4),
                      "nonzeros": nnz, "fr_muladds": nnz * n,
                      "note": "algorithmic: read mat and the matrices, write + read ext_mat, write leaves"}), flush=True)
    code.release()
    eng.close()


if __name__ == "__main__":
    main()
