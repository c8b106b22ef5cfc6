#!/usr/bin/env python3
"""Per-kernel device timings (CUDA events on the launching stream, inputs resident in HBM, 3 warm-ups,
working sets larger than L2 or rotated) for the members of the path other than the headline step:
the HBM-bound Fr kernels, the NTT, the MSM variants and the Hyrax / IPA batches.  Prints one JSON line per
kernel with the algorithmic bytes of SURVEY.md section 8d and the achieved fraction of the measured HBM peak.
Run on the GPU box:  python tests/perf/kernel_bench.py > perf_out/kernel_bench.jsonl"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import numpy as np
import torch

import pkgload

pc = pkgload.load()
from oracle import orc, pyref  # noqa: E402  (SRS scalar powers only)
from tests import util  # noqa: E402


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


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int64)).cuda()


def main():
    eng = pc.Engine(0)
    eng.set_stream(torch.cuda.current_stream().cuda_stream)
    P = peak()
    out = []

    def report(name, ms, algo_bytes, extra=None):
        gbs = algo_bytes / 1e9 / (ms / 1e3)
        d = {"kernel": name, "ms": round(ms, 4), "algorithmic_bytes": algo_bytes, "achieved_GBps": round(gbs, 1),
             "hbm_peak_GBps": P, "frac_of_measured_hbm": round(gbs / P, 4)}
        if extra:
            d.update(extra)
        print(json.dumps(d), flush=True)

    cname = "bls12_381"
    C = pyref.Curve(cname)
    logn = 22  # 2^22 x 32 B = 134 MB per vector: larger than the 50 MB L2
    n = 1 << logn
    x, y = dev(util.rand_fr_fast(cname, n, 1)), dev(util.rand_fr_fast(cname, n, 2))
    q = torch.empty_like(x)
    cfac = util.rand_fr(cname, 1, 3, mont=True)[0]
    z = util.rand_fr(cname, 1, 4, mont=True)[0]
    F = pc.DEVICE_PTRS
    report("fr_axpy (y += c*x), 2^22", timeit(lambda: eng.fr_axpy(C.id, y.data_ptr(), cfac, x.data_ptr(), n=n, flags=F)), 96 * n)
    report("fr_from_mont, 2^22", timeit(lambda: eng.fr_from_mont(C.id, x.data_ptr(), n=n, flags=F, out=q.data_ptr())), 64 * n)
    report("fr_div_linear (p/(X-z)), 2^22", timeit(lambda: eng.fr_div_linear(C.id, x.data_ptr(), z, n=n, flags=F, q=q.data_ptr())), 64 * n)
    report("fr_inner_product, 2^22", timeit(lambda: eng.fr_inner_product(C.id, x.data_ptr(), y.data_ptr(), n=n, flags=F)), 64 * n)
    nb = 1 << 20   # the benchmark's polynomial size: the one-pass division (tiles + decoupled look-back) runs up to 2^21 coefficients
    report("fr_div_linear (p/(X-z)), 2^20 (one pass)", timeit(lambda: eng.fr_div_linear(C.id, x.data_ptr(), z, n=nb, flags=F, q=q.data_ptr())), 64 * nb,
           {"note": "2 products per coefficient + 8 per thread: multiply-bound (fmaheavy 40 %), not HBM-bound"})
    report("fr_inner_product, 2^20", timeit(lambda: eng.fr_inner_product(C.id, x.data_ptr(), y.data_ptr(), n=nb, flags=F)), 64 * nb)
    for ln in (20, 22):
        m = 1 << ln
        report(f"ntt forward, 2^{ln}", timeit(lambda: eng.ntt(C.id, x.data_ptr(), ln, n_in=m, flags=F, out=q.data_ptr())), 64 * m,
               {"note": "(N/2)log2(N) - 7N/8 + N (2N beyond 2^20) modmuls; two passes over HBM"})
    del y
    # MSM variants at 2^20
    nm = (1 << 20) + 1
    beta = util.rand_fr(cname, 1, 1001, mont=True)[0]
    pows = dev(orc.fr_powers_canonical(C.id, beta, nm))
    bases = torch.empty((nm, 12), dtype=torch.int64, device="cuda")
    eng.fixed_base_mul(C.id, orc.g1_generator(C.id), pows.data_ptr(), n=nm, flags=F, out=bases.data_ptr())
    for name, flags in (("msm 2^20 window-folded tables (S=1)", pc.SRS_PRECOMPUTE), ("msm 2^20 raw bases (S=16)", 0)):
        srs = eng.srs_register(C.id, bases.data_ptr(), n=nm, flags=F | flags)
        ms = timeit(lambda: eng.msm(srs, x.data_ptr(), n=nm, flags=F | pc.SCALARS_MONT), reps=5)
        report(name, ms, 128 * nm, {"scalar_mults_per_s": round(nm / (ms / 1e3))})
        srs.release()
    # BASELINE.md second row: "witness-like" scalars (50 % zero / 25 % < 2^16 / 25 % uniform), and repeated small constants
    srs = eng.srs_register(C.id, bases.data_ptr(), n=nm, flags=F | pc.SRS_PRECOMPUTE)
    g = util.rng(3)
    w = util.rand_fr(cname, nm, seed=3, mont=False)
    kind = g.integers(0, 4, size=nm)
    w[kind < 2] = 0
    small = kind == 2
    w[small, 1:] = 0
    w[small, 0] &= np.uint64(0xFFFF)
    dw = dev(w)
    ms = timeit(lambda: eng.msm(srs, dw.data_ptr(), n=nm, flags=F), reps=5)
    report("msm 2^20 witness-like scalars (50% zero, 25% < 2^16, 25% uniform)", ms, 128 * nm, {"scalar_mults_per_s": round(nm / (ms / 1e3))})
    w2 = util.rand_fr(cname, nm, seed=4, mont=False)
    kind = g.integers(0, 10, size=nm)
    w2[kind < 3] = C.fr_to_limbs([1], False)[0]
    w2[(kind >= 3) & (kind < 5)] = C.fr_to_limbs([C.r - 1], False)[0]
    dw2 = dev(w2)
    ms = timeit(lambda: eng.msm(srs, dw2.data_ptr(), n=nm, flags=F), reps=5)
    report("msm 2^20 repeated scalars (30% = 1, 20% = -1, 50% uniform): heavy buckets", ms, 128 * nm, {"scalar_mults_per_s": round(nm / (ms / 1e3))})
    srs.release(); del dw, dw2
    # cfg5 shape: batch of 8 degree-2^22 commits over one SRS (what each of 8 GPUs does for the 64-polynomial batch)
    n5 = (1 << 22) + 1
    pows5 = dev(orc.fr_powers_canonical(C.id, beta, n5))
    bases5 = torch.empty((n5, 12), dtype=torch.int64, device="cuda")
    eng.fixed_base_mul(C.id, orc.g1_generator(C.id), pows5.data_ptr(), n=n5, flags=F, out=bases5.data_ptr())
    srs5 = eng.srs_register(C.id, bases5.data_ptr(), n=n5, flags=F | pc.SRS_PRECOMPUTE)
    polys5 = [dev(util.rand_fr_fast(cname, n5, 40 + i)) for i in range(8)]
    ms = timeit(lambda: eng.kzg_commit_batch(srs5, [(p.data_ptr(), n5) for p in polys5], flags=F), reps=2, warm=1)
    report("cfg5 per-GPU share: 8 x KZG commit, degree 2^22, BLS12-381 (pcgpu_kzg_commit_batch)", ms, 8 * 128 * n5,
           {"polys_per_s": round(8 / (ms / 1e3), 2), "scalar_mults_per_s": round(8 * n5 / (ms / 1e3))})
    srs5.release(); del polys5, bases5, pows5
    # Hyrax cfg4: 2^11 rows x (2^11 + 1) over one com_key, BN254
    cn = "bn254"
    C2 = pyref.Curve(cn)
    dim = 1 << 11
    pows2 = dev(orc.fr_powers_canonical(C2.id, util.rand_fr(cn, 1, 5, mont=True)[0], dim + 1))
    b2 = torch.empty((dim + 1, 8), dtype=torch.int64, device="cuda")
    eng.fixed_base_mul(C2.id, orc.g1_generator(C2.id), pows2.data_ptr(), n=dim + 1, flags=F, out=b2.data_ptr())
    srs2 = eng.srs_register(C2.id, b2.data_ptr(), n=dim + 1, flags=F | pc.SRS_COMB)
    mat = dev(util.rand_fr_fast(cn, dim * (dim + 1), 6))
    ms = timeit(lambda: eng.msm_batch(srs2, mat.data_ptr(), dim + 1, dim, flags=F | pc.SCALARS_MONT), reps=3, warm=1)
    report("hyrax commit rows (cfg4): 2^11 MSMs x (2^11+1), BN254, fixed-base comb (window chosen from free device memory)", ms, 64 * (dim + 1) + 32 * dim * (dim + 1),
           {"scalar_mults_per_s": round(dim * (dim + 1) / (ms / 1e3))})
    del mat
    # Ligero commit of a 2^20-coefficient polynomial (BLS12-381 Fr, rho_inv = 4): row NTTs + column hashes + Merkle tree, device-resident
    from poly_commit_b200 import linear_codes
    n_rows, n_cols = linear_codes.compute_dimensions(C.id, 128, 4, 1 << 20)
    log_ext = max(1, (n_cols * 4 - 1).bit_length())
    N = 1 << log_ext
    m = dev(util.rand_fr_fast(cname, n_rows * n_cols, 8))
    ext = torch.empty((n_rows, N, 4), dtype=torch.int64, device="cuda")
    leaves = torch.empty((N, 32), dtype=torch.uint8, device="cuda")
    nodes = torch.empty((N - 1, 32), dtype=torch.uint8, device="cuda")
    fused = lambda: eng.lincode_commit(C.id, m.data_ptr(), log_ext, n_rows=n_rows, n_cols=n_cols, flags=F, out_ext=ext.data_ptr(),
                                       out_leaves=leaves.data_ptr(), out_nodes=nodes.data_ptr())
    ms = timeit(fused, reps=5)
    report(f"ligero commit 2^20 coeffs ({n_rows} x {n_cols} -> x {N}): row NTTs + Blake2s columns + SHA-256 tree", ms,
           32 * n_rows * n_cols + 2 * 32 * n_rows * N + 32 * N, {"note": "algorithmic: read mat, write + read ext_mat, write leaves"})
    ms = timeit(lambda: eng.lincode_hash_columns(C.id, ext.data_ptr(), n_rows=n_rows, n_cols=N, flags=F, out=leaves.data_ptr()), reps=5)
    report(f"column hashes alone (Blake2s over {n_rows}-element columns, {N} columns)", ms, 32 * n_rows * N + 32 * N)
    ms = timeit(lambda: eng.ntt_batch_device(C.id, m.data_ptr(), n_cols, n_rows, log_ext, ext.data_ptr()) if hasattr(eng, "ntt_batch_device") else None, reps=1, warm=0)
    eng.close()


if __name__ == "__main__":
    main()
