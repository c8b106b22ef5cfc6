#!/usr/bin/env python3
"""Randomised parity sweep on one H100: the CUDA library through its C ABI against the C oracle on randomly drawn shapes that
the fixed pytest parameters do not enumerate -- MSM (three curves; raw and window-folded tables; canonical and Montgomery
scalars; base offsets; scalar mixtures of zeros / +-1 / r-1 / tiny / uniform; sizes across the small-path, split and bucket-pipeline
boundaries), division (both paths), NTT (forward / inverse, zero-padded), inner product, axpy, KZG commit + open with and
without hiding.  Bit-exact or it aborts.  python tests/perf/fuzz_gpu.py [cases] [seed] > perf_out/fuzz_gpu.log"""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import numpy as np

import pkgload

pc = pkgload.load()
from oracle import orc, pyref  # noqa: E402
from tests import util  # noqa: E402

CURVES = ["bls12_381", "bn254", "pallas"]
SIZES = [0, 1, 2, 3, 31, 33, 255, 511, 512, 513, 1000, 2047, 4095, 4096, 4097, 5000, 8191, 8193, 12345, 20000, 40000, 65537]


def mixed_scalars(C, cname, n, g, mont):
    s = util.rand_fr(cname, n, seed=int(g.integers(1 << 30)), mont=False).copy() if n else np.zeros((0, 4), dtype=np.uint64)
    kind = g.integers(0, 8, size=n)
    one = C.fr_to_limbs([1], False)[0]
    rm1 = C.fr_to_limbs([C.r - 1], False)[0]
    s[kind == 0] = 0
    s[kind == 1] = one
    s[kind == 2] = rm1
    small = kind == 3
    s[small, 1:] = 0
    s[small, 0] &= np.uint64(0xFFFF)
    if mont:
        ints = C.fr_from_limbs(s, False)
        return C.fr_to_limbs(ints, True), s
    return s, s


def main():
    cases = int(sys.argv[1]) if len(sys.argv) > 1 else 120
    seed = int(sys.argv[2]) if len(sys.argv) > 2 else 20260924
    g = np.random.default_rng(seed)
    eng = pc.Engine(0, lib_path=os.environ.get("FUZZ_LIB"))   # FUZZ_LIB: the host-emulation harness, to dry-run the script without a GPU
    if os.environ.get("FUZZ_MAXN"):
        SIZES[:] = [v for v in SIZES if v <= int(os.environ["FUZZ_MAXN"])]
    nmax = max(SIZES) + 64
    bases = {c: util.synthetic_srs(c, 6000, seed=7) for c in CURVES}          # oracle-built bases for the small / medium cases
    big = {}
    counts = {"msm": 0, "div": 0, "ntt": 0, "fr": 0, "kzg": 0}
    t0 = time.time()
    for it in range(cases):
        cname = CURVES[int(g.integers(3))]
        C = pyref.Curve(cname)
        what = ["msm", "msm", "msm", "div", "ntt", "fr", "kzg"][int(g.integers(7))]
        if what == "msm":
            n = int(SIZES[int(g.integers(len(SIZES)))])
            if n > 6000:
                if cname not in big:      # device-built bases (fixed-base kernel), spot-checked in the pytest suite
                    beta = util.rand_fr(cname, 1, 555, mont=True)[0]
                    big[cname] = eng.fixed_base_mul(C.id, orc.g1_generator(C.id), orc.fr_powers_canonical(C.id, beta, nmax))
                b = big[cname]
            else:
                b = bases[cname]
            off = int(g.integers(0, 5)) if n + 5 <= b.shape[0] else 0
            mont = bool(g.integers(2))
            pre = bool(g.integers(2))
            sc, canon = mixed_scalars(C, cname, n, g, mont)
            srs = eng.srs_register(C.id, b[: off + n + int(g.integers(0, 3))] if n else b[:4], flags=pc.SRS_PRECOMPUTE if pre else 0)
            got = eng.msm(srs, sc, n=n, base_offset=off, flags=pc.SCALARS_MONT if mont else 0)
            exp = orc.msm(C.id, b[off:off + n], canon, n=n) if n else (np.zeros_like(got[0]), 1)
            assert (got[0] == exp[0]).all() and got[1] == exp[1], ("msm", cname, n, off, mont, pre, it)
            srs.release()
        elif what == "div":
            n = int(g.integers(1, 30000))
            mode = ["tile", "tree"][int(g.integers(2))]
            os.environ["PCGPU_DIV_MODE"] = mode
            p = util.rand_fr_fast(cname, n, seed=int(g.integers(1 << 30)))
            z = util.rand_fr(cname, 1, seed=int(g.integers(1 << 30)), mont=True)[0]
            q, rem = eng.fr_div_linear(C.id, p, z)
            eq, erem = orc.fr_div_linear(C.id, p, z)
            assert (q == eq).all() and (rem == erem).all(), ("div", cname, n, mode, it)
            os.environ.pop("PCGPU_DIV_MODE", None)
        elif what == "ntt":
            logn = int(g.integers(1, 15))
            n_in = int(g.integers(1, (1 << logn) + 1))
            x = util.rand_fr_fast(cname, n_in, seed=int(g.integers(1 << 30)))
            got = eng.ntt(C.id, x, logn)
            assert (got == orc.fr_ntt(C.id, x, logn)).all(), ("ntt", cname, logn, n_in, it)
            back = eng.ntt(C.id, got, logn, inverse=True)
            assert (back[:n_in] == x).all() and not back[n_in:].any(), ("intt", cname, logn, n_in, it)
        elif what == "fr":
            n = int(g.integers(1, 50000))
            x = util.rand_fr_fast(cname, n, seed=int(g.integers(1 << 30)))
            y = util.rand_fr_fast(cname, n, seed=int(g.integers(1 << 30)))
            c = util.rand_fr(cname, 1, seed=int(g.integers(1 << 30)), mont=True)[0]
            assert (eng.fr_inner_product(C.id, x, y) == orc.fr_inner_product(C.id, x, y)).all(), ("ip", cname, n, it)
            assert (eng.fr_axpy(C.id, y, c, x) == orc.fr_axpy(C.id, y, c, x)).all(), ("axpy", cname, n, it)
        else:
            n = int(g.integers(1, 3000))
            nb = int(g.integers(0, 6))
            b = bases[cname]
            gam = util.synthetic_srs(cname, 8, seed=9)
            srs = eng.srs_register(C.id, b[: n + int(g.integers(0, 3))], flags=pc.SRS_PRECOMPUTE if g.integers(2) else 0)
            sg = eng.srs_register(C.id, gam)
            p = util.rand_fr_fast(cname, n, seed=int(g.integers(1 << 30)))
            blind = util.rand_fr_fast(cname, nb, seed=int(g.integers(1 << 30))) if nb else None
            z = util.rand_fr(cname, 1, seed=int(g.integers(1 << 30)), mont=True)[0]
            got = eng.kzg_commit(srs, p, powers_of_gamma_g=sg if nb else None, blind=blind)
            rc, exy, einf = orc.kzg_commit(C.id, b, p, gam if nb else None, blind)
            assert rc == 0 and (got[0] == exy).all() and got[1] == einf, ("commit", cname, n, nb, it)
            w = eng.kzg_open(srs, p, z, powers_of_gamma_g=sg if nb else None, blind=blind)
            rc, wxy, winf, rv = orc.kzg_open(C.id, b, p, z, gam if nb else None, blind)
            assert rc == 0 and (w[0] == wxy).all() and w[1] == winf, ("open", cname, n, nb, it)
            if nb:
                assert (w[2] == rv).all(), ("random_v", cname, n, nb, it)
            srs.release(); sg.release()
        counts[what] += 1
    print(json.dumps({"fuzz": "gpu vs oracle, bit-exact", "cases": cases, "seed": seed, "by_kind": counts, "seconds": round(time.time() - t0, 1), "ok": True}))


if __name__ == "__main__":
    main()
