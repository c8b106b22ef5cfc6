#!/usr/bin/env python3
"""Driver for one ncu capture of the kernels added late in round 1: MsmSmallBody (2^10 terms), G1DecodeBody (2^16 compressed
BLS12-381 points, validated), G1FoldGlvBody (2^14-point Pallas fold), NttBlockBody batched (1024 rows of 2^11).
  ncu --set full --clock-control none --import-source on --kernel-name-base demangled \
      -k regex:"MsmSmallBody|G1DecodeBody|G1FoldGlvBody|NttBlockBody" -c 8 -o perf_out/new_kernels python tests/perf/ncu_new_kernels.py"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import numpy as np
import pkgload
pc = pkgload.load()
from poly_commit_b200 import params, ipa_pc


def main():
    eng = pc.Engine(0)
    cid = pc.BLS12_381
    n = 1 << 16
    g = eng.fixed_base_mul(cid, params.g1_generator(cid), params.random_fr(cid, n, 1))
    srs = eng.srs_register(cid, g[:1024])
    eng.msm(srs, params.random_fr(cid, 1024, 2), flags=pc.SCALARS_MONT)                     # MsmSmallBody
    blob = eng.g1_serialize(cid, g, None, True)
    eng.g1_deserialize(cid, blob, n, True, True)                                            # G1DecodeBody
    pid = pc.PALLAS
    m = 1 << 15
    key = eng.fixed_base_mul(pid, params.g1_generator(pid), params.random_fr(pid, m, 3))
    st = eng.ipa_begin(pid, key, params.random_fr(pid, m, 4), params.random_fr(pid, 1, 5)[0])
    c = 0x1234567890abcdef1234567890abcdef1234567890abcdef1234567890abcdef % params.FR_MODULUS[pid]
    eng.ipa_round_fold(st, params.fr_mont(pid, c), params.fr_mont(pid, pow(c, -1, params.FR_MODULUS[pid])))   # G1FoldGlvBody
    rows = params.random_fr(cid, 1024 * 1024, 6).reshape(1024, 1024, 4)
    eng.ntt_batch(cid, rows, 11)                                                            # NttBlockBody, 1024 rows


if __name__ == "__main__":
    main()
