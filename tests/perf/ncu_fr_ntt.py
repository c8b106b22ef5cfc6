#!/usr/bin/env python3
"""Driver for one ncu capture of the Fr-vector kernels and the NTT at the benchmark's sizes (BLS12-381 Fr, device-resident):
fr_axpy / fr_from_mont / fr_inner_product / fr_div_linear (one-pass, 2^20) and the four-step NTT (2^20: both block passes).
  ncu --set full --clock-control none --import-source on --kernel-name-base demangled \
      -k regex:"NttBlockBody|DivTileBody|FrAxpyBody|FrFromMontBody|IpPartialBody" -c 12 -o perf_out/fr_ntt python tests/perf/ncu_fr_ntt.py"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import numpy as np
import torch

import pkgload

pc = pkgload.load()
from poly_commit_b200 import params  # noqa: E402


def main():
    eng = pc.Engine(0)
    cid = pc.BLS12_381
    n = 1 << 20
    x = torch.from_numpy(params.random_fr(cid, n, 1).view(np.int64)).cuda()
    y = torch.from_numpy(params.random_fr(cid, n, 2).view(np.int64)).cuda()
    q = torch.empty_like(x)
    c = params.random_fr(cid, 1, 3)[0]
    z = params.random_fr(cid, 1, 4)[0]
    F = pc.DEVICE_PTRS
    for _ in range(2):   # the second round of launches is the warm one
        eng.fr_axpy(cid, y.data_ptr(), c, x.data_ptr(), n=n, flags=F)
        eng.fr_from_mont(cid, x.data_ptr(), n=n, flags=F, out=q.data_ptr())
        eng.fr_inner_product(cid, x.data_ptr(), y.data_ptr(), n=n, flags=F)
        eng.fr_div_linear(cid, x.data_ptr(), z, n=n, flags=F, q=q.data_ptr())
        eng.ntt(cid, x.data_ptr(), 20, n_in=n, flags=F, out=q.data_ptr())
    torch.cuda.synchronize()


if __name__ == "__main__":
    main()
