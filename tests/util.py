"""Shared helpers for the parity tests: seeded synthetic inputs in the ABI's packed layout."""
import os

import numpy as np

from oracle import orc, pyref

CURVE_NAMES = ["bls12_381", "bn254", "pallas"]
_SRS_CACHE = {}


def rng(seed):
    return np.random.default_rng(seed)


def on_gpu(eng):
    """True for the CUDA library, False for the host-emulated one (tests/host_emul)"""
    return os.path.basename(eng.lib._name) != "libpcgpu_hostcheck.so"


def dev_ptr(eng, a):
    """(pointer, owner) of `a` for a DEVICE_PTRS call: the host array itself under host emulation, a CUDA copy on the GPU
    (pageable host memory is not device-accessible in general)"""
    if not on_gpu(eng):
        return a.ctypes.data, a
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a).reshape(-1).view(np.uint8)).cuda()
    torch.cuda.synchronize()
    return t.data_ptr(), t


def rand_fr_ints(curve, n, seed):
    """n uniform integers in [0, r)."""
    C = pyref.Curve(curve)
    g = rng(seed)
    out = []
    while len(out) < n:
        raw = g.integers(0, 1 << 63, size=(n, 5), dtype=np.uint64)
        for row in raw:
            v = 0
            for x in row:
                v = (v << 63) | int(x)
            v &= (1 << 256) - 1
            if v < C.r:
                out.append(v)
                if len(out) == n:
                    break
    return out


def _uniform_below_r(C, n, g):
    """(n, 4) uint64, uniform integers in [0, r): vectorised rejection sampling on 255/254-bit draws."""
    top_bits = C.r.bit_length() - 192
    r_l = [np.uint64((C.r >> (64 * j)) & (2**64 - 1)) for j in range(4)]
    out = np.empty((n, 4), dtype=np.uint64)
    todo = np.arange(n)
    while todo.size:
        a = g.integers(0, 1 << 64, size=(todo.size, 4), dtype=np.uint64)
        a[:, 3] &= np.uint64((1 << top_bits) - 1)
        lt = np.zeros(todo.size, dtype=bool)
        eq = np.ones(todo.size, dtype=bool)
        for j in (3, 2, 1, 0):
            lt |= eq & (a[:, j] < r_l[j])
            eq &= a[:, j] == r_l[j]
        out[todo[lt]] = a[lt]
        todo = todo[~lt]
    return out


def rand_fr(curve, n, seed, mont):
    """(n, 4) uint64 uniform field elements: canonical integers (mont=False) or Montgomery form (mont=True;
    converted through the oracle so that the canonical values are the seeded draws)."""
    C = pyref.Curve(curve)
    arr = _uniform_below_r(C, n, rng(seed))
    if mont and n:
        arr = orc.field_unop("orc_fr_to_mont", C.id, arr)
    return arr


def rand_fr_fast(curve, n, seed):
    """(n, 4) uint64 uniform field elements in Montgomery form: the uniform draw IS the Montgomery
    representation (x -> x*R^-1 is a bijection of Z_r), so no conversion pass is needed at 2^20+ sizes."""
    return _uniform_below_r(pyref.Curve(curve), n, rng(seed))


def fr_const(curve, value, mont=True):
    C = pyref.Curve(curve)
    return C.fr_to_limbs([value], mont)[0]


def synthetic_srs(curve, n, seed=1):
    """powers_of_g: P_i = beta^i * G (affine Montgomery, (n, 2*nq) uint64) via the oracle's fixed-base
    batch multiplication -- what KZG10::setup computes (kzg10/mod.rs:66-86) with beta from a seeded PRNG."""
    key = (curve, n, seed)
    if key not in _SRS_CACHE:
        C = pyref.Curve(curve)
        beta = rand_fr(curve, 1, 1000 + seed, mont=True)[0]
        pows = orc.fr_powers_canonical(C.id, beta, n)
        xy, inf = orc.fixed_base_batch_mul(C.id, orc.g1_generator(C.id), pows)
        assert not inf.any()
        _SRS_CACHE[key] = xy
    return _SRS_CACHE[key]


def random_points(curve, n, seed):
    """n points k_i * G for seeded random k_i (not a power sequence)."""
    C = pyref.Curve(curve)
    ks = rand_fr(curve, n, 2000 + seed, mont=False)
    xy, inf = orc.fixed_base_batch_mul(C.id, orc.g1_generator(C.id), ks)
    return xy
