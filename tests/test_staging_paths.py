"""Every entry point that stages its operands through the context's arena, called twice with the same values: once with host
arrays and once with PCGPU_DEVICE_PTRS (the caller's device buffers are read and written in place).  Both calls must return the
same code and bit-identical results, at n = 0, n = 1 and a few elements, on one error path per entry point, and with each
optional output of the fused commitments present or absent.  On the GPU the entry points outside the MSM pipeline must also
launch the same, pinned, number of kernels in both modes (test_gpu_msm_paths.py and test_comb_msm.py pin the MSM paths'
geometry through pcgpu_msm_last_geometry).

The calls go to the C ABI directly so that the two modes pass identical arguments apart from the pointers and the flag.  The same
case bodies run on the host-emulated library (CPU; a host array is a valid "device" pointer there) and, with -m gpu, on the
device (operands copied into CUDA tensors)."""
import ctypes

import numpy as np
import pytest

from oracle import pyref
from tests import brakedown_ref as bref
from tests import util

E_BADARG, E_LEN, E_RANGE, E_DEGREE, E_HIDING, E_INVALID = -3, -4, -5, -6, -7, -8
CN = "bn254"
CID = pyref.Curve(CN).id
NQ = 4           # Fq limbs of BN254
SRS_N = 8

# kernels launched by one call in either mode, keyed by case, as measured on an H100 before the staging helper existed.  The
# MSM-backed cases are not keyed: with device coefficients KZG10 trims trailing zeros on the device (FrLastNonzeroBody).
LAUNCHES = {
    "axpy/0": 0, "axpy/1": 1, "axpy/5": 1,
    "brakedown_commit/128/3/0000": 13, "brakedown_commit/128/3/0001": 13, "brakedown_commit/128/3/0010": 13,
    "brakedown_commit/128/3/0011": 13, "brakedown_commit/128/3/0100": 13, "brakedown_commit/128/3/0101": 13,
    "brakedown_commit/128/3/0110": 13, "brakedown_commit/128/3/0111": 13, "brakedown_commit/128/3/1000": 13,
    "brakedown_commit/128/3/1001": 13, "brakedown_commit/128/3/1010": 13, "brakedown_commit/128/3/1011": 13,
    "brakedown_commit/128/3/1100": 13, "brakedown_commit/128/3/1101": 13, "brakedown_commit/128/3/1110": 13,
    "brakedown_commit/128/3/1111": 13, "brakedown_commit/16/1/0000": 8, "brakedown_commit/16/1/0001": 8,
    "brakedown_commit/16/1/0010": 8, "brakedown_commit/16/1/0011": 8, "brakedown_commit/16/1/0100": 8,
    "brakedown_commit/16/1/0101": 8, "brakedown_commit/16/1/0110": 8, "brakedown_commit/16/1/0111": 8,
    "brakedown_commit/16/1/1000": 8, "brakedown_commit/16/1/1001": 8, "brakedown_commit/16/1/1010": 8,
    "brakedown_commit/16/1/1011": 8, "brakedown_commit/16/1/1100": 8, "brakedown_commit/16/1/1101": 8,
    "brakedown_commit/16/1/1110": 8, "brakedown_commit/16/1/1111": 8,
    "brakedown_encode/128/3": 5, "brakedown_encode/16/1": 3,
    "div/0": 0, "div/1": 2, "div/5": 2,
    "from_mont/0": 0, "from_mont/1": 1, "from_mont/5": 1,
    "g1_deserialize/0/0": 0, "g1_deserialize/0/1": 0, "g1_deserialize/1/0": 1, "g1_deserialize/1/1": 1, "g1_deserialize/4/0": 1,
    "g1_deserialize/4/1": 1,
    "g1_serialize/0/0/0": 0, "g1_serialize/0/0/1": 0, "g1_serialize/0/1/0": 0, "g1_serialize/0/1/1": 0, "g1_serialize/1/0/0": 1,
    "g1_serialize/1/0/1": 1, "g1_serialize/1/1/0": 1, "g1_serialize/1/1/1": 1, "g1_serialize/4/0/0": 1, "g1_serialize/4/0/1": 1,
    "g1_serialize/4/1/0": 1, "g1_serialize/4/1/1": 1,
    "hash_columns/0x4/0": 1, "hash_columns/0x4/1": 1, "hash_columns/1x1/0": 1, "hash_columns/1x1/1": 1, "hash_columns/2x0/0": 0,
    "hash_columns/2x0/1": 0, "hash_columns/3x5/0": 1, "hash_columns/3x5/1": 1,
    "ip/0": 2, "ip/1": 2, "ip/5": 2,
    "lincode_commit/1x0/2/0000": 4, "lincode_commit/1x0/2/0001": 4, "lincode_commit/1x0/2/0010": 4,
    "lincode_commit/1x0/2/0011": 4, "lincode_commit/1x0/2/0100": 4, "lincode_commit/1x0/2/0101": 4,
    "lincode_commit/1x0/2/0110": 4, "lincode_commit/1x0/2/0111": 4, "lincode_commit/1x0/2/1000": 4,
    "lincode_commit/1x0/2/1001": 4, "lincode_commit/1x0/2/1010": 4, "lincode_commit/1x0/2/1011": 4,
    "lincode_commit/1x0/2/1100": 4, "lincode_commit/1x0/2/1101": 4, "lincode_commit/1x0/2/1110": 4,
    "lincode_commit/1x0/2/1111": 4, "lincode_commit/2x3/3/0000": 5, "lincode_commit/2x3/3/0001": 5,
    "lincode_commit/2x3/3/0010": 5, "lincode_commit/2x3/3/0011": 5, "lincode_commit/2x3/3/0100": 5,
    "lincode_commit/2x3/3/0101": 5, "lincode_commit/2x3/3/0110": 5, "lincode_commit/2x3/3/0111": 5,
    "lincode_commit/2x3/3/1000": 5, "lincode_commit/2x3/3/1001": 5, "lincode_commit/2x3/3/1010": 5,
    "lincode_commit/2x3/3/1011": 5, "lincode_commit/2x3/3/1100": 5, "lincode_commit/2x3/3/1101": 5,
    "lincode_commit/2x3/3/1110": 5, "lincode_commit/2x3/3/1111": 5, "lincode_commit/3x1000/12/1111": 15,
    "merkle/1/00": 0, "merkle/1/01": 0, "merkle/1/10": 0, "merkle/1/11": 0, "merkle/2/00": 1, "merkle/2/01": 1,
    "merkle/2/10": 1, "merkle/2/11": 1, "merkle/5/00": 3, "merkle/5/01": 3, "merkle/5/10": 3, "merkle/5/11": 3,
    "merkle/8/00": 3, "merkle/8/01": 3, "merkle/8/10": 3, "merkle/8/11": 3,
    "mul/0": 0, "mul/1": 1, "mul/5": 1,
    "ntt/12/4000/0": 2, "ntt/12/4000/1": 2, "ntt/4/0/0": 1, "ntt/4/0/1": 1, "ntt/4/1/0": 1, "ntt/4/1/1": 1, "ntt/4/16/0": 1,
    "ntt/4/16/1": 1,
    "ntt_batch/12/100/2": 2, "ntt_batch/4/0/2": 1, "ntt_batch/4/16/3": 1, "ntt_batch/4/3/0": 0, "ntt_batch/4/5/1": 1,
    "row_mul/0x3": 1, "row_mul/1x1": 1, "row_mul/2x0": 0, "row_mul/3x4": 1,
    "sample_generators/0": 0, "sample_generators/1": 1, "sample_generators/3": 1,
    "sprs_row_mul/0/2/2": 1, "sprs_row_mul/3/4/2": 1, "sprs_row_mul/4/3/0": 0, "sprs_row_mul/5/2/1": 1,
}


@pytest.fixture(scope="module", params=["emul", pytest.param("gpu", marks=pytest.mark.gpu)])
def eng(request, pc):
    if request.param == "gpu":
        yield request.getfixturevalue("gpu_engine")
        return
    e = pc.Engine(0, lib_path=request.getfixturevalue("hostcheck_path"))
    yield e
    e.close()


class Operands:
    """the pointers of one call: host arrays, or (dev) copies the call may read and write in place"""

    def __init__(self, eng, pc, dev):
        self.eng, self.dev = eng, dev
        self.flags = pc.DEVICE_PTRS if dev else 0
        self.bufs = []          # (host template or None, owner)

    def _put(self, a, dev):
        flat = a.reshape(-1) if a.size else np.zeros(1, a.dtype)    # a valid, distinct pointer for empty operands too
        ptr, owner = util.dev_ptr(self.eng, flat) if dev else (flat.ctypes.data, flat)
        return ctypes.c_void_p(ptr), owner

    def inp(self, a):
        """an operand the call reads (a device copy with DEVICE_PTRS)"""
        ptr, owner = self._put(np.ascontiguousarray(a), self.dev)
        self.bufs.append((None, owner))
        return ptr

    def out(self, a, host=False):
        """an operand the call writes, starting from the contents of `a` (host=True: a host pointer in both modes)"""
        a = np.array(a)
        ptr, owner = self._put(a, self.dev and not host)
        self.bufs.append((a, owner))
        return ptr

    def results(self):
        res = []
        for a, owner in self.bufs:
            if a is None:
                continue
            if hasattr(owner, "cpu"):
                import torch
                torch.cuda.synchronize()
                owner = owner.cpu().numpy()
            res.append(np.ascontiguousarray(owner).view(a.dtype).reshape(-1)[:a.size].reshape(a.shape))
        return res


def both(eng, pc, call, key=None):
    """call(ops) -> rc with host operands and with device ones (after one unmeasured call that builds the context's cached
    tables); asserts equal codes and results, and on the GPU, when `key` is given, kernel counts equal to LAUNCHES[key] in
    both modes.  Returns (rc, results of the host call)."""
    call(Operands(eng, pc, False))
    runs = []
    for dev in (False, True):
        ops = Operands(eng, pc, dev)
        l0 = eng.launch_count()
        rc = call(ops)
        runs.append((rc, ops.results(), eng.launch_count() - l0))
    (rc_h, res_h, l_h), (rc_d, res_d, l_d) = runs
    assert rc_h == rc_d, (key, rc_h, rc_d)
    assert len(res_h) == len(res_d), key
    for i, (h, d) in enumerate(zip(res_h, res_d)):
        assert h.shape == d.shape and h.dtype == d.dtype and np.array_equal(h, d), (key, "result", i)
    if util.on_gpu(eng) and key is not None:
        assert l_h == l_d == LAUNCHES[key], (key, l_h, l_d, LAUNCHES[key])
    return rc_h, res_h


def fr(n, seed):
    return util.rand_fr_fast(CN, n, seed=seed)


def z4(n):
    return np.zeros((n, 4), dtype=np.uint64)


def canon_bad(n):
    """n canonical scalars, the last one equal to r (not reduced)"""
    s = util.rand_fr(CN, n, seed=77, mont=False)
    r = pyref.Curve(CN).r
    s[-1] = [(r >> (64 * j)) & (2**64 - 1) for j in range(4)]
    return s


# ---------------------------------------------------------------------------------------------------------------------------
# Fr vectors
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [0, 1, 5])
def test_fr_elementwise(eng, pc, n):
    L, ctx = eng.lib, eng.ctx
    a, b, y, c = fr(n, 1), fr(n, 2), fr(n, 3), fr(1, 4)
    both(eng, pc, lambda o: L.pcgpu_fr_from_mont(ctx, CID, o.inp(a), o.out(z4(n)), n, o.flags), f"from_mont/{n}")
    both(eng, pc, lambda o: L.pcgpu_fr_mul(ctx, CID, o.inp(a), o.inp(b), o.out(z4(n)), n, o.flags), f"mul/{n}")
    both(eng, pc, lambda o: L.pcgpu_fr_axpy(ctx, CID, o.out(y), o.out(c, host=True), o.inp(a), n, o.flags), f"axpy/{n}")
    both(eng, pc, lambda o: L.pcgpu_fr_div_linear(ctx, CID, o.inp(a), n, o.out(c, host=True), o.out(z4(max(n - 1, 0))),
                                                  o.out(z4(1), host=True), o.flags), f"div/{n}")
    both(eng, pc, lambda o: L.pcgpu_fr_inner_product(ctx, CID, o.inp(a), o.inp(b), n, o.out(z4(1), host=True), o.flags),
         f"ip/{n}")


def test_fr_elementwise_errors(eng, pc):
    L, ctx = eng.lib, eng.ctx
    a = fr(3, 5)
    for call in (lambda o: L.pcgpu_fr_from_mont(ctx, CID, None, o.out(z4(3)), 3, o.flags),
                 lambda o: L.pcgpu_fr_mul(ctx, CID, o.inp(a), None, o.out(z4(3)), 3, o.flags),
                 lambda o: L.pcgpu_fr_axpy(ctx, CID, o.out(a), None, o.inp(a), 3, o.flags),
                 lambda o: L.pcgpu_fr_div_linear(ctx, CID, o.inp(a), 3, None, o.out(z4(2)), None, o.flags),
                 lambda o: L.pcgpu_fr_inner_product(ctx, CID, o.inp(a), None, 3, o.out(z4(1), host=True), o.flags)):
        assert both(eng, pc, call)[0] == E_BADARG


@pytest.mark.parametrize("rows,cols", [(0, 3), (1, 1), (3, 4), (2, 0)])
def test_fr_row_mul(eng, pc, rows, cols):
    L, ctx = eng.lib, eng.ctx
    v, m = fr(rows, 6), fr(rows * cols, 7)
    rc, _ = both(eng, pc, lambda o: L.pcgpu_fr_row_mul(ctx, CID, o.inp(v), o.inp(m), rows, cols, o.out(z4(cols)), o.flags),
                 f"row_mul/{rows}x{cols}")
    assert rc == 0
    assert both(eng, pc, lambda o: L.pcgpu_fr_row_mul(ctx, CID, o.inp(v), None, rows, 2, o.out(z4(2)), o.flags))[0] == \
        (E_BADARG if rows else 0)


# ---------------------------------------------------------------------------------------------------------------------------
# NTT
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("logn,n_in", [(4, 0), (4, 1), (4, 16), (12, 4000)])
@pytest.mark.parametrize("inverse", [False, True])
def test_ntt(eng, pc, logn, n_in, inverse):
    L, ctx = eng.lib, eng.ctx
    f = pc.NTT_INVERSE if inverse else 0
    x = fr(n_in, 8)
    rc, _ = both(eng, pc, lambda o: L.pcgpu_ntt(ctx, CID, o.inp(x), n_in, logn, o.flags | f, o.out(z4(1 << logn))),
                 f"ntt/{logn}/{n_in}/{int(inverse)}")
    assert rc == 0


@pytest.mark.parametrize("logn,n_in,count", [(4, 0, 2), (4, 5, 1), (4, 16, 3), (12, 100, 2), (4, 3, 0)])
def test_ntt_batch(eng, pc, logn, n_in, count):
    L, ctx = eng.lib, eng.ctx
    x = fr(count * n_in, 9)
    rc, _ = both(eng, pc, lambda o: L.pcgpu_ntt_batch(ctx, CID, o.inp(x), n_in, count, logn, o.flags,
                                                      o.out(z4(count << logn))), f"ntt_batch/{logn}/{n_in}/{count}")
    assert rc == 0


def test_ntt_errors(eng, pc):
    L, ctx = eng.lib, eng.ctx
    x = fr(17, 10)
    assert both(eng, pc, lambda o: L.pcgpu_ntt(ctx, CID, o.inp(x), 17, 4, o.flags, o.out(z4(16))))[0] == E_LEN
    assert both(eng, pc, lambda o: L.pcgpu_ntt_batch(ctx, CID, o.inp(x), 17, 1, 4, o.flags, o.out(z4(16))))[0] == E_LEN


# ---------------------------------------------------------------------------------------------------------------------------
# column hashes, Merkle trees, Ligero / Brakedown commitments, sparse row products
# ---------------------------------------------------------------------------------------------------------------------------
def b32(n):
    return np.zeros((n, 32), dtype=np.uint8)


@pytest.mark.parametrize("rows,cols", [(0, 4), (1, 1), (3, 5), (2, 0)])
@pytest.mark.parametrize("hash", [0, 1])
def test_hash_columns(eng, pc, rows, cols, hash):
    L, ctx = eng.lib, eng.ctx
    m = fr(rows * cols, 11)
    rc, _ = both(eng, pc, lambda o: L.pcgpu_lincode_hash_columns(ctx, CID, o.inp(m), rows, cols, hash, o.flags, o.out(b32(cols))),
                 f"hash_columns/{rows}x{cols}/{hash}")
    assert rc == 0
    assert both(eng, pc, lambda o: L.pcgpu_lincode_hash_columns(ctx, CID, o.inp(m), rows, cols, 2, o.flags,
                                                                 o.out(b32(cols))))[0] == (E_BADARG if cols else 0)


@pytest.mark.parametrize("n_leaves", [1, 2, 5, 8])
def test_merkle_tree(eng, pc, n_leaves):
    L, ctx = eng.lib, eng.ctx
    leaves = util.rng(n_leaves).integers(0, 256, size=(n_leaves, 32), dtype=np.uint8)
    P = 1 << max(1, (n_leaves - 1).bit_length())
    for with_nodes in (False, True):
        for with_root in (False, True):
            rc, _ = both(eng, pc, lambda o: L.pcgpu_merkle_tree(ctx, o.inp(leaves), n_leaves, o.flags,
                                                                o.out(b32(P - 1)) if with_nodes else None,
                                                                o.out(b32(1), host=True) if with_root else None),
                         f"merkle/{n_leaves}/{int(with_nodes)}{int(with_root)}")
            assert rc == (E_BADARG if n_leaves < 2 else 0)


OPTIONAL = [(e, l, n, r) for e in (0, 1) for l in (0, 1) for n in (0, 1) for r in (0, 1)]


@pytest.mark.parametrize("rows,cols,log_ext", [(2, 3, 3), (1, 0, 2), (3, 1000, 12)])
def test_lincode_commit(eng, pc, rows, cols, log_ext):
    L, ctx = eng.lib, eng.ctx
    m = fr(rows * cols, 12)
    N = 1 << log_ext
    for want in (OPTIONAL if log_ext < 12 else [(1, 1, 1, 1)]):
        e, lv, nd, r = want
        rc, _ = both(eng, pc, lambda o: L.pcgpu_lincode_commit(
            ctx, CID, o.inp(m), rows, cols, log_ext, 1, o.flags, o.out(z4(rows * N)) if e else None, o.out(b32(N)) if lv else None,
            o.out(b32(N - 1)) if nd else None, o.out(b32(1), host=True) if r else None),
            f"lincode_commit/{rows}x{cols}/{log_ext}/{e}{lv}{nd}{r}")
        assert rc == 0
    assert both(eng, pc, lambda o: L.pcgpu_lincode_commit(ctx, CID, o.inp(fr(2 * (N + 1), 13)), 2, N + 1, log_ext, 1, o.flags,
                                                          o.out(z4(2 * N)), None, None, None))[0] == E_LEN


_CODES = {}


def brakedown_code(eng, poly_len):
    key = (id(eng), poly_len)
    if key not in _CODES:
        from poly_commit_b200 import linear_codes
        p = linear_codes.brakedown_params(CID, poly_len, bref.u64_source(7))
        _CODES[key] = (p, linear_codes.brakedown_register(eng, p))
    return _CODES[key]


@pytest.mark.parametrize("poly_len,n_rows", [(16, 1), (128, 3)])
def test_brakedown_commit(eng, pc, poly_len, n_rows):
    L, ctx = eng.lib, eng.ctx
    p, code = brakedown_code(eng, poly_len)
    m, N = p["m"], p["m_ext"]
    P = 1 << max(1, (N - 1).bit_length())
    mat = fr(n_rows * m, 14)
    for want in OPTIONAL:
        e, lv, nd, r = want
        rc, _ = both(eng, pc, lambda o: L.pcgpu_brakedown_commit(
            ctx, code.handle, o.inp(mat), n_rows, m, 0, o.flags, o.out(z4(n_rows * N)) if e else None,
            o.out(b32(N)) if lv else None, o.out(b32(P - 1)) if nd else None, o.out(b32(1), host=True) if r else None),
            f"brakedown_commit/{poly_len}/{n_rows}/{e}{lv}{nd}{r}")
        assert rc == 0
    rc, _ = both(eng, pc, lambda o: L.pcgpu_brakedown_encode(ctx, code.handle, o.inp(mat), n_rows, m, o.flags, o.out(z4(n_rows * N))),
                 f"brakedown_encode/{poly_len}/{n_rows}")
    assert rc == 0
    bad = fr(n_rows * (m + 1), 15)
    assert both(eng, pc, lambda o: L.pcgpu_brakedown_commit(ctx, code.handle, o.inp(bad), n_rows, m + 1, 0, o.flags,
                                                            o.out(z4(n_rows * N)), None, None, None))[0] == E_LEN


@pytest.mark.parametrize("n,m,count", [(3, 4, 2), (5, 2, 1), (4, 3, 0), (0, 2, 2)])
def test_sprs_row_mul(eng, pc, n, m, count):
    L, ctx = eng.lib, eng.ctx
    g = util.rng(100 + n)
    cols = [sorted(set(g.integers(0, n, size=2).tolist())) if n else [] for _ in range(m)]
    ind_ptr = np.cumsum([0] + [len(c) for c in cols]).astype(np.uint64)
    col_ind = np.array([i for c in cols for i in c], dtype=np.uint64)
    val = fr(col_ind.size, 16)
    v = fr(count * n, 17)

    def call(o, val=val):
        return L.pcgpu_fr_sprs_row_mul(ctx, CID, n, m, o.out(ind_ptr, host=True), o.out(col_ind, host=True), o.out(val, host=True),
                                       o.inp(v), count, o.flags, o.out(z4(count * m)))
    assert both(eng, pc, call, f"sprs_row_mul/{n}/{m}/{count}")[0] == 0
    if val.size:
        bad = val.copy()
        bad[-1] = np.uint64(2**64 - 1)
        assert both(eng, pc, lambda o: call(o, bad))[0] == E_RANGE


# ---------------------------------------------------------------------------------------------------------------------------
# G1 wire formats, hash-to-curve generators, SRS registration
# ---------------------------------------------------------------------------------------------------------------------------
def points(n, seed=20):
    return util.random_points(CN, max(n, 1), seed=seed)[:n]


@pytest.mark.parametrize("n", [0, 1, 4])
@pytest.mark.parametrize("compressed", [False, True])
def test_g1_wire(eng, pc, n, compressed):
    L, ctx = eng.lib, eng.ctx
    xy = points(n)
    inf = np.zeros(n, dtype=np.uint8)
    inf[1::2] = 1
    f = pc.binding.WIRE_COMPRESSED if compressed else 0
    sz = eng.g1_wire_size(CID, compressed)
    for with_inf in (False, True):
        rc, res = both(eng, pc, lambda o: L.pcgpu_g1_serialize(ctx, CID, o.inp(xy), o.inp(inf) if with_inf else None, n, o.flags | f,
                                                               o.out(np.zeros((n, sz), dtype=np.uint8))),
                       f"g1_serialize/{n}/{int(compressed)}/{int(with_inf)}")
        assert rc == 0
    wire = res[0]

    def deser(o, data):
        return L.pcgpu_g1_deserialize(ctx, CID, o.inp(data), n, o.flags | f, o.out(np.zeros((n, 2 * NQ), dtype=np.uint64)),
                                      o.out(np.zeros(n, dtype=np.uint8)),
                                      ctypes.cast(o.out(np.zeros(1, dtype=np.uint64), host=True), ctypes.POINTER(ctypes.c_size_t)),
                                      ctypes.cast(o.out(np.zeros(1, dtype=np.int32), host=True), ctypes.POINTER(ctypes.c_int)))
    assert both(eng, pc, lambda o: deser(o, wire), f"g1_deserialize/{n}/{int(compressed)}")[0] == 0
    if n:
        bad = wire.copy()
        bad[n - 1] ^= 0xff
        assert both(eng, pc, lambda o: deser(o, bad))[0] == E_INVALID


@pytest.mark.parametrize("n", [0, 1, 3])
def test_sample_generators(eng, pc, n):
    L, ctx = eng.lib, eng.ctx
    name = np.frombuffer(b"staging-paths", dtype=np.uint8).copy()
    for nl, code in ((name.size, 0), (41, E_BADARG)):
        long = np.zeros(nl, dtype=np.uint8)
        long[:min(nl, name.size)] = name[:nl]
        rc, _ = both(eng, pc, lambda o: L.pcgpu_g1_sample_generators(ctx, CID, o.out(long, host=True), nl, 5, n, o.flags,
                                                                     o.out(np.zeros((n, 2 * NQ), dtype=np.uint64))),
                     f"sample_generators/{n}" if code == 0 else None)
        assert rc == code


@pytest.mark.parametrize("n", [0, 1, 5])
def test_srs_register(eng, pc, n):
    """the identity flags are staged (host) or read in place (device); the registered key is checked through one host MSM"""
    L, ctx = eng.lib, eng.ctx
    xy = points(n, seed=21)
    inf = np.zeros(n, dtype=np.uint8)
    inf[::3] = 1
    sc = util.rand_fr(CN, n, seed=22, mont=False)

    def call(o, count=n):
        h = ctypes.c_void_p()
        rc = L.pcgpu_srs_register(ctx, CID, o.inp(xy), o.inp(inf), count, o.flags, ctypes.byref(h))
        if rc:
            return rc
        rc = L.pcgpu_msm(ctx, h, 0, o.out(sc, host=True), n, 0, o.out(np.zeros(2 * NQ, dtype=np.uint64), host=True),
                         o.out(np.zeros(1, dtype=np.uint8), host=True))
        L.pcgpu_srs_release(ctx, h)
        return rc
    assert both(eng, pc, call)[0] == 0
    assert both(eng, pc, lambda o: call(o, 1 << 26))[0] == E_BADARG


# ---------------------------------------------------------------------------------------------------------------------------
# MSM and KZG10 (outputs are host points; the device operands are the scalars / coefficients)
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def srs(eng):
    s = eng.srs_register(CID, points(SRS_N, seed=23))
    yield s
    s.release()


def pt_out(o):
    return o.out(np.zeros(2 * NQ, dtype=np.uint64), host=True), o.out(np.zeros(1, dtype=np.uint8), host=True)


@pytest.mark.parametrize("n", [0, 1, 5])
def test_msm(eng, pc, srs, n):
    L, ctx = eng.lib, eng.ctx
    sc = util.rand_fr(CN, n, seed=24, mont=False)
    assert both(eng, pc, lambda o: L.pcgpu_msm(ctx, srs.handle, 2, o.inp(sc), n, o.flags, *pt_out(o)))[0] == 0
    assert both(eng, pc, lambda o: L.pcgpu_msm(ctx, srs.handle, SRS_N - n + 1, o.inp(sc), n, o.flags, *pt_out(o)))[0] == E_LEN
    if n:
        bad = canon_bad(n)
        assert both(eng, pc, lambda o: L.pcgpu_msm(ctx, srs.handle, 0, o.inp(bad), n, o.flags, *pt_out(o)))[0] == E_RANGE


@pytest.mark.parametrize("n,count", [(0, 2), (1, 1), (5, 3)])
def test_msm_batch(eng, pc, srs, n, count):
    L, ctx = eng.lib, eng.ctx
    sc = util.rand_fr(CN, n * count, seed=25, mont=False)

    def call(o, n=n):
        return L.pcgpu_msm_batch(ctx, srs.handle, o.inp(sc), n, count, o.flags, o.out(np.zeros((count, 2 * NQ), dtype=np.uint64),
                                                                                        host=True),
                                 o.out(np.zeros(count, dtype=np.uint8), host=True))
    assert both(eng, pc, call)[0] == 0
    assert both(eng, pc, lambda o: call(o, SRS_N + 1))[0] == E_LEN


@pytest.mark.parametrize("n", [0, 1, 5])
def test_fixed_base(eng, pc, n):
    L, ctx = eng.lib, eng.ctx
    base = points(1, seed=26)[0]
    sc = util.rand_fr(CN, n, seed=27, mont=False)
    both(eng, pc, lambda o: L.pcgpu_g1_fixed_base_mul(ctx, CID, o.out(base, host=True), o.inp(sc), n, o.flags,
                                                      o.out(np.zeros((n, 2 * NQ), dtype=np.uint64))))
    assert both(eng, pc, lambda o: L.pcgpu_g1_fixed_base_mul(ctx, CID, o.out(base, host=True), None, 2, o.flags,
                                                             o.out(np.zeros((2, 2 * NQ), dtype=np.uint64))))[0] == E_BADARG


def poly(n, trailing_zeros, seed):
    p = fr(n + trailing_zeros, seed)
    p[n:] = 0
    return p


@pytest.mark.parametrize("n,tz", [(0, 0), (0, 3), (1, 0), (5, 2), (SRS_N, 4)])
def test_kzg(eng, pc, srs, n, tz):
    """commit (with and without a blinding polynomial), open and the fused commit + open; trailing zero coefficients are
    trimmed on the host or on the device"""
    L, ctx = eng.lib, eng.ctx
    p, blind, z = poly(n, tz, 28), poly(3, 1, 29), fr(1, 30)
    m = n + tz
    for nb in (0, 4):
        g = srs.handle if nb else None
        assert both(eng, pc, lambda o: L.pcgpu_kzg_commit(ctx, srs.handle, o.inp(p), m, g, o.inp(blind), nb, o.flags, *pt_out(o)))[0] == 0
        assert both(eng, pc, lambda o: L.pcgpu_kzg_open(ctx, srs.handle, o.inp(p), m, o.out(z, host=True), g, o.inp(blind), nb,
                                                        o.flags, *pt_out(o), o.out(z4(1), host=True)))[0] == 0
    assert both(eng, pc, lambda o: L.pcgpu_kzg_commit_open(ctx, srs.handle, o.inp(p), m, o.out(z, host=True), o.flags, *pt_out(o),
                                                           *pt_out(o)))[0] == 0


def test_kzg_errors(eng, pc, srs):
    L, ctx = eng.lib, eng.ctx
    big, blind, z = fr(SRS_N + 1, 31), fr(3, 32), fr(1, 33)
    assert both(eng, pc, lambda o: L.pcgpu_kzg_commit(ctx, srs.handle, o.inp(big), SRS_N + 1, None, None, 0, o.flags,
                                                      *pt_out(o)))[0] == E_DEGREE
    assert both(eng, pc, lambda o: L.pcgpu_kzg_open(ctx, srs.handle, o.inp(big), 4, o.out(z, host=True), None, o.inp(blind), 3,
                                                    o.flags, *pt_out(o), o.out(z4(1), host=True)))[0] == E_HIDING
    assert both(eng, pc, lambda o: L.pcgpu_kzg_commit_open(ctx, srs.handle, o.inp(big), SRS_N + 1, o.out(z, host=True), o.flags,
                                                           *pt_out(o), *pt_out(o)))[0] == E_DEGREE


def test_msm_peer_single_rank(eng, pc, srs):
    """the index-sharded MSM with one rank: its own window receives its record"""
    L, ctx = eng.lib, eng.ctx
    win, _ = eng.peer_alloc(eng.peer_window_bytes())
    arr = (ctypes.c_void_p * 1)(win)
    epoch = [0]

    def call(o, n, off=0, sc=None):
        epoch[0] += 1
        sc = util.rand_fr(CN, n, seed=34, mont=False) if sc is None else sc
        return L.pcgpu_msm_peer(ctx, srs.handle, off, o.inp(sc), n, o.flags, arr, 0, 1, epoch[0], *pt_out(o))
    try:
        for n in (0, 1, 5):
            assert both(eng, pc, lambda o: call(o, n))[0] == 0
        assert both(eng, pc, lambda o: call(o, 5, off=SRS_N - 4))[0] == E_LEN
        assert both(eng, pc, lambda o: call(o, 3, sc=canon_bad(3)))[0] == E_RANGE
    finally:
        eng.peer_free(win)
