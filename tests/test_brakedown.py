"""Brakedown (MultilinearBrakedown) encoding and commitment: csrc/sprs.cuh behind pcgpu_brakedown_* / pcgpu_fr_sprs_row_mul.
References: the reference's SprsMat::row_mul KATs (linear_codes/utils.rs:274-301), a Python-integer transcription of encode and
the C oracle tests/brakedown_oracle.c (tests/brakedown_ref.py), hashlib for the column hashes and the tree
(test_lincode_hash.ref_column_hashes / ref_merkle).  CPU: host-emulated kernels; GPU: the CUDA library on the bench range."""
import numpy as np
import pytest

from oracle import pyref
from tests import brakedown_ref as bref
from tests import util
from tests.test_lincode_hash import ref_column_hashes, ref_merkle

E_BADARG, E_LEN, E_RANGE = -3, -4, -5


@pytest.fixture(scope="module")
def emul(pc, hostcheck_path):
    e = pc.Engine(0, lib_path=hostcheck_path)
    yield e
    e.close()


def _lc():
    from poly_commit_b200 import linear_codes
    return linear_codes


_PARAMS = {}


def params_for(cname, poly_len, seed=7):
    key = (cname, poly_len, seed)
    if key not in _PARAMS:
        C = pyref.Curve(cname)
        _PARAMS[key] = _lc().brakedown_params(C.id, poly_len, bref.u64_source(seed))
    return _PARAMS[key]


# ---- 1. the reference's row_mul KATs ---------------------------------------------------------------------------------------
_FLAT = [10, 23, 55, 100, 1, 58, 4, 0, 9]       # column-major 3 x 3


@pytest.mark.parametrize("cname", util.CURVE_NAMES)
@pytest.mark.parametrize("form", ["flat", "columns"])
def test_sprs_row_mul_reference_kats(emul, cname, form):
    C = pyref.Curve(cname)
    if form == "flat":      # SprsMat::new_from_flat skips the zero entry
        cols = [[(c, _FLAT[j * 3 + c]) for c in range(3) if _FLAT[j * 3 + c]] for j in range(3)]
    else:                   # new_from_columns keeps it
        cols = [[(c, _FLAT[j * 3 + c]) for c in range(3)] for j in range(3)]
    ind_ptr = np.cumsum([0] + [len(c) for c in cols]).astype(np.uint64)
    col_ind = np.array([i for c in cols for i, _ in c], dtype=np.uint64)
    val = bref.from_ints([v for c in cols for _, v in c], C.r)
    v = bref.from_ints([12, 41, 55], C.r)
    out = emul.sprs_row_mul(C.id, 3, 3, (ind_ptr, col_ind, val), v)
    assert bref.to_ints(out, C.r) == [4088, 4431, 543]


# ---- 2. parameters and their wire form --------------------------------------------------------------------------------------
@pytest.mark.parametrize("cname", util.CURVE_NAMES)
@pytest.mark.parametrize("log_len", [4, 7, 12, 16, 20, 22])
def test_brakedown_dims(cname, log_len):
    lc = _lc()
    C = pyref.Curve(cname)
    poly_len = 1 << log_len
    d = lc.brakedown_dims(C.id, poly_len)
    a_dims, b_dims = d["a_dims"], d["b_dims"]
    assert d["n"] * d["m"] >= poly_len
    if a_dims:
        assert d["m_ext"] == lc.brakedown_codeword_len(a_dims, b_dims)
        assert d["end"][-1] - d["start"][-1] == lc.ceil_mul(a_dims[-1][1], lc.BRAKEDOWN_RHO_INV)
        assert a_dims[0][0] == d["m"]
        for i in range(len(a_dims) - 1):
            assert a_dims[i][1] == a_dims[i + 1][0]
        for i, b in enumerate(b_dims):
            assert b[0] == d["end"][i] - d["start"][i]
    else:
        assert d["m"] < lc.BRAKEDOWN_BASE_LEN and d["m_ext"] == lc.ceil_mul(d["m"], lc.BRAKEDOWN_RHO_INV)
    for dims in a_dims + b_dims:
        assert dims[2] <= dims[1]


def test_brakedown_params_wire_roundtrip():
    from poly_commit_b200 import wire
    p = params_for("bn254", 1 << 12)
    data = wire.brakedown_params_serialize(p)
    q = wire.brakedown_params_deserialize(p["curve"], data)
    assert wire.brakedown_params_serialize(q) == data
    for k in ("n", "m", "m_ext", "start", "end", "check_well_formedness"):
        assert q[k] == p[k]
    assert [tuple(x) for x in q["a_dims"]] == [tuple(x) for x in p["a_dims"]]
    for x, y in zip(q["a_mats"] + q["b_mats"], p["a_mats"] + p["b_mats"]):
        assert all((np.asarray(u) == np.asarray(w)).all() for u, w in zip(x, y))
    for cut in (1, 8, len(data) // 2, len(data) - 1):
        with pytest.raises(ValueError):
            wire.brakedown_params_deserialize(p["curve"], data[:cut])


# ---- 3. encode against both oracles -----------------------------------------------------------------------------------------
# poly_len 16: m = 8 < base_len (Reed-Solomon only); 128: one level; 2^12: three levels
@pytest.mark.parametrize("cname", util.CURVE_NAMES)
@pytest.mark.parametrize("poly_len,levels", [(16, 0), (128, 1), (1 << 12, 3)])
def test_encode_vs_oracles(emul, cname, poly_len, levels):
    C = pyref.Curve(cname)
    p = params_for(cname, poly_len)
    assert len(p["a_dims"]) == levels
    code = _lc().brakedown_register(emul, p)
    for n_rows in (1, 2, 33):
        mat = util.rand_fr_fast(cname, n_rows * p["m"], seed=40 + n_rows).reshape(n_rows, p["m"], 4)
        got = emul.brakedown_encode(code, mat)
        exp = bref.c_encode(mat, p, C.r)
        assert (got == exp).all(), (cname, poly_len, n_rows)
    # the two oracles agree (Python integers on two rows)
    bref.int_mats(p, C.r)
    for row in range(2):
        assert bref.to_ints(exp[row], C.r) == bref.encode(bref.to_ints(mat[row], C.r), p, C.r)
    if levels >= 3:       # the B order matters here: deepest-first gives another codeword, and the case sees it
        deep = bref.c_encode(mat[:2], p, C.r, deep_first=True)
        assert not (deep == exp[:2]).all()
        assert bref.to_ints(deep[0], C.r) == bref.encode(bref.to_ints(mat[0], C.r), p, C.r, deep_first=True)
    code.release()


def test_sprs_row_mul_vs_oracle(emul):
    C = pyref.Curve("pallas")
    p = params_for("pallas", 1 << 12)
    ind_ptr, col_ind, val = p["b_mats"][0]
    n, m, _ = p["b_dims"][0]
    v = util.rand_fr_fast("pallas", 3 * n, seed=50).reshape(3, n, 4)
    got = emul.sprs_row_mul(C.id, n, m, (ind_ptr, col_ind, val), v)
    assert (got == bref.c_sprs_row_mul(C.r, n, m, (ind_ptr, col_ind, val), v, 3)).all()


# ---- 4. commit ----------------------------------------------------------------------------------------------------------------
def _commit_check(eng, cname, poly_len, seed, n_rows=None, sample=None):
    lc = _lc()
    C = pyref.Curve(cname)
    p = params_for(cname, poly_len)
    code = lc.brakedown_register(eng, p)
    n_rows = p["n"] if n_rows is None else n_rows
    evals = util.rand_fr_fast(cname, min(poly_len, n_rows * p["m"]), seed=seed)
    comm, st = lc.brakedown_commit(eng, code, evals, n_rows)
    assert comm["metadata"] == (n_rows, p["m"], p["m_ext"])
    exp_ext = bref.c_encode(st["mat"], p, C.r)
    assert (st["ext_mat"] == exp_ext).all()
    cols = range(p["m_ext"]) if sample is None else sample
    exp_leaves = ref_column_hashes(C, np.ascontiguousarray(exp_ext[:, list(cols), :]), "blake2s")
    assert [st["leaves"][j].tobytes() for j in cols] == exp_leaves
    nodes, root = ref_merkle([bytes(x) for x in st["leaves"]])          # m_ext is not a power of two: empty padding leaves
    assert comm["root"] == root and [bytes(x) for x in st["nodes"]] == nodes
    # fused == encode -> lincode_hash_columns -> merkle_tree
    ext = eng.brakedown_encode(code, st["mat"])
    leaves = eng.lincode_hash_columns(C.id, ext)
    assert (leaves == st["leaves"]).all() and eng.merkle_tree(leaves)[1].tobytes() == comm["root"]
    return code, p, st


@pytest.mark.parametrize("cname,poly_len", [("bn254", 1 << 12), ("bls12_381", 128), ("pallas", 16)])
def test_commit_vs_hashlib(emul, cname, poly_len):
    code, _, _ = _commit_check(emul, cname, poly_len, seed=60)
    code.release()


# ---- 6. errors ----------------------------------------------------------------------------------------------------------------
def _expect(pc, code, fn):
    with pytest.raises(pc.PcgpuError) as e:
        fn()
    assert e.value.code == code


def test_register_and_encode_errors(emul, pc):
    C = pyref.Curve("bn254")
    p = params_for("bn254", 1 << 12)
    m, m_ext, A, B = p["m"], p["m_ext"], list(p["a_dims"]), list(p["b_dims"])
    reg = lambda **kw: emul.brakedown_register(C.id, kw.get("m", m), kw.get("m_ext", m_ext), kw.get("a", A), kw.get("b", B),
                                               kw.get("am", p["a_mats"]), kw.get("bm", p["b_mats"]))
    code = reg()
    # a_dims[i].1 != a_dims[i+1].0
    a2 = [A[0], (A[1][0] + 1, A[1][1], A[1][2])] + A[2:]
    _expect(pc, E_BADARG, lambda: reg(a=a2))
    # b_dims[i].0 != end[i] - start[i]
    _expect(pc, E_BADARG, lambda: reg(b=[(B[0][0] - 1, B[0][1], B[0][2])] + B[1:]))
    # m_ext != codeword_len
    _expect(pc, E_BADARG, lambda: reg(m_ext=m_ext + 1))
    # ind_ptr not monotone; ind_ptr[m] > n * d
    ip, ci, v = p["a_mats"][0]
    bad = ip.copy(); bad[1], bad[2] = bad[2], bad[1]
    if bad[1] == bad[2]:
        bad[1] += 1
    _expect(pc, E_BADARG, lambda: reg(am=[(bad, ci, v)] + p["a_mats"][1:]))
    A0 = (A[0][0], A[0][1], A[0][2] - 1)
    _expect(pc, E_BADARG, lambda: reg(a=[A0] + A[1:]))
    # col_ind >= n
    ci2 = ci.copy(); ci2[0] = A[0][0]
    _expect(pc, E_BADARG, lambda: reg(am=[(ip, ci2, v)] + p["a_mats"][1:]))
    # an unreduced value
    v2 = v.copy(); v2[0] = [2**64 - 1] * 4
    _expect(pc, E_RANGE, lambda: reg(am=[(ip, ci, v2)] + p["a_mats"][1:]))
    # a row of the wrong length: Error::EncodingError
    mat = util.rand_fr_fast("bn254", 2 * (m + 1), seed=70).reshape(2, m + 1, 4)
    _expect(pc, E_LEN, lambda: emul.brakedown_encode(code, mat))
    code.release()


# ---- 5. the device, on the bench range ----------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cname,log_len", [("bn254", 12), ("bn254", 16), ("bn254", 20), ("bls12_381", 16), ("pallas", 16)])
def test_gpu_brakedown_commit(gpu_engine, cname, log_len):
    eng = gpu_engine
    p = params_for(cname, 1 << log_len)
    sample = [0, 1, p["m"], p["m_ext"] // 2, p["end"][-1] if p["end"] else 2, p["m_ext"] - 1]
    code, p, st = _commit_check(eng, cname, 1 << log_len, seed=80 + log_len, sample=sample if log_len >= 20 else None)
    C = pyref.Curve(cname)
    # linearity: encode(c x + y) = c encode(x) + encode(y)
    x, y = st["mat"], util.rand_fr_fast(cname, st["mat"].shape[0] * p["m"], seed=90).reshape(st["mat"].shape)
    c = util.rand_fr_fast(cname, 1, seed=91)[0]
    cxy = eng.fr_axpy(C.id, y.reshape(-1, 4), c, x.reshape(-1, 4))
    lhs = eng.brakedown_encode(code, cxy.reshape(x.shape))
    rhs = eng.fr_axpy(C.id, eng.brakedown_encode(code, y).reshape(-1, 4), c, st["ext_mat"].reshape(-1, 4))
    assert (lhs.reshape(-1, 4) == rhs).all()
    # the verifier's shape: one row
    one = eng.brakedown_encode(code, x[3:4] if x.shape[0] > 3 else x[:1])
    assert (one == bref.c_encode(x[3:4] if x.shape[0] > 3 else x[:1], p, C.r)).all()
    code.release()


@pytest.mark.gpu
def test_gpu_brakedown_2p22_bn254(gpu_engine, pc):
    """the largest benched shape: all 64 rows against the C oracle, the tree against hashlib over the device leaves, a sample of
    columns re-hashed, and PCGPU_DEVICE_PTRS == the host-pointer path"""
    eng = gpu_engine
    code, p, st = _commit_check(eng, "bn254", 1 << 22, seed=100, sample=[0, 5, 65536, 70001, 99680])
    assert st["mat"].shape[0] == 64
    n, m, N = 64, p["m"], p["m_ext"]
    P = 1 << (N - 1).bit_length()
    din, dext = eng.buffer(n * m), eng.buffer(n * N)
    dleaves, dnodes = eng.buffer(N), eng.buffer(P - 1)
    din.write(st["mat"].reshape(-1, 4))
    r = eng.brakedown_commit(code, din.ptr(), n_rows=n, n_cols=m, flags=pc.DEVICE_PTRS, out_ext=dext.ptr(),
                             out_leaves=dleaves.ptr(), out_nodes=dnodes.ptr())
    assert (dext.read() == st["ext_mat"].reshape(-1, 4)).all()
    assert dleaves.read().view(np.uint8).reshape(N, 32).tobytes() == st["leaves"].tobytes()
    assert dnodes.read().view(np.uint8).reshape(P - 1, 32).tobytes() == st["nodes"].tobytes()
    assert r["root"].tobytes() == bytes(st["nodes"][0])
    for b in (din, dext, dleaves, dnodes):
        b.release()
    code.release()
