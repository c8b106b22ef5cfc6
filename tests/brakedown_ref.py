"""Brakedown test references, independent of the library:
  - a literal Python-integer transcription of SprsMat::row_mul (linear_codes/utils.rs:41-52) and MultilinearBrakedown::encode
    (multilinear_brakedown/mod.rs:56-84), including the ascending B loop and naive_reed_solomon (:111-122);
  - tests/brakedown_oracle.c, the same encode in C over every row (OpenMP), compiled on first use into a temporary directory.
Elements cross this module as (.., 4) uint64 Montgomery limbs, like the ABI."""
import ctypes
import os
import shutil
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
R256 = 1 << 256


def to_ints(arr, r):
    """(.., 4) Montgomery limbs -> list of canonical ints"""
    rinv = pow(R256, -1, r)
    a = np.asarray(arr, dtype=np.uint64).reshape(-1, 4)
    return [(int(x[0]) | int(x[1]) << 64 | int(x[2]) << 128 | int(x[3]) << 192) * rinv % r for x in a]


def from_ints(vals, r):
    """canonical ints -> (n, 4) Montgomery limbs"""
    out = np.zeros((len(vals), 4), dtype=np.uint64)
    for i, v in enumerate(vals):
        w = v % r * R256 % r
        for j in range(4):
            out[i, j] = (w >> (64 * j)) & 0xFFFFFFFFFFFFFFFF
    return out


def row_mul(mat, v, m, r):
    """SprsMat::row_mul over ints: mat = (ind_ptr, col_ind, val ints)"""
    ind_ptr, col_ind, val = mat
    return [sum(v[int(col_ind[k])] * val[k] for k in range(int(ind_ptr[j]), int(ind_ptr[j + 1]))) % r for j in range(m)]


def encode(msg, params, r, deep_first=False):
    """MultilinearBrakedown::encode of one row of canonical ints; params as linear_codes.brakedown_params (values converted
    once with int_mats)"""
    m, m_ext, a_dims, b_dims = params["m"], params["m_ext"], params["a_dims"], params["b_dims"]
    start, end, a_mats, b_mats = params["start"], params["end"], params["a_ints"], params["b_ints"]
    if len(msg) != m:
        raise ValueError("EncodingError")
    cw = list(msg)
    for i, s in enumerate(start):
        cw += row_mul(a_mats[i], cw[s - a_dims[i][0]:s], a_dims[i][1], r)
    cw += [0] * (m_ext - len(cw))
    rss = start[-1] if start else 0
    rsie = rss + (a_dims[-1][1] if a_dims else m)
    rsoe = end[-1] if end else m_ext
    res, x = [], 1
    for _ in range(rsoe - rss):
        acc = 0
        for j in reversed(range(rss, rsie)):
            acc = (acc * x + cw[j]) % r
        res.append(acc)
        x += 1
    cw[rss:rsoe] = res
    order = range(len(start) - 1, -1, -1) if deep_first else range(len(start))
    for i in order:
        s, e = start[i], end[i]
        cw[e:e + b_dims[i][1]] = row_mul(b_mats[i], cw[s:e], b_dims[i][1], r)
    return cw


def int_mats(params, r):
    """adds a_ints / b_ints (matrices with canonical int values) to a params dict"""
    params["a_ints"] = [(p, c, to_ints(v, r)) for p, c, v in params["a_mats"]]
    params["b_ints"] = [(p, c, to_ints(v, r)) for p, c, v in params["b_mats"]]
    return params


# ---- the C oracle ---------------------------------------------------------------------------------------------------------
_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        d = tempfile.mkdtemp(prefix="bdo_")
        so = os.path.join(d, "libbdo.so")
        cc = shutil.which("gcc") or shutil.which("cc")
        subprocess.check_call([cc, "-O2", "-fopenmp", "-shared", "-fPIC", "-o", so, os.path.join(_HERE, "brakedown_oracle.c")])
        _LIB = ctypes.CDLL(so)
        shutil.rmtree(d, ignore_errors=True)      # the loaded image stays mapped
    return _LIB


def _limbs(v):
    return np.array([(v >> (64 * j)) & 0xFFFFFFFFFFFFFFFF for j in range(4)], dtype=np.uint64)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def c_encode(mat, params, r, deep_first=False):
    """every row of mat (n_rows, m, 4) Montgomery -> (n_rows, m_ext, 4) through brakedown_oracle.c"""
    mat = np.ascontiguousarray(mat, dtype=np.uint64)
    n_rows = mat.shape[0]
    L = len(params["a_dims"])
    mats = [tuple(np.ascontiguousarray(x, dtype=np.uint64) for x in t) for t in list(params["a_mats"]) + list(params["b_mats"])]
    P = (ctypes.c_void_p * max(1, 2 * L))(*[_p(t[0]) for t in mats])
    C = (ctypes.c_void_p * max(1, 2 * L))(*[_p(t[1]) for t in mats])
    V = (ctypes.c_void_p * max(1, 2 * L))(*[_p(t[2]) for t in mats])
    ad = np.ascontiguousarray(np.asarray(params["a_dims"], dtype=np.uint64).reshape(-1)) if L else np.zeros(3, dtype=np.uint64)
    bd = np.ascontiguousarray(np.asarray(params["b_dims"], dtype=np.uint64).reshape(-1)) if L else np.zeros(3, dtype=np.uint64)
    out = np.zeros((n_rows, params["m_ext"], 4), dtype=np.uint64)
    pl, one = _limbs(r), _limbs(R256 % r)
    lib = _lib()
    lib.bdo_encode.argtypes = [ctypes.c_void_p] * 2 + [ctypes.c_uint64] * 3 + [ctypes.c_void_p] * 5 + [ctypes.c_void_p, ctypes.c_uint64,
                                                                                                          ctypes.c_void_p, ctypes.c_int]
    lib.bdo_encode(_p(pl), _p(one), params["m"], params["m_ext"], L, _p(ad), _p(bd), P, C, V, _p(mat), n_rows, _p(out),
                   1 if deep_first else 0)
    return out


def c_sprs_row_mul(r, n, m, mat, v, count):
    ind_ptr, col_ind, val = (np.ascontiguousarray(x, dtype=np.uint64) for x in mat)
    v = np.ascontiguousarray(v, dtype=np.uint64)
    out = np.zeros((count, m, 4), dtype=np.uint64)
    pl = _limbs(r)
    lib = _lib()
    lib.bdo_sprs_row_mul.argtypes = [ctypes.c_void_p, ctypes.c_uint64, ctypes.c_uint64] + [ctypes.c_void_p] * 4 + [ctypes.c_uint64,
                                                                                                                   ctypes.c_void_p]
    lib.bdo_sprs_row_mul(_p(pl), n, m, _p(ind_ptr), _p(col_ind), _p(val), _p(v), count, _p(out))
    return out


def u64_source(seed):
    """a fast seeded u64 stream (numpy PCG64 in blocks) as a next_u64 callable"""
    g = np.random.default_rng(seed)
    buf = []

    def nxt():
        if not buf:
            buf.extend(reversed(g.integers(0, 2**64, size=1 << 20, dtype=np.uint64).tolist()))
        return buf.pop()
    return nxt
