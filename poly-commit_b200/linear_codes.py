"""Host mirror of the Ligero prover's matrix step (poly-commit/src/linear_codes) over the C ABI -- SURVEY.md section 8f
rank 4: the one place the reference exercises the NTT.

  calculate_t            linear_codes/utils.rs:156-184
  compute_dimensions     linear_codes/ligero.rs:118-128
  Matrix::new_from_flat  utils.rs:61-77            (row-major: entry[row][col] = flat[m * row + col])
  reed_solomon           linear_codes/utils.rs:112-127   -> one row of Engine.ntt_batch
  compute_matrices       linear_codes/mod.rs:118-138     -> Engine.ntt_batch over all rows (one launch up to 2^11 columns)
  b^T . M                linear_codes/mod.rs:? (open) via Matrix::row_mul, utils.rs:127-146  -> Engine.fr_row_mul

  commit steps 2-3       linear_codes/mod.rs:253-275: column hashes (FieldToBytesColHasher<F, Blake2s256>) and the Merkle tree
                         (LeafIdentityHasher + SHA-256 two-to-one, the configuration of the reference's tests and benches) run on
                         the device behind Engine.lincode_commit; `commit` below is LinearCodePCS::commit for one polynomial and
                         `merkle_path` is MerkleTree::generate_proof (used by generate_proof, linear_codes/mod.rs:553-558).
"""
import math

import numpy as np

FIELD_BITS = {0: 255, 1: 254, 2: 255}


def ceil_div(x, y):
    return (x + y - 1) // y


def calculate_t(field_bits, sec_param, distance, codeword_len):
    """linear_codes/utils.rs:156-184 (same f64 arithmetic); field_bits = F::MODULUS_BIT_SIZE"""
    residual = codeword_len / 2.0 ** field_bits
    arg = 2.0 ** (-sec_param) - residual
    if not arg > 0.0:
        raise ValueError("InvalidParameters: the field is not big enough")
    nom = math.log2(arg) - 1.0
    denom = math.log2(1.0 - 0.5 * distance[0] / distance[1])
    if denom == 0.0 or not math.isfinite(denom):
        raise ValueError("InvalidParameters: the distance is wrong")
    t = math.ceil(nom / denom)
    return t if t < codeword_len else codeword_len


def compute_dimensions(curve, sec_param, rho_inv, poly_len):
    """linear_codes/ligero.rs:118-128 with distance = (rho_inv - 1, rho_inv) (ligero.rs distance())"""
    t = calculate_t(FIELD_BITS[curve], sec_param, (rho_inv - 1, rho_inv), poly_len)
    root = math.ceil(math.sqrt(ceil_div(2 * poly_len, t)))
    n = 1 << max(0, (root - 1).bit_length())                 # 1 << log2(x): ark_std::log2 is ceil(log2 x)
    return n, ceil_div(poly_len, n)


def _domain_log(size):
    return max(0, (size - 1).bit_length())


def reed_solomon(eng, curve, msg, rho_inv):
    """linear_codes/utils.rs:112-127: msg (m, 4) -> evaluations over the smallest domain of size >= m * rho_inv"""
    msg = np.asarray(msg, dtype=np.uint64).reshape(1, -1, 4)
    return eng.ntt_batch(curve, msg, _domain_log(msg.shape[1] * rho_inv))[0]


def compute_matrices(eng, curve, coeffs, n_rows, n_cols, rho_inv):
    """linear_codes/mod.rs:118-138 -> (mat (n_rows, n_cols, 4), ext_mat (n_rows, domain, 4)); coeffs zero-padded to n_rows*n_cols"""
    coeffs = np.asarray(coeffs, dtype=np.uint64).reshape(-1, 4)
    if coeffs.shape[0] > n_rows * n_cols:
        raise ValueError("more coefficients than matrix entries")
    flat = np.zeros((n_rows * n_cols, 4), dtype=np.uint64)
    flat[:coeffs.shape[0]] = coeffs
    mat = flat.reshape(n_rows, n_cols, 4)
    return mat, eng.ntt_batch(curve, mat, _domain_log(n_cols * rho_inv))


BLAKE2S, SHA256 = 0, 1


def commit(eng, curve, coeffs, sec_param=128, rho_inv=4, hash=BLAKE2S):
    """LinearCodePCS::commit for one polynomial given as its coefficient vector (linear_codes/mod.rs:228-298) ->
    (commitment dict(metadata=(n_rows, n_cols, n_ext_cols), root=bytes), state dict(mat, ext_mat, leaves, nodes)).
    Row encoding, column hashing and the tree run in ONE device-resident call."""
    coeffs = np.asarray(coeffs, dtype=np.uint64).reshape(-1, 4)
    n_rows, n_cols = compute_dimensions(curve, sec_param, rho_inv, coeffs.shape[0])
    flat = np.zeros((n_rows * n_cols, 4), dtype=np.uint64)
    flat[:coeffs.shape[0]] = coeffs
    mat = flat.reshape(n_rows, n_cols, 4)
    log_ext = _domain_log(n_cols * rho_inv)
    r = eng.lincode_commit(curve, mat, log_ext, hash=hash)
    n_ext = 1 << log_ext
    return (dict(metadata=(n_rows, n_cols, n_ext), root=r["root"].tobytes()),
            dict(mat=mat, ext_mat=r["ext"], leaves=r["leaves"], nodes=r["nodes"]))


def merkle_path(state, index):
    """MerkleTree::generate_proof(index) over the state's tree -> dict(leaf_sibling_hash, auth_path (root's children first, as
    ark-crypto-primitives stores it), leaf_index).  The padding leaves are empty (Vec::default())."""
    leaves, nodes = state["leaves"], state["nodes"]
    P = nodes.shape[0] + 1
    sib = index ^ 1
    leaf_sibling = leaves[sib].tobytes() if sib < leaves.shape[0] else b""
    node = P // 2 - 1 + index // 2                    # heap index of the leaf pair's parent
    path = []
    while node > 0:
        sibling = node + 1 if node % 2 == 1 else node - 1
        path.append(nodes[sibling].tobytes())
        node = (node - 1) // 2
    return dict(leaf_sibling_hash=leaf_sibling, auth_path=path[::-1], leaf_index=index)


# ---- Brakedown (linear_codes/brakedown.rs, multilinear_brakedown/mod.rs) ----------------------------------------------------
#   BrakedownPCParams::default  brakedown.rs:103-143    -> brakedown_params (the matrices from a caller-supplied u64 source)
#   MultilinearBrakedown::encode multilinear_brakedown/mod.rs:56-84 -> Engine.brakedown_encode / brakedown_commit
#   tensor_vec                   linear_codes/utils.rs:240-258   -> b = tensor_vec(point[..log2 n]) for the open's row_mul
BRAKEDOWN_ALPHA, BRAKEDOWN_BETA, BRAKEDOWN_RHO_INV, BRAKEDOWN_BASE_LEN = (178, 1000), (61, 1000), (1521, 1000), 30


def ceil_mul(a, b):
    """utils.rs:37-39"""
    return (a * b[0] + b[1] - 1) // b[1]


def _ent(x):
    """utils.rs:26-33 (binary entropy, f64)"""
    assert 0.0 <= x <= 1.0
    if x == 0.0 or x == 1.0:
        return 0.0
    return -x * math.log2(x) - (1.0 - x) * math.log2(1.0 - x)


def _fdiv(a):
    return a[0] / a[1]


def _cn_const(a, b):
    """brakedown.rs:218-226"""
    a, b = _fdiv(a), _fdiv(b)
    arg = 1.28 * b / a
    return (_ent(b) + a * _ent(arg), -b * math.log2(arg))


def _dn_const(a, b, r):
    """brakedown.rs:237-248, with mu (:205-210) and nu (:211-217)"""
    mu = (r[0] * (a[1] - a[0]) - r[1] * a[1]) / (r[1] * a[1])
    c = (3, 100)
    nu = (b[0] * (a[1] + a[0]) * c[1] + c[0] * b[1] * a[1]) / (b[1] * a[1] * c[1])
    a, b, r = _fdiv(a), _fdiv(b), _fdiv(r)
    nm = nu / mu
    return (r * a * _ent(b / r) + mu * _ent(nm), -a * b * math.log2(nm))


def _cn(n, b, c):
    """brakedown.rs:227-235"""
    return min(max(ceil_mul(n, (32 * b[0], 25 * b[1])), 4 + ceil_mul(n, b)), math.ceil((110.0 / n + c[0]) / c[1]))


def _dn(n, b, r, d, field_bits):
    """brakedown.rs:249-259"""
    return min(ceil_mul(n, (2 * b[0], b[1])) + math.ceil((ceil_mul(n, r) - n + 110) / field_bits),
               math.ceil((110.0 / n + d[0]) / d[1]))


def brakedown_mat_size(m, field_bits, a=BRAKEDOWN_ALPHA, b=BRAKEDOWN_BETA, r=BRAKEDOWN_RHO_INV, base_len=BRAKEDOWN_BASE_LEN):
    """brakedown.rs:260-288 -> (a_dims, b_dims), lists of (rows, cols, nonzeros per row)"""
    c, d = _cn_const(a, b), _dn_const(a, b, r)
    a_dims, n = [], m
    while n >= base_len:
        mm = ceil_mul(n, a)
        a_dims.append((n, mm, min(_cn(n, b, c), mm)))
        n = mm
    b_dims = []
    for an, am, _ in a_dims:
        bn = ceil_mul(am, r)
        bm = ceil_mul(an, r) - an - bn
        b_dims.append((bn, bm, min(_dn(bn, b, r, d, field_bits), bm)))
    return a_dims, b_dims


def brakedown_codeword_len(a_dims, b_dims):
    """brakedown.rs:292-299"""
    return sum(x[1] for x in b_dims) + sum(x[0] for x in a_dims) + b_dims[-1][0]


def _rand_fr_nonzero(curve, next_u64):
    """a uniform nonzero element of Fr in Montgomery form (4 u64 limbs), by rejection on the bit length of r"""
    from .params import FR_MODULUS, fr_mont
    r = FR_MODULUS[curve]
    mask = (1 << r.bit_length()) - 1
    while True:
        v = sum(next_u64() << (64 * i) for i in range(4)) & mask
        if 0 < v < r:
            return fr_mont(curve, v)


def brakedown_make_mat(curve, n, m, d, next_u64):
    """make_mat (brakedown.rs:305-333): d distinct columns per row by a Fisher-Yates shuffle over a `tmp` that is not reset
    between rows, a nonzero value for each; F::rand is replaced by a uniform nonzero draw -> SprsMat as
    (ind_ptr (m+1,), col_ind (nnz,), val (nnz, 4)) in new_from_columns order"""
    tmp = list(range(m))
    cols = [[] for _ in range(m)]
    for i in range(n):
        idxs = []
        for j in range(d):
            k = next_u64() % (m - j)
            tmp[k], tmp[m - 1 - j] = tmp[m - 1 - j], tmp[k]
            idxs.append(tmp[m - 1 - j])
        for j in idxs:
            cols[j].append((i, _rand_fr_nonzero(curve, next_u64)))
    ind_ptr = np.zeros(m + 1, dtype=np.uint64)
    ind_ptr[1:] = np.cumsum([len(c) for c in cols]) if m else []
    col_ind = np.array([i for c in cols for i, _ in c], dtype=np.uint64)
    val = np.array([v for c in cols for _, v in c], dtype=np.uint64).reshape(-1, 4)
    return ind_ptr, col_ind, val


def brakedown_dims(curve, poly_len, sec_param=128):
    """the shapes of BrakedownPCParams::default (brakedown.rs:103-181) without the matrices -> dict(n, m, m_ext, a_dims, b_dims,
    start, end)"""
    a, b, r, base_len = BRAKEDOWN_ALPHA, BRAKEDOWN_BETA, BRAKEDOWN_RHO_INV, BRAKEDOWN_BASE_LEN
    t = calculate_t(FIELD_BITS[curve], sec_param, (b[0] * r[1], b[1] * r[0]), poly_len)
    root = math.ceil(math.sqrt(ceil_div(2 * poly_len, t)))
    n = 1 << max(0, (root - 1).bit_length())                 # 1 << log2(x): ark_std::log2 is ceil(log2 x)
    m = ceil_div(poly_len, n)
    a_dims, b_dims = brakedown_mat_size(m, FIELD_BITS[curve], a, b, r, base_len)
    m_ext = ceil_mul(m, r) if not a_dims else brakedown_codeword_len(a_dims, b_dims)
    start, acc = [], 0
    for x in a_dims:
        acc += x[0]
        start.append(acc)
    end, acc = [], m_ext
    for x in b_dims:
        acc -= x[1]
        end.append(acc)
    return dict(n=n, m=m, m_ext=m_ext, a_dims=a_dims, b_dims=b_dims, start=start, end=end)


def brakedown_params(curve, poly_len, next_u64, sec_param=128, check_well_formedness=True):
    """BrakedownPCParams::default (brakedown.rs:103-143) with `next_u64` (a callable returning u64) in place of the RNG ->
    dict with the fields of BrakedownPCParams (matrices as SprsMat triples, see brakedown_make_mat)"""
    p = brakedown_dims(curve, poly_len, sec_param)
    p["a_mats"] = [brakedown_make_mat(curve, *dims, next_u64) for dims in p["a_dims"]]
    p["b_mats"] = [brakedown_make_mat(curve, *dims, next_u64) for dims in p["b_dims"]]
    p.update(curve=curve, sec_param=sec_param, alpha=BRAKEDOWN_ALPHA, beta=BRAKEDOWN_BETA, rho_inv=BRAKEDOWN_RHO_INV,
             base_len=BRAKEDOWN_BASE_LEN, check_well_formedness=check_well_formedness)
    return p


def brakedown_register(eng, params):
    """upload the code of brakedown_params' output -> binding.BrakedownCode"""
    return eng.brakedown_register(params["curve"], params["m"], params["m_ext"], params["a_dims"], params["b_dims"],
                                  params["a_mats"], params["b_mats"])


def brakedown_commit(eng, code, evals, n_rows, hash=BLAKE2S):
    """LinearCodePCS::commit (linear_codes/mod.rs:228-298) of one multilinear polynomial given as its 2^k hypercube evaluations,
    `code` a registered BrakedownCode and `n_rows` the params' n -> (commitment dict(metadata=(n_rows, m, m_ext), root=bytes),
    state dict(mat, ext_mat, leaves, nodes)).  Encoding, column hashes and the tree run in ONE device-resident call."""
    evals = np.asarray(evals, dtype=np.uint64).reshape(-1, 4)
    m = code.m
    if evals.shape[0] > n_rows * m:
        raise ValueError("more evaluations than matrix entries")
    flat = np.zeros((n_rows * m, 4), dtype=np.uint64)
    flat[:evals.shape[0]] = evals
    mat = flat.reshape(n_rows, m, 4)
    res = eng.brakedown_commit(code, mat, hash=hash)
    return (dict(metadata=(n_rows, m, code.m_ext), root=res["root"].tobytes()),
            dict(mat=mat, ext_mat=res["ext"], leaves=res["leaves"], nodes=res["nodes"]))


def tensor_vec(curve, values):
    """utils.rs:240-258: values (k, 4) Montgomery -> the 2^k products prod_i (z_i or 1 - z_i), low variable first, Montgomery"""
    from .params import FR_MODULUS
    r = FR_MODULUS[curve]
    rinv = pow(1 << 256, -1, r)
    vals = [sum(int(x) << (64 * j) for j, x in enumerate(row)) * rinv % r for row in np.asarray(values, dtype=np.uint64).reshape(-1, 4)]
    layer = [1]
    for v in vals:
        layer = [x * (1 - v) % r for x in layer] + [x * v % r for x in layer]
    R = 1 << 256
    return np.array([[(x * R % r >> (64 * j)) & 0xFFFFFFFFFFFFFFFF for j in range(4)] for x in layer], dtype=np.uint64)
