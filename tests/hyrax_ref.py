"""A pure-Python restatement of HyraxPC's commit, open and check (poly-commit/src/hyrax) over oracle/pyref.py curve arithmetic
and Python integers: the reference the device proofs are compared with byte for byte.

Scalars are canonical integers mod r, points pyref affine tuples (None = identity).  The sponge and the rng are replaced by
their outputs: the blinds in the order open draws them, the challenges in the order the sponge squeezes them.
"""


def flat_to_matrix_column_major(flat, n, m):
    """hyrax/utils.rs:13-21: n rows of m, row[r][c] = flat[c * n + r]"""
    return [[flat[c * n + r] for c in range(m)] for r in range(n)]


def tensor_prime(values, r):
    """hyrax/utils.rs:27-39: [tail * (1 - v0), tail * v0] with tail = tensor_prime(values[1:]); [1] for no values"""
    if not values:
        return [1]
    tail = tensor_prime(values[1:], r)
    v = values[0]
    return [t * (1 - v) % r for t in tail] + [t * v % r for t in tail]


def tensors(point, r):
    """hyrax/mod.rs:299-307 (open) and :440-448 (check): the point reversed, split, and both halves through tensor_prime"""
    n = len(point)
    point_rev = point[::-1]
    return tensor_prime(point_rev[n // 2:], r), tensor_prime(point_rev[:n // 2], r)    # l (point_lower), r (point_upper)


def pedersen_commit(C, com_key, scalars):
    """hyrax/mod.rs:86-93"""
    return C.msm(com_key[:len(scalars)], scalars)


def commit(C, com_key, h, evals, randomness):
    """hyrax/mod.rs:213-252 for one polynomial of 2^nv evaluations: -> (row_coms, mat)"""
    dim = len(randomness)
    mat = flat_to_matrix_column_major(evals, dim, dim)
    return [C.add(pedersen_commit(C, com_key, row), C.mul(rr, h)) for row, rr in zip(mat, randomness)], mat


def open_one(C, com_key, h, mat, randomness, point, blinds, c):
    """hyrax/mod.rs:335-402 for one polynomial.  blinds = [r_eval] + d + [r_d, r_b], the rng draws of :360, :367-368, :373,
    :377 in that order; c the squeezed challenge (:389)."""
    r_ = C.r
    dim = len(mat)
    l, rt = tensors(point, r_)
    lt = [sum(l[i] * mat[i][j] for i in range(dim)) % r_ for j in range(dim)]                # :347
    r_lt = sum(a * b for a, b in zip(l, randomness)) % r_                                     # :351-354
    ev = sum(a * b for a, b in zip(lt, rt)) % r_                                              # :356
    r_eval, d, r_d, r_b = blinds[0], blinds[1:dim + 1], blinds[dim + 1], blinds[dim + 2]
    com_eval = C.add(C.mul(ev, com_key[0]), C.mul(r_eval, h))                                 # :359-362
    b = sum(a * x for a, x in zip(rt, d)) % r_                                                # :370
    com_d = C.add(pedersen_commit(C, com_key, d), C.mul(r_d, h))                              # :373-374
    com_b = C.add(C.mul(b, com_key[0]), C.mul(r_b, h))                                        # :377-378
    z = [(x + c * y) % r_ for x, y in zip(d, lt)]                                             # :391
    return {"com_eval": com_eval, "com_d": com_d, "com_b": com_b, "z": z, "z_d": (c * r_lt + r_d) % r_,
            "z_b": (c * r_eval + r_b) % r_, "lt": lt, "r_lt": r_lt, "eval": ev}


def check_one(C, com_key, h, row_coms, point, proof, c):
    """hyrax/mod.rs:450-507 for one proof: both of the verifier's equations"""
    r_ = C.r
    l, rt = tensors(point, r_)
    z = proof["z"]
    lhs14 = C.add(C.mul(sum(a * b for a, b in zip(rt, z)) % r_, com_key[0]), C.mul(proof["z_b"], h))   # (14), :492
    if lhs14 != C.add(C.mul(c, proof["com_eval"]), proof["com_b"]):
        return False
    t_prime = C.msm(row_coms, l)                                                                     # :498-501
    lhs13 = C.add(pedersen_commit(C, com_key, z), C.mul(proof["z_d"], h))                           # (13), :504
    return lhs13 == C.add(C.mul(c, t_prime), proof["com_d"])


def mle_eval(evals, point, r):
    """the multilinear polynomial with evaluations `evals` (index bit i = variable i) at `point`: fold variable 0 first"""
    v = list(evals)
    for x in point:
        v = [(v[2 * k] * (1 - x) + v[2 * k + 1] * x) % r for k in range(len(v) // 2)]
    return v[0]
