"""Host mirror of HyraxPC's prover hot path (poly-commit/src/hyrax/mod.rs) over the C ABI.

  flat_to_matrix_column_major   hyrax/utils.rs:13-21
  pedersen_commit               hyrax/mod.rs:86-93
  commit (row loop)             hyrax/mod.rs:230-242   -> Engine.msm_batch over comb tables of com_key || h
  open: lt = mat.row_mul(l)     hyrax/mod.rs:347 -> utils.rs:127-146 -> Engine.fr_row_mul
  check: t_prime                hyrax/mod.rs:498-504   msm_bigint(&row_coms, &l_bigint) -> Engine.msm_bases (fresh bases)

and the whole scheme on the device (pcgpu_hyrax_*):
  setup / trim                  hyrax/mod.rs:119-183   -> Engine.g1_sample_generators, CommitterKey
  commit_resident               hyrax/mod.rs:213-252   -> Engine.hyrax_commit: row commitments + the resident HyraxState
  open                          hyrax/mod.rs:273-406   -> Engine.hyrax_open, the caller's challenge, Engine.fr_axpy
  check                         hyrax/mod.rs:418-511   -> Engine.hyrax_check: every proof of a batch in one call

The reference draws the row randomness r_i from `thread_rng()` when built with the `parallel` feature (:237-238), so its
commitments are not reproducible; here the randomness is an argument, and so are the opening's blinds (laid out in the order
the reference draws them from its rng) and the challenges (the sponge stays with the caller).  Every Fr is Montgomery.
"""
import numpy as np

from .binding import BLS12_381, SCALARS_MONT, SRS_COMB

PROTOCOL_NAME = b"Hyrax protocol"   # hyrax/mod.rs:26


def flat_to_matrix_column_major(flat, n, m):
    """(n*m, 4) flat vector -> n rows of length m, row[r][c] = flat[c*n + r]  (hyrax/utils.rs:13-21)."""
    flat = np.asarray(flat, dtype=np.uint64).reshape(m, n, 4)
    return np.ascontiguousarray(flat.transpose(1, 0, 2))


class CommitterKey:
    """com_key (dim generators) and the hiding generator h (hyrax/data_structures.rs), resident on the device with comb
    tables; h is stored as base `dim` so `pedersen_commit(row) + h * r` is one pass."""

    def __init__(self, eng, curve, com_key_xy, h_xy):
        self.eng, self.curve = eng, curve
        com_key_xy = np.asarray(com_key_xy, dtype=np.uint64)
        self.dim = com_key_xy.shape[0]
        self.srs_point_words = com_key_xy.shape[1]
        self.srs = eng.srs_register(curve, np.concatenate([com_key_xy, np.asarray(h_xy, dtype=np.uint64).reshape(1, -1)]),
                                    flags=SRS_COMB)


def pedersen_commit(ck, scalars):
    """hyrax/mod.rs:86-93: MSM of `scalars` (Montgomery Fr) over the first len(scalars) generators."""
    scalars = np.asarray(scalars, dtype=np.uint64).reshape(-1, 4)
    return ck.eng.msm(ck.srs, scalars, flags=SCALARS_MONT)


def commit(ck, evaluations, randomness):
    """hyrax/mod.rs:230-242: evaluations (dim*dim Montgomery Fr, the multilinear polynomial's evaluation vector),
    randomness (dim Montgomery Fr, one r per row) -> (row_coms (dim affine points), mat (dim x dim rows))."""
    dim = ck.dim
    mat = flat_to_matrix_column_major(evaluations, dim, dim)
    rows = np.concatenate([mat, np.asarray(randomness, dtype=np.uint64).reshape(dim, 1, 4)], axis=1)
    row_coms, inf = ck.eng.msm_batch(ck.srs, rows, dim + 1, dim, flags=SCALARS_MONT)
    return row_coms, inf, mat


def open_row_mul(ck, mat, l):
    """lt = mat.row_mul(l)  (hyrax/mod.rs:347): l (dim) times the dim x dim matrix."""
    dim = ck.dim
    return ck.eng.fr_row_mul(ck.curve, l, np.ascontiguousarray(mat).reshape(-1, 4), dim, dim)


def check_t_prime(eng, curve, row_coms_xy, l, row_coms_inf=None):
    """hyrax/mod.rs:498-504: the verifier's multi-exponentiation of the row commitments by the tensor l (Montgomery Fr)."""
    return eng.msm_bases(curve, row_coms_xy, np.asarray(l, dtype=np.uint64).reshape(-1, 4), inf=row_coms_inf, flags=SCALARS_MONT)


class UniversalParams:
    """HyraxUniversalParams (hyrax/data_structures.rs): com_key (dim affine points) and h, host arrays."""

    def __init__(self, curve, com_key_xy, h_xy):
        self.curve, self.com_key_xy, self.h_xy = curve, com_key_xy, h_xy


def setup(eng, curve, num_vars):
    """HyraxPC::setup (hyrax/mod.rs:119-168): dim + 1 hash-derived points, h the last.  BN254 and Pallas only: on BLS12-381 the
    reference clears the cofactor of every point, which pcgpu_g1_sample_generators leaves to the caller."""
    if num_vars % 2:
        raise ValueError("HyraxPC needs an even number of variables (InvalidNumberOfVariables)")
    if curve == BLS12_381:
        raise ValueError("hyrax.setup: BLS12-381 generators need cofactor clearing, which the library leaves to the caller")
    dim = 1 << (num_vars // 2)
    pts = eng.g1_sample_generators(curve, PROTOCOL_NAME, dim + 1)
    return UniversalParams(curve, pts[:dim], pts[dim])


def trim(eng, pp):
    """HyraxPC::trim (hyrax/mod.rs:176-183) clones the parameters into both keys: one device key, com_key || h with comb
    tables, serves as committer and verifier key."""
    ck = CommitterKey(eng, pp.curve, pp.com_key_xy, pp.h_xy)
    return ck, ck


def num_vars_of(ck):
    return 2 * (ck.dim.bit_length() - 1)


def commit_resident(ck, evaluations, randomness, flags=0):
    """HyraxPC::commit of one polynomial on the device: evaluations (2^nv, the to_evaluations() order) and randomness (dim,
    one r per row), Montgomery Fr (device pointers with DEVICE_PTRS) -> (row_coms (dim affine points), identity flags,
    HyraxState holding [T | r] on the device for open)."""
    return ck.eng.hyrax_commit(ck.srs, num_vars_of(ck), evaluations, randomness, flags=flags)


def open(ck, states, point, blinds, challenge):
    """HyraxPC::open (hyrax/mod.rs:273-406) of the committed states at `point` (nv Montgomery Fr).  blinds: per polynomial
    r_eval || d (dim) || r_d || r_b, the order the reference draws them from its rng.  challenge(j, com_eval, com_d, com_b) is
    called in polynomial order with the affine points ((xy, is_identity) pairs) the sponge absorbs and returns c_j
    (Montgomery).  Returns one HyraxProof-shaped dict per polynomial: com_eval, com_d, com_b ((xy, is_identity)), z (dim),
    z_d, z_b, and eval (the polynomial's value at the point)."""
    eng, curve, dim = ck.eng, ck.curve, ck.dim
    point = np.asarray(point, dtype=np.uint64).reshape(-1, 4)
    blinds = np.asarray(blinds, dtype=np.uint64).reshape(len(states), dim + 3, 4)
    coms, inf, lt, ev = eng.hyrax_open(ck.srs, states, point, blinds, nv=point.shape[0])
    proofs = []
    for j in range(len(states)):
        pts = [(coms[j, k], bool(inf[j, k])) for k in range(3)]
        c = np.asarray(challenge(j, *pts), dtype=np.uint64).reshape(4)
        r_eval, d, r_d, r_b = blinds[j, 0], blinds[j, 1:dim + 1], blinds[j, dim + 1], blinds[j, dim + 2]
        proofs.append({"com_eval": pts[0], "com_d": pts[1], "com_b": pts[2],
                       "z": eng.fr_axpy(curve, d, c, lt[j, :dim]),                        # d + c lt, mod.rs:391
                       "z_d": eng.fr_axpy(curve, r_d, c, lt[j, dim]).reshape(4),         # c r_lt + r_d, :392
                       "z_b": eng.fr_axpy(curve, r_b, c, r_eval).reshape(4),             # c r_eval + r_b, :393
                       "eval": ev[j]})
    return proofs


def check(vk, row_coms, point, proofs, challenges):
    """HyraxPC::check (hyrax/mod.rs:418-511) of every proof in one device call.  row_coms: per proof its commitment, (dim affine
    points, identity flags or None); proofs: open's dicts; challenges: per proof c_j (Montgomery).  Returns per-proof booleans;
    the reference's answer is their all()."""
    eng, dim = vk.eng, vk.dim
    point = np.asarray(point, dtype=np.uint64).reshape(-1, 4)
    count = len(proofs)
    limbs = vk.srs_point_words
    rc_xy = np.concatenate([np.asarray(xy, dtype=np.uint64).reshape(dim, limbs) for xy, _ in row_coms]) if count else None
    rc_inf = np.concatenate([np.zeros(dim, np.uint8) if f is None else np.asarray(f, np.uint8).reshape(dim) for _, f in row_coms]) \
        if count else None
    pxy = np.array([[p[k][0] for k in ("com_eval", "com_d", "com_b")] for p in proofs], dtype=np.uint64).reshape(-1, limbs)
    pinf = np.array([[p[k][1] for k in ("com_eval", "com_d", "com_b")] for p in proofs], dtype=np.uint8).reshape(-1)
    zs = np.concatenate([np.concatenate([np.asarray(p["z"], np.uint64).reshape(dim, 4), np.asarray(p["z_d"], np.uint64).reshape(1, 4),
                                         np.asarray(p["z_b"], np.uint64).reshape(1, 4)]) for p in proofs]) if count else None
    ch = np.asarray(challenges, dtype=np.uint64).reshape(count, 4)
    return eng.hyrax_check(vk.srs, point.shape[0], count, rc_xy, point, pxy, zs, ch, row_coms_inf=rc_inf, proof_inf=pinf)
