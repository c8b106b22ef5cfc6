"""Host mirror of KZG10's verifier (poly-commit/src/kzg10/mod.rs) over the C ABI: the G1 combinations on the device MSMs
(SURVEY.md section 8f rank 2, "verifier-side combination MSMs") and the pairings on pcgpu_multi_pairing.

  check_inner          kzg10/mod.rs:322-325   inner = comm - g * value - gamma_g * random_v
  check                kzg10/mod.rs:314-333   e(inner, h) == e(w, beta_h - point * h), as one equation
                                              e(inner, h) * e(-w, beta_h - point * h) == 1
  batch_check_combine  kzg10/mod.rs:345-377   total_c = sum r_i (c_i + z_i w_i) - g * sum r_i v_i - gamma_g * sum r_i rv_i,
                                              total_w = sum r_i w_i; returns normalize_batch([-total_w, total_c])
  batch_check          kzg10/mod.rs:337-391   e(-total_w, beta_h) * e(total_c, h) == 1                  (:382-387)

A verifier key is a dict with the G1 points g, gamma_g and the G2 points h, beta_h (VerifierKey, data_structures.rs:204-220).

The randomizers (u128::rand(rng), :371, the first one fixed to 1, :352) are an argument: they are data to the kernels.
All field elements are (.., 4) uint64 Montgomery Fr; points are Montgomery x||y rows.
"""
import numpy as np

from .binding import G2_OF, SCALARS_MONT, fq_limbs

from .params import FQ_MODULUS, FR_MODULUS


def _neg_limbs(limbs, mod):
    """-x for one field element given as little-endian uint64 limbs (Montgomery form negates like the integer)"""
    limbs = np.asarray(limbs, dtype=np.uint64).reshape(-1)
    v = sum(int(limbs[j]) << (64 * j) for j in range(limbs.size))
    v = (mod - v) % mod
    return np.array([(v >> (64 * j)) & 0xFFFFFFFFFFFFFFFF for j in range(limbs.size)], dtype=np.uint64)


def neg_point(curve, xy):
    n = fq_limbs(curve)
    xy = np.asarray(xy, dtype=np.uint64).reshape(-1).copy()
    xy[n:] = _neg_limbs(xy[n:], FQ_MODULUS[curve])
    return xy


def check_inner(eng, curve, g, gamma_g, comm, value, random_v=None):
    """kzg10/mod.rs:322-325: the G1 argument of the left-hand pairing, comm - g*value - gamma_g*random_v -> (xy, is_identity)"""
    r = FR_MODULUS[curve]
    one = np.zeros(4, dtype=np.uint64)
    one_int = (1 << 256) % r
    for j in range(4):
        one[j] = (one_int >> (64 * j)) & 0xFFFFFFFFFFFFFFFF
    bases = [np.asarray(comm, dtype=np.uint64).reshape(-1), np.asarray(g, dtype=np.uint64).reshape(-1)]
    scalars = [one, _neg_limbs(value, r)]
    if random_v is not None:
        bases.append(np.asarray(gamma_g, dtype=np.uint64).reshape(-1))
        scalars.append(_neg_limbs(random_v, r))
    return eng.msm_bases(curve, np.stack(bases), np.stack(scalars), flags=SCALARS_MONT)


def batch_check_combine(eng, curve, g, gamma_g, commitments, points, values, proofs_w, randomizers, random_vs=None):
    """kzg10/mod.rs:345-377.  commitments / proofs_w: (m, 2*limbs) points; points / values / randomizers: (m, 4) Fr;
    random_vs: (m, 4) Fr or None (no hiding).  Returns ((neg_total_w_xy, is_identity), (total_c_xy, is_identity))."""
    r = FR_MODULUS[curve]
    commitments = np.asarray(commitments, dtype=np.uint64)
    m = commitments.shape[0]
    proofs_w = np.asarray(proofs_w, dtype=np.uint64).reshape(m, -1)
    points, values, rnd = (np.asarray(a, dtype=np.uint64).reshape(m, 4) for a in (points, values, randomizers))
    rz = eng.fr_mul(curve, rnd, points)                                        # randomizer * z_i          (:360, :368)
    g_mult = eng.fr_inner_product(curve, rnd, values)                          # sum randomizer * v_i      (:363)
    bases = [commitments, proofs_w, np.asarray(g, dtype=np.uint64).reshape(1, -1)]
    scalars = [rnd, rz, _neg_limbs(g_mult, r).reshape(1, 4)]
    if random_vs is not None:
        gg_mult = eng.fr_inner_product(curve, rnd, np.asarray(random_vs, dtype=np.uint64).reshape(m, 4))   # (:364-366)
        bases.append(np.asarray(gamma_g, dtype=np.uint64).reshape(1, -1))
        scalars.append(_neg_limbs(gg_mult, r).reshape(1, 4))
    total_c = eng.msm_bases(curve, np.concatenate(bases), np.concatenate(scalars), flags=SCALARS_MONT)       # (:368, :373-374)
    total_w = eng.msm_bases(curve, proofs_w, rnd, flags=SCALARS_MONT)                                        # (:369)
    neg_w = (np.zeros_like(total_w[0]), True) if total_w[1] else (neg_point(curve, total_w[0]), False)
    return neg_w, total_c


def _point(pt):
    """(xy, is_identity) or a bare xy row -> (xy, is_identity)"""
    if isinstance(pt, tuple):
        return np.asarray(pt[0], dtype=np.uint64).reshape(-1), bool(pt[1])
    return np.asarray(pt, dtype=np.uint64).reshape(-1), False


def _one_mont(curve):
    r = FR_MODULUS[curve]
    v = (1 << 256) % r
    return np.array([(v >> (64 * j)) & 0xFFFFFFFFFFFFFFFF for j in range(4)], dtype=np.uint64)


def pairing_is_one(eng, curve, g1_points, g2_points):
    """prod_i e(g1_points[i], g2_points[i]) == 1 as one equation of pcgpu_multi_pairing; points are (xy, is_identity) pairs"""
    g1 = np.stack([xy for xy, _ in g1_points])
    g2 = np.stack([xy for xy, _ in g2_points])
    g1_inf = np.array([inf for _, inf in g1_points], dtype=np.uint8)
    g2_inf = np.array([inf for _, inf in g2_points], dtype=np.uint8)
    _, one = eng.multi_pairing(curve, g1, g2, len(g1_points), g1_inf=g1_inf, g2_inf=g2_inf)
    return bool(one[0])


def check(eng, curve, vk, comm, point, value, proof_w, random_v=None):
    """KZG10::check (kzg10/mod.rs:314-333): comm and proof_w are G1 xy rows or (xy, is_identity); point, value, random_v:
    (4,) Montgomery Fr.  The G2 side beta_h - point * h is one two-term G2 MSM."""
    comm, _ = _point(comm)
    w_xy, w_inf = _point(proof_w)
    inner = check_inner(eng, curve, vk["g"], vk["gamma_g"], comm, value, random_v)
    h = np.asarray(vk["h"], dtype=np.uint64).reshape(-1)
    rhs_g2 = eng.msm_bases(G2_OF[curve], np.stack([np.asarray(vk["beta_h"], dtype=np.uint64).reshape(-1), h]),
                           np.stack([_one_mont(curve), _neg_limbs(point, FR_MODULUS[curve])]), flags=SCALARS_MONT)
    neg_w = (np.zeros_like(w_xy), True) if w_inf else (neg_point(curve, w_xy), False)
    return pairing_is_one(eng, curve, [inner, neg_w], [(h, False), rhs_g2])


def batch_check(eng, curve, vk, commitments, points, values, proofs_w, randomizers, random_vs=None):
    """KZG10::batch_check (kzg10/mod.rs:337-391) with the randomizers as an argument (batch_check_combine)"""
    neg_w, total_c = batch_check_combine(eng, curve, vk["g"], vk["gamma_g"], commitments, points, values, proofs_w, randomizers,
                                         random_vs)
    return pairing_is_one(eng, curve, [neg_w, total_c], [(np.asarray(vk["beta_h"], dtype=np.uint64).reshape(-1), False),
                                                          (np.asarray(vk["h"], dtype=np.uint64).reshape(-1), False)])
