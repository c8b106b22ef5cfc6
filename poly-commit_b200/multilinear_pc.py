"""MultilinearPC, the multilinear KZG of XZZPD19 (poly-commit/src/multilinear_pc/mod.rs), over the C ABI.

  setup   :28-86    pp_powers from eq(t, x); powers_of_g = g.batch_mul(pp_powers) (pcgpu_g1_fixed_base_mul), powers_of_h =
                    h.batch_mul(pp_powers) (pcgpu_g2_fixed_base_mul), g_mask = g.batch_mul(t)
  trim    :91-111   drop the first num_vars - nv levels
  commit  :114-128  one G1 MSM over powers_of_g[0] with the evaluations as scalars (pcgpu_msm, SCALARS_MONT)
  open    :131-168  fold chain and nv G2 MSMs on the device (pcgpu_mlpc_open over a key with pair-folded powers_of_h)
  check   :172-200  e(comm - g value, h) == prod_i e(g_mask_i - point_i g, proof_i), as one equation of nv + 1 pairs
                    e(comm - g value, h) * prod_i e(point_i g - g_mask_i, proof_i) == 1 (G1 side: pcgpu_msm_bases)

The reference samples t, g and h from its RNG; here they are inputs (the Rust RNG is not reproducible outside Rust).  Scalars
are plain ints below r (t) or (.., 4) uint64 Montgomery Fr (evaluations, point); points are Montgomery limb rows.
"""
import numpy as np

from .binding import G2_OF, SCALARS_MONT
from .params import FR_MODULUS

_U64 = 0xFFFFFFFFFFFFFFFF


def eq_extension(t, r):
    """eq_extension (:218-234): nv tables of 2^nv values, table i = t_i x_i + t_i x_i - x_i - t_i + 1 over x in {0,1}^nv"""
    dim = len(t)
    out = []
    for i in range(dim):
        ti = t[i]
        out.append([(2 * ti * ((x >> i) & 1) - ((x >> i) & 1) - ti + 1) % r for x in range(1 << dim)])
    return out


def remove_dummy_variable(poly, pad):
    """remove_dummy_variable (:203-214): fix the first `pad` variables to zero"""
    if pad == 0:
        return list(poly)
    nv = (len(poly) - 1).bit_length() - pad
    return [poly[x << pad] for x in range(1 << nv)]


def pp_powers(t, r):
    """The scalars setup multiplies g and h by (:39-59), level 0 first, 2^(nv-i) values for level i.  Level i is
    remove_dummy_variable(prod_{j >= i} eq_j, i): entry y = prod_{j >= i} (t_j if bit j - i of y else 1 - t_j).  Built here
    by doubling the table once per variable (2^(nv+1) products instead of nv 2^nv); equal, value for value, to the
    reference's construction (eq_extension / remove_dummy_variable above; tests/test_multilinear_pc.py checks it)."""
    nv = len(t)
    out = []
    for i in range(nv):
        tab = [1]
        for j in range(i, nv):
            tab = [v * (1 - t[j]) % r for v in tab] + [v * t[j] % r for v in tab]
        out.extend(tab)
    return out


def _fr_limbs(vals):
    a = np.zeros((len(vals), 4), dtype=np.uint64)
    for i, v in enumerate(vals):
        for j in range(4):
            a[i, j] = (v >> (64 * j)) & 0xFFFFFFFFFFFFFFFF
    return a


def setup(eng, curve, t, g_xy, h_xy):
    """UniversalParams for num_vars = len(t) >= 1 from the trapdoor t (ints below r) and the generators g (G1) and h (G2)"""
    nv = len(t)
    if nv == 0:
        raise ValueError("constant polynomial not supported")
    r = FR_MODULUS[curve]
    scalars = _fr_limbs(pp_powers(t, r))
    pp_g = eng.fixed_base_mul(curve, g_xy, scalars)
    pp_h = eng.g2_fixed_base_mul(G2_OF[curve], h_xy, scalars)
    powers_of_g, powers_of_h, start = [], [], 0
    for i in range(nv):
        size = 1 << (nv - i)
        powers_of_g.append(pp_g[start:start + size])
        powers_of_h.append(pp_h[start:start + size])
        start += size
    g_mask = eng.fixed_base_mul(curve, g_xy, _fr_limbs(t))
    return dict(num_vars=nv, g=np.asarray(g_xy, dtype=np.uint64), h=np.asarray(h_xy, dtype=np.uint64), g_mask=g_mask,
                powers_of_g=powers_of_g, powers_of_h=powers_of_h)


def trim(params, supported_num_vars):
    """(committer key, verifier key) for polynomials in supported_num_vars variables"""
    if not 1 <= supported_num_vars <= params["num_vars"]:
        raise ValueError("supported_num_vars must be in 1..=num_vars")
    k = params["num_vars"] - supported_num_vars
    ck = dict(nv=supported_num_vars, g=params["g"], h=params["h"], powers_of_g=params["powers_of_g"][k:],
              powers_of_h=params["powers_of_h"][k:])
    vk = dict(nv=supported_num_vars, g=params["g"], h=params["h"], g_mask_random=params["g_mask"][k:])
    return ck, vk


class Committer:
    """A committer key on the device: the G1 key of powers_of_g[0] (commit) and the pair-folded G2 levels (open)."""

    def __init__(self, eng, curve, ck):
        self.eng, self.curve, self.nv = eng, curve, ck["nv"]
        self.g_srs = eng.srs_register(curve, ck["powers_of_g"][0])
        self.h_key = eng.mlpc_register(curve, ck["powers_of_h"])

    def commit(self, evals):
        """Commitment.g_product: (xy, is_identity) of sum_x evals[x] powers_of_g[0][x]"""
        return self.eng.msm(self.g_srs, evals, flags=SCALARS_MONT)

    def open(self, evals, point):
        """Proof.proofs as (nv, 4*limbs) uint64 with identity flags, and p(point) (Montgomery Fr)"""
        return self.eng.mlpc_open(self.h_key, evals, point)

    def release(self):
        self.g_srs.release()
        self.h_key.release()


def check(eng, curve, vk, comm, point, value, proofs):
    """MultilinearPC::check (:172-200).  vk from trim; comm: Commitment.g_product as xy or (xy, is_identity); point: (nv, 4)
    Montgomery Fr; value: (4,) Montgomery Fr; proofs: (proofs_xy (nv, 4*limbs), identity flags (nv,) or None) as
    Committer.open returns them."""
    r = FR_MODULUS[curve]

    def neg(x):
        v = sum(int(w) << (64 * j) for j, w in enumerate(np.asarray(x, dtype=np.uint64).reshape(-1)))
        v = (r - v) % r
        return np.array([(v >> (64 * j)) & _U64 for j in range(4)], dtype=np.uint64)

    one = np.array([((1 << 256) % r >> (64 * j)) & _U64 for j in range(4)], dtype=np.uint64)
    nv = vk["nv"]
    g = np.asarray(vk["g"], dtype=np.uint64).reshape(-1)
    comm_xy = np.asarray(comm[0] if isinstance(comm, tuple) else comm, dtype=np.uint64).reshape(-1)
    point = np.asarray(point, dtype=np.uint64).reshape(nv, 4)
    g1 = [eng.msm_bases(curve, np.stack([comm_xy, g]), np.stack([one, neg(value)]), flags=SCALARS_MONT)]
    for i in range(nv):
        mask = np.asarray(vk["g_mask_random"][i], dtype=np.uint64).reshape(-1)
        g1.append(eng.msm_bases(curve, np.stack([mask, g]), np.stack([neg(one), point[i]]), flags=SCALARS_MONT))
    proofs_xy = np.asarray(proofs[0], dtype=np.uint64).reshape(nv, -1)
    pinf = np.zeros(nv, dtype=np.uint8) if len(proofs) < 2 or proofs[1] is None else np.asarray(proofs[1], dtype=np.uint8)
    g2 = np.concatenate([np.asarray(vk["h"], dtype=np.uint64).reshape(1, -1), proofs_xy])
    g1_xy = np.stack([xy for xy, _ in g1])
    g1_inf = np.array([inf for _, inf in g1], dtype=np.uint8)
    _, ok = eng.multi_pairing(curve, g1_xy, g2, nv + 1, g1_inf=g1_inf, g2_inf=np.concatenate([[0], pinf]).astype(np.uint8))
    return bool(ok[0])
