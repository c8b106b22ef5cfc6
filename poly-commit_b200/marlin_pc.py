"""Host mirror of MarlinKZG10's prover calls (poly-commit/src/marlin/marlin_pc/mod.rs) over the C ABI, hiding and
degree-bound branches included.

  CommitterKey.powers / shifted_powers     marlin_pc/data_structures.rs:46-84
  shift_polynomial                          marlin_pc/mod.rs:34-53
  commit   (per-polynomial loop)            marlin_pc/mod.rs:172-242   -> KZG10::commit (+ shifted commitment for a degree bound),
                                                                          each with its own blinding polynomial when hiding
  open     (challenge-weighted combination) marlin_pc/mod.rs:245-336   -> p += (challenge_j, poly_j) :286, r += (challenge_j, rand) :287,
                                                                          witness :292-297, shifted_w / shifted_r / shifted_r_witness
                                                                          :300-307, KZG10::open :310, shifted opening :317-326

Verifier side (the G1 combinations on device MSMs, the pairings on pcgpu_multi_pairing):
  check        marlin_pc/mod.rs:340-364   accumulate_commitments_and_values, then KZG10::check
  batch_check  marlin_pc/mod.rs:366-398   combine_and_normalize (marlin/mod.rs:151-219), then KZG10::batch_check

The opening challenges are squeezed from a Poseidon sponge in the reference (:282, :299) and the blinding polynomials are
sampled from its RNG (kzg10/mod.rs:182-195); here both are arguments (sponge and RNG are out of scope, SURVEY.md section 2)
-- they are data to the kernels.  Polynomials are (n, 4) uint64 arrays of Montgomery Fr coefficients, low degree first.
The accumulators of `open` live in device buffers (binding.DeviceBuffer): every polynomial is uploaded once, the combined
polynomials never cross PCIe, and each witness is computed once.
"""
import numpy as np

from .binding import DEVICE_PTRS, SCALARS_MONT
from .params import fq_mont


class CommitterKey:
    def __init__(self, eng, curve, powers_xy, shifted_powers_xy=None, enforced_degree_bounds=None, flags=0, powers_of_gamma_g_xy=None):
        self.eng, self.curve = eng, curve
        self.powers = eng.srs_register(curve, powers_xy, flags=flags)                      # powers_of_g[0 ..= supported_degree]
        # powers_of_gamma_g (hiding): shared by powers() and shifted_powers() (data_structures.rs:48-53, :78-82)
        self.gamma = eng.srs_register(curve, powers_of_gamma_g_xy) if powers_of_gamma_g_xy is not None else None
        self.enforced_degree_bounds = sorted(enforced_degree_bounds) if enforced_degree_bounds else None
        self.shifted = eng.srs_register(curve, shifted_powers_xy, flags=flags) if shifted_powers_xy is not None else None

    def supported_degree(self):
        return len(self.powers) - 1

    def shifted_offset(self, degree_bound):
        """shifted_powers(bound) = shifted_powers[(max_bound - bound)..]   (data_structures.rs:56-83)."""
        if self.shifted is None:
            raise ValueError("UnsupportedDegreeBound")
        if degree_bound is None:
            return 0
        if degree_bound not in self.enforced_degree_bounds:
            raise ValueError("UnsupportedDegreeBound")
        return self.enforced_degree_bounds[-1] - degree_bound


def _degree(coeffs):
    nz = np.nonzero(np.asarray(coeffs, dtype=np.uint64).reshape(-1, 4).any(axis=1))[0]
    return int(nz[-1]) if nz.size else 0


def shift_polynomial(ck, p, degree_bound):
    """marlin_pc/mod.rs:34-53: prepend (largest enforced bound - degree_bound) zero coefficients."""
    p = np.asarray(p, dtype=np.uint64).reshape(-1, 4)
    if not p.any():
        return np.zeros((0, 4), dtype=np.uint64)
    pad = ck.enforced_degree_bounds[-1] - degree_bound
    return np.concatenate([np.zeros((pad, 4), dtype=np.uint64), p])


def _blind(rands, i, key):
    if rands is None or rands[i] is None:
        return None
    b = rands[i].get(key)
    return None if b is None else np.asarray(b, dtype=np.uint64).reshape(-1, 4)


def commit(ck, polynomials, rands=None):
    """polynomials: list of (coeffs, degree_bound or None); rands: None (non-hiding) or per polynomial None / a dict with the
    blinding polynomials `rand` and (with a degree bound) `shifted_rand` -- Randomness { rand, shifted_rand },
    marlin_pc/data_structures.rs.  Returns [(comm, shifted_comm or None)] as (xy, inf) pairs."""
    out = []
    for i, (coeffs, bound) in enumerate(polynomials):
        if bound is not None and (bound < _degree(coeffs) or bound not in (ck.enforced_degree_bounds or [])):
            raise ValueError("IncorrectDegreeBound")                                  # check_degrees_and_bounds, kzg10/mod.rs:424-450
        rnd, srnd = _blind(rands, i, "rand"), _blind(rands, i, "shifted_rand")
        comm = ck.eng.kzg_commit(ck.powers, coeffs, powers_of_gamma_g=ck.gamma, blind=rnd)        # :217
        shifted = None
        if bound is not None:                                                         # :219-225: KZG10::commit over shifted_powers(bound)
            c = np.asarray(coeffs, dtype=np.uint64).reshape(-1, 4)
            parts = [ck.eng.msm_partial(ck.shifted, c, base_offset=ck.shifted_offset(bound), flags=SCALARS_MONT)]
            if srnd is not None:
                parts.append(ck.eng.msm_partial(ck.gamma, srnd, flags=SCALARS_MONT))
            shifted = ck.eng.g1_sum_xyzz(ck.curve, np.concatenate(parts))
        out.append((comm, shifted))
    return out


def _affine_as_xyzz(curve, xy, is_identity):
    """an affine point as an XYZZ partial (ZZ = ZZZ = 1; the identity is ZZ = 0) for pcgpu_g1_sum_xyzz"""
    nq = xy.size // 2
    out = np.zeros(4 * nq, dtype=np.uint64)
    if not is_identity:
        out[:2 * nq] = xy
        out[2 * nq:3 * nq] = out[3 * nq:] = fq_mont(curve, 1)
    return out


def open(ck, polynomials, point, challenges, rands=None):
    """polynomials / rands as in commit; challenges: iterator of Montgomery Fr (one per polynomial, one more per degree bound).
    Returns the proof (w_xy, w_is_identity, random_v or None)."""
    eng, cid = ck.eng, ck.curve
    ch = iter(challenges)
    polys = [(np.asarray(c, dtype=np.uint64).reshape(-1, 4), b) for c, b in polynomials]
    nmax = max([c.shape[0] for c, _ in polys] + [1])
    hiding = rands is not None and any(r is not None for r in rands)
    rmax = max([_blind(rands, i, k).shape[0] for i in range(len(polys)) for k in ("rand", "shifted_rand") if _blind(rands, i, k) is not None] + [1])
    F = DEVICE_PTRS
    d_p, d_tmp = eng.buffer(nmax), eng.buffer(max(nmax, rmax))
    d_r = eng.buffer(rmax) if hiding else None
    bounded = any(b is not None for _, b in polys)
    if bounded:
        top = ck.enforced_degree_bounds[-1]
        d_wit, d_sw = eng.buffer(nmax), eng.buffer(top + 1)
        d_sr = eng.buffer(rmax) if hiding else None
    for i, (coeffs, bound) in enumerate(polys):
        n = coeffs.shape[0]
        cj = next(ch)
        d_tmp.write(coeffs)
        eng.fr_axpy(cid, d_p.ptr(), cj, d_tmp.ptr(), n=n, flags=F)                    # p += (challenge_j, polynomial)     :286
        if bound is not None:
            if n > 1:
                eng.fr_div_linear(cid, d_tmp.ptr(), point, n=n, flags=F, q=d_wit.ptr())    # compute_witness_polynomial     :292-297
            cj1 = next(ch)
            pad = top - bound                                                              # shift_polynomial               :300
            if n > 1:
                eng.fr_axpy(cid, d_sw.ptr(pad), cj1, d_wit.ptr(), n=n - 1, flags=F)       # shifted_w += (challenge_j_1, .) :302
        rnd = _blind(rands, i, "rand")
        if rnd is not None:
            d_tmp.write(rnd)
            eng.fr_axpy(cid, d_r.ptr(), cj, d_tmp.ptr(), n=rnd.shape[0], flags=F)          # r += (challenge_j, &rand.rand)   :287
        srnd = _blind(rands, i, "shifted_rand")
        if bound is not None and srnd is not None:
            d_tmp.write(srnd)
            eng.fr_axpy(cid, d_sr.ptr(), cj1, d_tmp.ptr(), n=srnd.shape[0], flags=F)       # shifted_r += (challenge_j_1, .)  :303
    # KZG10::open(&ck.powers(), &p, point, &r)  :310 -- witness, hiding witness and blind(point) in one device-resident call
    if hiding:
        h = ctypes_open_hiding(eng, ck, d_p.ptr(), nmax, point, d_r.ptr(), rmax)
        w_xy, w_inf, random_v = h
    else:
        w_xy, w_inf, random_v = eng.kzg_open(ck.powers, d_p.ptr(), point, n=nmax, flags=F)
    if not bounded:
        return w_xy, w_inf, random_v
    # open_with_witness_polynomial(&ck.shifted_powers(None), point, &shifted_r, &shifted_w, Some(&shifted_r_witness))  :317-326
    parts = [_affine_as_xyzz(cid, w_xy, w_inf), eng.msm_partial(ck.shifted, d_sw.ptr(), n=top + 1, flags=SCALARS_MONT | F)]
    if hiding:
        # shifted_r_witness = sum_j challenge_j_1 * (shifted_rand_j / (X - point)) = shifted_r / (X - point)   (division is linear)
        _, sv = eng.fr_div_linear(cid, d_sr.ptr(), point, n=rmax, flags=F, q=d_tmp.ptr())
        if rmax > 1:
            parts.append(eng.msm_partial(ck.gamma, d_tmp.ptr(), n=rmax - 1, flags=SCALARS_MONT | F))
        random_v = _fr_add(cid, random_v, sv)                                                # :329-331
    w = eng.g1_sum_xyzz(cid, np.concatenate(parts))                                          # w += shifted_proof.w  :328
    return w[0], w[1], random_v


def ctypes_open_hiding(eng, ck, p_ptr, n, point, r_ptr, n_blind):
    """pcgpu_kzg_open with a device-resident blinding polynomial (the binding's kzg_open sizes `blind` from a numpy array)"""
    import ctypes
    from .binding import _ptr, fq_limbs
    out = np.zeros(2 * fq_limbs(ck.curve), dtype=np.uint64)
    inf = np.zeros(1, dtype=np.uint8)
    rv = np.zeros(4, dtype=np.uint64)
    eng._ck(eng.lib.pcgpu_kzg_open(eng.ctx, ck.powers.handle, ctypes.c_void_p(p_ptr), n, _ptr(np.ascontiguousarray(point, dtype=np.uint64)),
                                   ck.gamma.handle, ctypes.c_void_p(r_ptr), n_blind, DEVICE_PTRS, _ptr(out), _ptr(inf), _ptr(rv)))
    return out, int(inf[0]), rv


def _fr_add(curve, a, b):
    from .params import FR_MODULUS
    r = FR_MODULUS[curve]
    va = sum(int(x) << (64 * j) for j, x in enumerate(np.asarray(a, dtype=np.uint64).reshape(-1)))
    vb = sum(int(x) << (64 * j) for j, x in enumerate(np.asarray(b, dtype=np.uint64).reshape(-1)))
    v = (va + vb) % r                       # Montgomery form adds like the integers
    return np.array([(v >> (64 * j)) & 0xFFFFFFFFFFFFFFFF for j in range(4)], dtype=np.uint64)


def accumulate_commitments_and_values(eng, curve, commitments, values, challenges, shift_powers=None):
    """Marlin::accumulate_commitments_and_values (marlin/mod.rs:109-148), the verifier-side combination:
         combined_comm  = sum_i challenge_i * comm_i + challenge_i' * (shifted_comm_i - value_i * shift_power(bound_i))
         combined_value = sum_i challenge_i * value_i
    commitments: list of (comm_xy, shifted_comm_xy or None, degree_bound or None); values: (m, 4) Montgomery Fr;
    challenges: iterator of Montgomery Fr in the order the sponge yields them (:123, :129-130); shift_powers: {bound: point}
    (VerifierKey::get_shift_power).  One MSM over the commitments (pcgpu_msm_bases); returns ((xy, is_identity), value)."""
    from .kzg10 import _neg_limbs
    from .params import FR_MODULUS
    ch = iter(challenges)
    values = np.asarray(values, dtype=np.uint64).reshape(-1, 4)
    bases, scalars, ch_plain = [], [], []
    for (comm, shifted, bound), v in zip(commitments, values):
        if (bound is None) != (shifted is None):
            raise ValueError("degree bound and shifted commitment must come together")      # assert_eq!, :119
        c = np.asarray(next(ch), dtype=np.uint64).reshape(4)
        bases.append(np.asarray(comm, dtype=np.uint64).reshape(-1)); scalars.append(c); ch_plain.append(c)
        if bound is not None:
            if shift_powers is None or bound not in shift_powers:
                raise ValueError("UnsupportedDegreeBound")                                  # :136
            c1 = np.asarray(next(ch), dtype=np.uint64).reshape(4)
            c1v = eng.fr_mul(curve, c1.reshape(1, 4), v.reshape(1, 4))[0]
            bases += [np.asarray(shifted, dtype=np.uint64).reshape(-1), np.asarray(shift_powers[bound], dtype=np.uint64).reshape(-1)]
            scalars += [c1, _neg_limbs(c1v, FR_MODULUS[curve])]
    combined_value = eng.fr_inner_product(curve, np.stack(ch_plain), values[: len(ch_plain)])
    return eng.msm_bases(curve, np.stack(bases), np.stack(scalars), flags=SCALARS_MONT), combined_value


def check(eng, curve, vk, commitments, point, values, proof, challenges, shift_powers=None):
    """MarlinKZG10::check (marlin_pc/mod.rs:340-364).  vk: the KZG10 verifier key dict (kzg10.check); commitments, values,
    challenges, shift_powers as in accumulate_commitments_and_values; point: (4,) Montgomery Fr; proof: (w_xy or (w_xy,
    is_identity), random_v or None)."""
    from . import kzg10
    comm, value = accumulate_commitments_and_values(eng, curve, commitments, values, challenges, shift_powers)
    return kzg10.check(eng, curve, vk, comm, point, value, proof[0], proof[1])


def batch_check(eng, curve, vk, commitments, query_set, evaluations, proofs, challenges, randomizers, shift_powers=None):
    """MarlinKZG10::batch_check (marlin_pc/mod.rs:366-398).  commitments: {label: (comm_xy, shifted_xy or None, degree_bound or
    None)}; query_set: iterable of (label, (point_label, point)); evaluations: {(label, point_label): value}; proofs: one
    (w, random_v or None) per distinct point label, in point-label order; challenges: the sponge's challenges in the order
    combine_and_normalize draws them; randomizers: one (4,) Montgomery Fr per distinct point (the first is 1 in the reference).
    Queries are grouped by point label and each group's labels taken in sorted order (marlin/mod.rs:151-219)."""
    from . import kzg10
    groups = {}
    for label, (point_label, point) in query_set:
        groups.setdefault(point_label, (point, set()))[1].add(label)
    ch = iter(challenges)
    combined, points, values = [], [], []
    for point_label in sorted(groups):
        point, labels = groups[point_label]
        labels = sorted(labels)
        vals = np.stack([np.asarray(evaluations[(lb, point_label)], dtype=np.uint64).reshape(4) for lb in labels])
        (c_xy, c_inf), v = accumulate_commitments_and_values(eng, curve, [commitments[lb] for lb in labels], vals, ch, shift_powers)
        if c_inf:
            raise ValueError("combined commitment is the identity")
        combined.append(c_xy); points.append(np.asarray(point, dtype=np.uint64).reshape(4)); values.append(np.asarray(v).reshape(4))
    ws = [kzg10._point(w)[0] for w, _ in proofs]
    rvs = [rv for _, rv in proofs]
    hiding = any(rv is not None for rv in rvs)
    random_vs = np.stack([np.zeros(4, dtype=np.uint64) if rv is None else np.asarray(rv, dtype=np.uint64).reshape(4) for rv in rvs]) \
        if hiding else None
    return kzg10.batch_check(eng, curve, vk, np.stack(combined), np.stack(points), np.stack(values), np.stack(ws), randomizers,
                             random_vs)
