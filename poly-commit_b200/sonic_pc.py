"""Host mirror of SonicKZG10 (poly-commit/src/sonic_pc/mod.rs) over the C ABI: keys, hiding commit and open, check and batch_check.

  CommitterKey.shifted_powers      sonic_pc/data_structures.rs:81-114 (shifted_powers(bound) = shifted_powers_of_g[(max_bound -
                                   bound)..] with that bound's own shifted_powers_of_gamma_g)
  VerifierKey.get_shift_power      sonic_pc/data_structures.rs:143-172 (h, beta_h and the neg powers are kept prepared)
  trim                             sonic_pc/mod.rs:159-271
  commit                           sonic_pc/mod.rs:274-337   ONE commitment per polynomial: over shifted_powers(bound) when the
                                                             polynomial carries a degree bound (:319-325), else over powers()
  open                             sonic_pc/mod.rs:340-382   combined_polynomial / combined_rand += (curr_challenge, .) (:373-374),
                                                             then ONE KZG10::open over powers() (:379)
  batch_open                       lib.rs:269-350            the trait's default: one open per distinct point
  check / batch_check              sonic_pc/mod.rs:384-494   accumulate_elems (:39-89) and check_elems (:91-133)

The opening challenges come from a sponge in the reference (:362, :375, :53, :74), the batch_check randomizers from its RNG
(:476) and the blinding polynomials from the commit RNG; here all three are arguments (data to the kernels; the sponge is out
of scope, SURVEY.md section 2).  One challenge is taken per polynomial or commitment, in order: the reference's unused last
squeeze of each open and each accumulate_elems is not represented.  Polynomials are (n, 4) uint64 arrays of Montgomery Fr
coefficients, low degree first.  Differences from MarlinKZG10 (marlin_pc.py): no second "shifted" commitment and no shifted
witness -- a bounded polynomial is committed ONLY against the shifted key, and the verifier pairs each degree-bound group of
commitments with that bound's negative power of h.

The verifier's G1 combinations are device MSMs and its pairing one pcgpu_multi_pairing_prepared equation against the verifier
key's prepared G2 points.
"""
import numpy as np

from . import g2_host
from .binding import SCALARS_MONT
from .kzg10 import _neg_limbs, _one_mont, _point
from .marlin_pc import _degree
from .params import FR_MODULUS


class TrimmingDegreeTooLarge(ValueError):
    """Error::TrimmingDegreeTooLarge"""


class UnsupportedDegreeBound(ValueError):
    """Error::UnsupportedDegreeBound(bound)"""


def _register(eng, curve, pts, flags=0):
    """xy rows or (xy, inf) -> Srs"""
    if isinstance(pts, tuple):
        return eng.srs_register(curve, pts[0], inf=pts[1], flags=flags)
    return eng.srs_register(curve, pts, flags=flags)


class CommitterKey:
    """SonicKZG10's CommitterKey (data_structures.rs:40-68) with every key registered on the device.  powers_of_g,
    shifted_powers_of_g: G1 rows (or (xy, inf)); powers_of_gamma_g: the hiding key of powers(); shifted_powers_of_gamma_g:
    {bound: G1 rows}, one hiding key per enforced bound; max_degree: of the UniversalParams the key was trimmed from."""

    def __init__(self, eng, curve, powers_of_g, shifted_powers_of_g=None, enforced_degree_bounds=None, flags=0, *,
                 powers_of_gamma_g=None, shifted_powers_of_gamma_g=None, max_degree=None):
        self.eng, self.curve = eng, curve
        self.powers_of_g = _register(eng, curve, powers_of_g, flags)
        self.powers_of_gamma_g = _register(eng, curve, powers_of_gamma_g) if powers_of_gamma_g is not None else None
        self.shifted_powers_of_g = _register(eng, curve, shifted_powers_of_g, flags) if shifted_powers_of_g is not None else None
        self.shifted_powers_of_gamma_g = {b: _register(eng, curve, p) for b, p in (shifted_powers_of_gamma_g or {}).items()}
        self.enforced_degree_bounds = sorted(set(enforced_degree_bounds)) if enforced_degree_bounds else None
        self.max_degree = len(self.powers_of_g) - 1 if max_degree is None else max_degree

    @property
    def powers(self):
        """powers().powers_of_g"""
        return self.powers_of_g

    def supported_degree(self):
        return len(self.powers_of_g) - 1

    def shifted_offset(self, degree_bound):
        """the start of shifted_powers(bound) in shifted_powers_of_g: max_bound - bound"""
        if self.shifted_powers_of_g is None or degree_bound not in (self.enforced_degree_bounds or []):
            raise UnsupportedDegreeBound(degree_bound)
        return self.enforced_degree_bounds[-1] - degree_bound

    def shifted_powers(self, degree_bound):
        """shifted_powers(bound) -> (shifted_powers_of_g, offset, that bound's powers_of_gamma_g or None)"""
        return self.shifted_powers_of_g, self.shifted_offset(degree_bound), self.shifted_powers_of_gamma_g.get(degree_bound)


class VerifierKey:
    """SonicKZG10's VerifierKey (data_structures.rs:118-172).  g, gamma_g: G1 rows; h, beta_h: G2 points as g2_host tuples;
    degree_bounds_and_neg_powers_of_h: None or [(bound, G2 point)] (h * beta^-(max_degree - bound)).  The key is always
    prepared: one G2Prepared over [h, beta_h, the neg powers in ascending bound order] is built here."""

    def __init__(self, eng, curve, g, gamma_g, h, beta_h, degree_bounds_and_neg_powers_of_h=None, supported_degree=0, max_degree=0):
        self.eng, self.curve = eng, curve
        self.g, self.gamma_g = np.asarray(g, dtype=np.uint64).reshape(-1), np.asarray(gamma_g, dtype=np.uint64).reshape(-1)
        self.h, self.beta_h = h, beta_h
        self.degree_bounds_and_neg_powers_of_h = sorted(degree_bounds_and_neg_powers_of_h) \
            if degree_bounds_and_neg_powers_of_h is not None else None
        self.supported_degree, self.max_degree = supported_degree, max_degree
        pts = [h, beta_h] + [p for _, p in (self.degree_bounds_and_neg_powers_of_h or [])]
        limbs = [g2_host.g2_to_limbs(curve, p) for p in pts]
        self.prepared = eng.g2_prepare(curve, np.stack([xy for xy, _ in limbs]), np.array([inf for _, inf in limbs], dtype=np.uint8))

    PREPARED_H, PREPARED_BETA_H = 0, 1

    def get_shift_power(self, degree_bound):
        """the index of the bound's prepared neg power of h, or None"""
        for i, (b, _) in enumerate(self.degree_bounds_and_neg_powers_of_h or []):
            if b == degree_bound:
                return 2 + i
        return None


def trim(eng, curve, pp, supported_degree, supported_hiding_bound, enforced_degree_bounds=None):
    """sonic_pc/mod.rs:159-271.  pp: the dict wire.universal_params_deserialize returns.  Returns (CommitterKey, VerifierKey)."""
    g_xy, g_inf = pp["powers_of_g"]
    keys, gam_xy, gam_inf = pp["powers_of_gamma_g"]
    gamma = {int(k): (gam_xy[i], gam_inf[i]) for i, k in enumerate(keys)}
    max_degree = g_xy.shape[0] - 1
    if supported_degree > max_degree:
        raise TrimmingDegreeTooLarge(supported_degree)                                   # :167-169

    def gamma_rows(idx):
        return np.stack([gamma[i][0] for i in idx]), np.array([gamma[i][1] for i in idx], dtype=np.uint8)

    bounds = sorted(set(enforced_degree_bounds)) if enforced_degree_bounds is not None else None
    shifted, shifted_gamma, neg = None, None, None
    if bounds:
        highest = bounds[-1]
        if highest > supported_degree:
            raise UnsupportedDegreeBound(highest)                                        # :183-185
        lowest_shift_degree = max_degree - highest
        shifted = (g_xy[lowest_shift_degree:], g_inf[lowest_shift_degree:])              # :194
        shifted_gamma = {}
        for b in bounds:                                                                 # :196-210
            shift_degree = max_degree - b
            shifted_gamma[b] = gamma_rows([shift_degree + i for i in range(supported_hiding_bound + 2)
                                           if shift_degree + i < max_degree + 2])
        neg = []
        for b in bounds:                                                                 # :219-222
            if max_degree - b not in pp["neg_powers_of_h"]:
                raise UnsupportedDegreeBound(b)
            neg.append((b, pp["neg_powers_of_h"][max_degree - b]))
    ck = CommitterKey(eng, curve, (g_xy[:supported_degree + 1], g_inf[:supported_degree + 1]), shifted, bounds or None,
                      powers_of_gamma_g=gamma_rows(range(supported_hiding_bound + 2)), shifted_powers_of_gamma_g=shifted_gamma,
                      max_degree=max_degree)
    vk = VerifierKey(eng, curve, g_xy[0], gamma[0][0], pp["h"], pp["beta_h"], neg, supported_degree, max_degree)
    return ck, vk


def _check_bound(ck, coeffs, bound):
    if bound is not None and (bound < _degree(coeffs) or bound not in (ck.enforced_degree_bounds or [])):
        raise ValueError("IncorrectDegreeBound")                                         # check_degrees_and_bounds, kzg10/mod.rs:424-450


def _blind(rands, i):
    if rands is None or rands[i] is None:
        return None
    return np.asarray(rands[i], dtype=np.uint64).reshape(-1, 4)


def commit(ck, polynomials, rands=None):
    """polynomials: list of (coeffs, degree_bound or None); rands: None (non-hiding) or per polynomial None / its blinding
    polynomial (Randomness.blinding_polynomial).  Returns [(comm_xy, is_identity)]  (sonic_pc/mod.rs:274-337)."""
    eng, out = ck.eng, []
    for i, (coeffs, bound) in enumerate(polynomials):
        coeffs = np.asarray(coeffs, dtype=np.uint64).reshape(-1, 4)
        _check_bound(ck, coeffs, bound)
        rnd = _blind(rands, i)
        if bound is None:                                                                # ck.powers()
            out.append(eng.kzg_commit(ck.powers_of_g, coeffs, powers_of_gamma_g=ck.powers_of_gamma_g if rnd is not None else None,
                                      blind=rnd))
            continue
        shifted, off, gamma = ck.shifted_powers(bound)                                   # ck.shifted_powers(bound)  :319-321
        if coeffs.shape[0] > len(shifted) - off:
            raise ValueError("TooManyCoefficients")
        if rnd is None:
            out.append(eng.msm(shifted, coeffs, base_offset=off, flags=SCALARS_MONT))
            continue
        if gamma is None or rnd.shape[0] > len(gamma):
            raise ValueError("HidingBoundToolarge")
        parts = [eng.msm_partial(shifted, coeffs, base_offset=off, flags=SCALARS_MONT), eng.msm_partial(gamma, rnd, flags=SCALARS_MONT)]
        xy, inf = eng.g1_sum_xyzz(ck.curve, np.concatenate(parts))                      # KZG10::commit's two MSMs, summed
        out.append((xy, int(inf)))
    return out


def open(ck, polynomials, point, challenges, rands=None):
    """sonic_pc/mod.rs:340-382: one challenge per polynomial (bounded or not), one KZG10 opening of the combination over
    powers(); rands as in commit.  Returns the proof (w_xy, w_is_identity, random_v or None)."""
    eng, cid = ck.eng, ck.curve
    ch = iter(challenges)
    polys = [np.asarray(c, dtype=np.uint64).reshape(-1, 4) for c, _ in polynomials]
    p = np.zeros((max(c.shape[0] for c in polys), 4), dtype=np.uint64)
    blinds = [_blind(rands, i) for i in range(len(polys))]
    hiding = any(b is not None for b in blinds)
    r = np.zeros((max([b.shape[0] for b in blinds if b is not None] + [1]), 4), dtype=np.uint64)
    for coeffs, (_, bound), rnd in zip(polys, polynomials, blinds):
        _check_bound(ck, coeffs, bound)
        c = next(ch)
        p[: coeffs.shape[0]] = eng.fr_axpy(cid, p[: coeffs.shape[0]], c, coeffs)       # combined_polynomial += (challenge, p)  :373
        if rnd is not None:
            r[: rnd.shape[0]] = eng.fr_axpy(cid, r[: rnd.shape[0]], c, rnd)             # combined_rand += (challenge, state)    :374
    if hiding:                                                                           # KZG10::open(&ck.powers(), ..)         :379
        return eng.kzg_open(ck.powers_of_g, p, point, powers_of_gamma_g=ck.powers_of_gamma_g, blind=r)
    w_xy, w_inf, _ = eng.kzg_open(ck.powers_of_g, p, point)
    return w_xy, w_inf, None


def _query_groups(query_set):
    """query_to_labels_map: {point_label: (point, sorted labels)} in point-label order"""
    groups = {}
    for label, (point_label, point) in query_set:
        groups.setdefault(point_label, (point, set()))[1].add(label)
    return [(pl, groups[pl][0], sorted(groups[pl][1])) for pl in sorted(groups)]


def batch_open(ck, polynomials, query_set, challenges, rands=None):
    """The trait's default batch_open (lib.rs:269-350): polynomials {label: (coeffs, degree_bound or None)}; rands None or
    {label: blinding polynomial or None}; query_set: iterable of (label, (point_label, point)); challenges: one iterator over
    every open's challenges in turn.  Returns one proof per distinct point label, in point-label order."""
    ch = iter(challenges)
    proofs = []
    for _, point, labels in _query_groups(query_set):
        polys = [polynomials[lb] for lb in labels]
        rs = None if rands is None else [rands.get(lb) for lb in labels]
        proofs.append(open(ck, polys, point, ch, rs))
    return proofs


def _fr(a):
    return np.asarray(a, dtype=np.uint64).reshape(-1, 4)


def accumulate_elems(eng, curve, acc, commitments, point, values, proof, challenges, randomizer):
    """accumulate_elems (sonic_pc/mod.rs:39-89) for one point, recorded as MSM terms: every commitment with scalar challenge *
    randomizer in its degree-bound group; w with randomizer (combined_witness) and -randomizer * point (adjusted); the
    randomizer-weighted combined value and random_v as scalars of g and gamma_g."""
    ch = iter(challenges)
    values = _fr(values)
    comms, bounds, chals = [], [], []
    for comm, bound in commitments:
        comms.append(_point(comm)); bounds.append(bound); chals.append(np.asarray(next(ch), dtype=np.uint64).reshape(4))
    chals = np.stack(chals)
    combined_value = eng.fr_inner_product(curve, chals, values[: len(comms)])            # combined_values += value * challenge  :60
    scaled = eng.fr_mul(curve, chals, np.tile(randomizer, (len(comms), 1)))              # comm * challenge * randomizer       :65-69
    for c, bound, s in zip(comms, bounds, scaled):
        acc["groups"].setdefault(bound, []).append((c, s))
    w = _point((proof[0], proof[1]))
    rv = proof[2] if len(proof) > 2 else None
    acc["w"].append(w)
    acc["r"].append(randomizer)
    acc["rz"].append(eng.fr_mul(curve, randomizer.reshape(1, 4), np.asarray(point, dtype=np.uint64).reshape(1, 4))[0])
    acc["v"].append(combined_value)
    acc["rv"].append(np.zeros(4, dtype=np.uint64) if rv is None else np.asarray(rv, dtype=np.uint64).reshape(4))
    acc["hiding"] = acc["hiding"] or rv is not None


def new_accumulator():
    """accumulate_elems' state: combined_comms, combined_witness and combined_adjusted_witness as MSM terms"""
    return dict(groups={}, w=[], r=[], rz=[], v=[], rv=[], hiding=False)


def _msm(eng, curve, terms):
    """sum of s * P over terms [((xy, is_identity), s)] -> (xy, is_identity)"""
    bases = np.stack([xy for (xy, _), _ in terms])
    inf = np.array([i for (_, i), _ in terms], dtype=np.uint8)
    return eng.msm_bases(curve, bases, np.stack([s for _, s in terms]), inf=inf, flags=SCALARS_MONT)


def equation(eng, curve, vk, acc):
    """check_elems (sonic_pc/mod.rs:91-133) up to the pairing: the G1 arguments [combined comm of each degree-bound group
    (None first, then ascending bounds), -combined_adjusted_witness, -combined_witness] and the prepared-point indices
    [h or the bound's shift power, h, beta_h]"""
    r = FR_MODULUS[curve]
    g1, idx = [], []
    for bound in sorted(acc["groups"], key=lambda b: -1 if b is None else b):
        q = VerifierKey.PREPARED_H if bound is None else vk.get_shift_power(bound)
        if q is None:
            raise UnsupportedDegreeBound(bound)                                          # :105-107
        g1.append(_msm(eng, curve, acc["groups"][bound])); idx.append(q)
    rs = np.stack(acc["r"])
    neg = lambda a: _neg_limbs(a, r)                                                     # noqa: E731
    # -(g * sum r_j v_j - sum r_j z_j w_j + gamma_g * sum r_j rv_j): the negation is taken on the scalars
    adj = [((vk.g, False), neg(eng.fr_inner_product(curve, rs, np.stack(acc["v"]))))]
    adj += [(w, rz) for w, rz in zip(acc["w"], acc["rz"])]
    if acc["hiding"]:
        adj.append(((vk.gamma_g, False), neg(eng.fr_inner_product(curve, rs, np.stack(acc["rv"])))))
    g1.append(_msm(eng, curve, adj)); idx.append(VerifierKey.PREPARED_H)
    g1.append(_msm(eng, curve, [(w, neg(rj)) for w, rj in zip(acc["w"], acc["r"])])); idx.append(VerifierKey.PREPARED_BETA_H)
    return g1, idx


def _pairing_is_one(eng, curve, vk, g1, idx):
    xy = np.stack([p for p, _ in g1])
    inf = np.array([i for _, i in g1], dtype=np.uint8)
    _, one = eng.multi_pairing_prepared(curve, xy, vk.prepared, np.array(idx, dtype=np.uint32), len(g1), g1_inf=inf)
    return bool(one[0])


def check(eng, curve, vk, commitments, point, values, proof, challenges):
    """SonicKZG10::check (sonic_pc/mod.rs:384-415).  commitments: [(comm, degree_bound or None)] with comm an xy row or (xy,
    is_identity); values: (m, 4) Montgomery Fr; proof: what open returns, (w_xy, w_is_identity, random_v or None);
    challenges: one per commitment."""
    acc = new_accumulator()
    accumulate_elems(eng, curve, acc, commitments, point, values, proof, challenges, _one_mont(curve))
    return _pairing_is_one(eng, curve, vk, *equation(eng, curve, vk, acc))


def batch_check(eng, curve, vk, commitments, query_set, evaluations, proofs, challenges, randomizers):
    """SonicKZG10::batch_check (sonic_pc/mod.rs:417-494).  commitments: {label: (comm, degree_bound or None)}; query_set:
    iterable of (label, (point_label, point)); evaluations: {(label, point_label): value}; proofs: one per distinct point label,
    in point-label order (what batch_open returns); challenges: one iterator over every point's challenges in turn;
    randomizers: one (4,) Montgomery Fr per distinct point, the first 1 as in the reference (:457)."""
    groups = _query_groups(query_set)
    if len(proofs) != len(groups):
        raise ValueError("one proof per queried point")                                  # assert_eq!, :455
    ch = iter(challenges)
    acc = new_accumulator()
    for (point_label, point, labels), proof, rnd in zip(groups, proofs, randomizers):
        vals = np.stack([np.asarray(evaluations[(lb, point_label)], dtype=np.uint64).reshape(4) for lb in labels])
        accumulate_elems(eng, curve, acc, [commitments[lb] for lb in labels], point, vals, proof, ch,
                    np.asarray(rnd, dtype=np.uint64).reshape(4))
    return _pairing_is_one(eng, curve, vk, *equation(eng, curve, vk, acc))

