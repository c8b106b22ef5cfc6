"""Prepared G2 points (pcgpu_g2_prepare, pcgpu_multi_pairing_prepared) and the SonicKZG10 scheme built on them (sonic_pc.trim,
commit / open with hiding and degree bounds, batch_open, check, batch_check, the verifier key's wire format) on BLS12-381 and
BN254: one set of case bodies, run on the host-emulated kernels and, under -m gpu, on the device.

References: pcgpu_multi_pairing on the same points (bit-exact GT values), tests/pairing_ref.py (an independent pairing), and a
Python Sonic verifier from pyref curve arithmetic that restates accumulate_elems / check_elems (sonic_pc/mod.rs:39-133).
"""
import ctypes
import struct

import numpy as np
import pytest

from oracle import orc, pyref
from tests import g2_cases as gc
from tests import util
from tests.pairing_ref import Pairing

PAIRING = gc.PAIRING
_REF = {}


def ref(cname):
    if cname not in _REF:
        _REF[cname] = Pairing(cname)
    return _REF[cname]


@pytest.fixture(scope="module")
def emul(pc, hostcheck_path):
    e = pc.Engine(0, lib_path=hostcheck_path)
    yield e
    e.close()


def g1_limbs(cname, pts):
    return pyref.Curve(cname).points_to_limbs(pts)


def fr_canon(cname, vals):
    return gc.fr_limbs([v % pyref.Curve(cname).r for v in vals])


def fr_int(cname, limbs):
    return pyref.Curve(cname).fr_from_limbs(np.asarray(limbs, dtype=np.uint64).reshape(-1, 4), True)[0]


# ---- prepared pairing ----------------------------------------------------------------------------------------------------
def prepared_case(eng, cname, seed=3):
    """k = 0 .. 3 with identities in either slot (an identity flag and the all-zero encoding), one prepared point used by
    several pairs and several equations: GT values equal multi_pairing's on the same points and the oracle's"""
    E, C = ref(cname), pyref.Curve(cname)
    H = gc.generator(cname)
    g = util.rng(seed)
    ks = [int(v) for v in g.integers(2, 1 << 30, size=6)]
    Ps = [C.mul(k, C.g) for k in ks[:3]]
    Qs = [E.G2.mul(k, H) for k in ks[3:]] + [None]                       # index 3: the identity
    q_xy, q_inf = gc.to_limbs(cname, Qs)
    prep = eng.g2_prepare(C.id, q_xy, q_inf)
    zero_enc = eng.g2_prepare(C.id, q_xy)                                 # no flags: index 3 is the all-zero encoding
    assert len(prep) == 4
    cases = [([Ps[0]], [0]), ([Ps[0], None], [0, 1]), ([Ps[0], Ps[1], Ps[2]], [0, 3, 2]), ([C.neg(Ps[0]), Ps[0]], [1, 1]),
             ([Ps[1], Ps[2], Ps[0]], [2, 2, 2])]
    for Ps_, idx in cases:
        k = len(Ps_)
        g1, g1i = g1_limbs(cname, Ps_)
        exp = E.multi_pairing(Ps_, [Qs[i] for i in idx])
        plain, plain_one = eng.multi_pairing(C.id, g1, q_xy[idx], k, g1_inf=g1i, g2_inf=q_inf[idx])
        for h in (prep, zero_enc):
            gt, one = eng.multi_pairing_prepared(C.id, g1, h, idx, k, g1_inf=g1i)
            assert (gt == plain).all() and (one == plain_one).all(), (cname, idx)
            assert E.from_limbs(gt) == [exp] and list(one) == [int(exp == E.ONE)], (cname, idx)
    gt, one = eng.multi_pairing_prepared(C.id, None, prep, None, 0, count=2)      # k = 0: the identity
    assert E.from_limbs(gt) == [E.ONE, E.ONE] and list(one) == [1, 1]
    # three equations of two pairs, prepared point 0 in four of the six pairs
    idx = [0, 0, 0, 1, 2, 0]
    g1, _ = g1_limbs(cname, [Ps[0], Ps[1], Ps[2], Ps[0], Ps[1], C.neg(Ps[1])])
    gt, one = eng.multi_pairing_prepared(C.id, g1, prep, idx, 2)
    plain, plain_one = eng.multi_pairing(C.id, g1, q_xy[idx], 2)
    assert (gt == plain).all() and (one == plain_one).all()
    assert E.from_limbs(gt)[1] == E.multi_pairing([Ps[2], Ps[0]], [Qs[0], Qs[1]])
    prep.release()
    zero_enc.release()


def honest_bn254_case(eng, pc):
    """an honest BN254 equation e(ab P, Q) e(-P, ab Q) = 1 through prepared points: the loop's pi(Q) and -pi^2(Q) lines are
    right, or the product would not be one"""
    cname = "bn254"
    C = pyref.Curve(cname)
    a, b = 0x1234567890abcdef, 0xfedcba987654321
    H, _ = gc.to_limbs(cname, [gc.generator(cname)])
    Q = eng.g2_fixed_base_mul(gc.group(pc, cname), H[0], fr_canon(cname, [1, a * b]))
    prep = eng.g2_prepare(C.id, Q)
    g1, _ = g1_limbs(cname, [C.mul(a * b, C.g), C.neg(C.g), C.g, C.g])
    _, one = eng.multi_pairing_prepared(C.id, g1, prep, [0, 1, 0, 1], 2)
    assert list(one) == [1, 0]
    prep.release()


def prepared_errors_case(eng, pc, cname):
    """an index out of range, a handle of the other curve, Pallas and G2 ids, k = 65, both outputs NULL, bad flags: BADARG
    before anything runs; *out is cleared on bad arguments"""
    C = pyref.Curve(cname)
    other = "bn254" if cname == "bls12_381" else "bls12_381"
    g1, _ = g1_limbs(cname, [C.g])
    H, _ = gc.to_limbs(cname, [gc.generator(cname)])
    Ho, _ = gc.to_limbs(other, [gc.generator(other)])
    prep = eng.g2_prepare(C.id, H)
    prep_other = eng.g2_prepare(pyref.Curve(other).id, Ho)

    def badarg(f):
        with pytest.raises(pc.PcgpuError) as e:
            f()
        assert e.value.code == -3

    badarg(lambda: eng.multi_pairing_prepared(C.id, g1, prep, [1], 1))
    badarg(lambda: eng.multi_pairing_prepared(C.id, np.tile(g1, (2, 1)), prep, [0, 7], 2))
    badarg(lambda: eng.multi_pairing_prepared(C.id, g1, prep_other, [0], 1))
    for curve in (2, gc.group(pc, cname)):
        badarg(lambda: eng.g2_prepare(curve, H))
        badarg(lambda: eng.multi_pairing_prepared(curve, g1, prep, [0], 1))
    badarg(lambda: eng.multi_pairing_prepared(C.id, np.tile(g1, (65, 1)), prep, [0] * 65, 65))
    badarg(lambda: eng.multi_pairing_prepared(C.id, g1, prep, [0], 1, flags=1 << 7))
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)                              # noqa: E731
    idx = np.zeros(1, dtype=np.uint32)
    assert eng.lib.pcgpu_multi_pairing_prepared(eng.ctx, C.id, p(g1), None, prep.handle, p(idx), 1, 1, 0, None, None) == -3
    assert eng.lib.pcgpu_multi_pairing_prepared(eng.ctx, C.id, p(g1), None, None, p(idx), 1, 1, 0, None, p(idx)) == -3
    out = np.zeros(1, dtype=np.uint8)
    assert eng.lib.pcgpu_multi_pairing_prepared(eng.ctx, C.id, None, None, prep.handle, None, 1, 0, 0, None, p(out)) == 0
    for curve, ptr, n, flags in ((2, p(H), 1, 0), (gc.group(pc, cname), p(H), 1, 0), (C.id, None, 1, 0), (C.id, p(H), 1, 1 << 7)):
        h = ctypes.c_void_p(0x1234)
        assert eng.lib.pcgpu_g2_prepare(eng.ctx, curve, ptr, None, n, flags, ctypes.byref(h)) == -3
        assert h.value is None
    assert eng.lib.pcgpu_g2_prepare(eng.ctx, C.id, p(H), None, 1, 0, None) == -3
    prep.release()
    prep_other.release()


# ---- Sonic keys from a known beta ------------------------------------------------------------------------------------------
class SonicKeys:
    """UniversalParams from a known beta (powers beta^i G, the gamma powers trim reads, h, beta_h and the neg powers
    h * beta^-(max_degree - bound)), run through wire.universal_params_serialize / _deserialize and sonic_pc.trim"""

    def __init__(self, eng, pc, cname, max_degree, supported, hiding_bound, bounds, seed=1):
        from poly_commit_b200 import sonic_pc, wire
        C = pyref.Curve(cname)
        self.eng, self.cname, self.id, r = eng, cname, C.id, C.r
        beta_m = util.rand_fr(cname, 1, 1000 + seed, mont=True)[0]
        beta = fr_int(cname, beta_m)
        gamma = util.rand_fr_ints(cname, 1, 1500 + seed)[0]
        G = orc.g1_generator(C.id)
        powers = eng.fixed_base_mul(C.id, G, orc.fr_powers_canonical(C.id, beta_m, max_degree + 1))
        keys = sorted(set(range(hiding_bound + 2)) | {max_degree - b + i for b in bounds for i in range(hiding_bound + 2)
                                                         if max_degree - b + i < max_degree + 2})
        gG = eng.fixed_base_mul(C.id, G, fr_canon(cname, [gamma]))[0]
        gamma_xy = eng.fixed_base_mul(C.id, gG, fr_canon(cname, [pow(beta, k, r) for k in keys]))
        H, _ = gc.to_limbs(cname, [gc.generator(cname)])
        g2 = eng.g2_fixed_base_mul(gc.group(pc, cname), H[0],
                                   fr_canon(cname, [beta] + [pow(beta, -(max_degree - b), r) for b in bounds]))
        self.h, self.beta_h = gc.generator(cname), gc.from_limbs(cname, g2[0])
        neg = {max_degree - b: gc.from_limbs(cname, row) for b, row in zip(bounds, g2[1:])}
        data = wire.universal_params_serialize(eng, C.id, powers, np.array(keys, dtype=np.uint64), gamma_xy, self.h, self.beta_h, neg)
        pp = wire.universal_params_deserialize(eng, C.id, data)
        self.ck, self.vk = sonic_pc.trim(eng, C.id, pp, supported, hiding_bound, bounds)
        self.powers, self.max_degree = powers, max_degree

    def value(self, coeffs, z):
        return self.eng.fr_div_linear(self.id, coeffs, z)[1]

    def prove(self, polys, rands, point, seed):
        """commit + open; returns (commitments [(comm, bound)], values, proof, challenges)"""
        from poly_commit_b200 import sonic_pc
        coms = sonic_pc.commit(self.ck, polys, rands)
        chals = list(util.rand_fr(self.cname, len(polys), seed, mont=True))
        proof = sonic_pc.open(self.ck, polys, point, chals, rands)
        vals = np.stack([self.value(c, point) for c, _ in polys])
        return [(c, b) for c, (_, b) in zip(coms, polys)], vals, proof, chals


def poly_sets(cname, seed, n_big=30):
    """no bound; one bound; hiding; hiding with a bound; five polynomials across three bounds (bounds 10, 20, 33)"""
    f = lambda n, s: util.rand_fr(cname, n, seed + s, mont=True)                 # noqa: E731
    return [([(f(n_big, 1), None)], None),
            ([(f(18, 2), 20)], None),
            ([(f(n_big, 3), None)], [f(4, 4)]),
            ([(f(n_big, 5), None), (f(18, 6), 20)], [f(4, 7), f(3, 8)]),
            ([(f(n_big, 9), None), (f(9, 10), 10), (f(18, 11), 20), (f(21, 12), 20), (f(34, 13), 33)],
             [f(4, 14), None, f(2, 15), f(4, 16), f(3, 17)])]


def sonic_check_case(eng, keys, seed=40):
    """check is true on honest proofs of every polynomial set, and false with one thing tampered"""
    from poly_commit_b200 import kzg10, sonic_pc
    cname, cid, vk = keys.cname, keys.id, keys.vk
    point = util.rand_fr(cname, 1, seed, mont=True)[0]
    for i, (polys, rands) in enumerate(poly_sets(cname, seed)):
        comms, vals, proof, chals = keys.prove(polys, rands, point, seed + 20 + i)
        assert (proof[2] is None) == (rands is None)
        assert sonic_pc.check(eng, cid, vk, comms, point, vals, proof, chals), (cname, i)
    two = util.fr_const(cname, 2).reshape(1, 4)
    bad = vals.copy()
    bad[2] = eng.fr_mul(cid, vals[2].reshape(1, 4), two)[0]
    assert not sonic_pc.check(eng, cid, vk, comms, point, bad, proof, chals)                               # a value
    w_bad = (kzg10.neg_point(cid, proof[0]), proof[1], proof[2])
    assert not sonic_pc.check(eng, cid, vk, comms, point, vals, w_bad, chals)                              # w
    rv_bad = (proof[0], proof[1], eng.fr_mul(cid, proof[2].reshape(1, 4), two)[0])
    assert not sonic_pc.check(eng, cid, vk, comms, point, vals, rv_bad, chals)                             # random_v
    c_bad = list(comms)
    c_bad[3] = (comms[2][0], comms[3][1])
    assert not sonic_pc.check(eng, cid, vk, c_bad, point, vals, proof, chals)                              # a commitment
    c_bad = list(comms)
    c_bad[2] = (comms[2][0], 33)
    assert not sonic_pc.check(eng, cid, vk, c_bad, point, vals, proof, chals)                              # wrong bound label
    c_bad[2] = (comms[2][0], 21)
    with pytest.raises(sonic_pc.UnsupportedDegreeBound):
        sonic_pc.check(eng, cid, vk, c_bad, point, vals, proof, chals)                                     # no shift power


def sonic_batch_case(eng, keys, seed=60, n_big=30):
    """batch_open / batch_check over three points: true, and false with one evaluation perturbed"""
    from poly_commit_b200 import sonic_pc
    cname, cid = keys.cname, keys.id
    polys_l, rands_l = poly_sets(cname, seed, n_big)[4]
    polys = dict(zip("abcde", polys_l))
    rands = dict(zip("abcde", rands_l))
    x, y, z = util.rand_fr(cname, 3, seed, mont=True)
    query_set = [("a", ("x", x)), ("b", ("x", x)), ("c", ("y", y)), ("e", ("y", y)), ("d", ("z", z)), ("a", ("z", z))]
    chals = list(util.rand_fr(cname, 6, seed + 1, mont=True))
    proofs = sonic_pc.batch_open(keys.ck, polys, query_set, chals, rands)
    comms = dict(zip("abcde", [(c, b) for c, (_, b) in zip(sonic_pc.commit(keys.ck, polys_l, rands_l), polys_l)]))
    pts = dict(x=x, y=y, z=z)
    evaluations = {(lb, pl): keys.value(polys[lb][0], pts[pl]) for lb, (pl, _) in query_set}
    rnd = np.stack([util.fr_const(cname, 1)] + list(util.rand_fr(cname, 2, seed + 2, mont=True)))
    assert sonic_pc.batch_check(eng, cid, keys.vk, comms, query_set, evaluations, proofs, chals, rnd)
    evaluations[("e", "y")] = evaluations[("c", "y")]
    assert not sonic_pc.batch_check(eng, cid, keys.vk, comms, query_set, evaluations, proofs, chals, rnd)


def python_verifier_case(eng, keys, seed=80):
    """at degree <= 16: sonic_pc's G1 arguments and boolean equal a Python restatement of accumulate_elems / check_elems over
    pyref points and tests/pairing_ref, on an honest and a tampered proof"""
    from poly_commit_b200 import sonic_pc
    cname, cid, vk = keys.cname, keys.id, keys.vk
    C, E, r = pyref.Curve(cname), ref(cname), pyref.Curve(cname).r
    f = lambda n, s: util.rand_fr(cname, n, seed + s, mont=True)                 # noqa: E731
    polys = [(f(12, 1), None), (f(5, 2), 6), (f(9, 3), 10), (f(4, 4), 6)]
    rands = [f(2, 5), f(3, 6), None, f(1, 7)]
    point = f(1, 8)[0]
    comms, vals, proof, chals = keys.prove(polys, rands, point, seed + 9)
    neg_h = dict(vk.degree_bounds_and_neg_powers_of_h)
    for tamper in (False, True):
        if tamper:
            vals = vals.copy()
            vals[1] = vals[0]
        acc = sonic_pc.new_accumulator()
        sonic_pc.accumulate_elems(eng, cid, acc, comms, point, vals, proof, chals, util.fr_const(cname, 1))
        g1, idx = sonic_pc.equation(eng, cid, vk, acc)
        got = [C.points_from_limbs(xy.reshape(1, -1), np.array([inf], dtype=np.uint8))[0] for xy, inf in g1]
        # the restatement
        ch = [fr_int(cname, c) for c in chals]
        vs = [fr_int(cname, v) for v in vals]
        z, rv = fr_int(cname, point), fr_int(cname, proof[2])
        w = C.points_from_limbs(proof[0].reshape(1, -1))[0]
        groups = {}
        for (c, b), c_i in zip(comms, ch):
            P = C.mul(c_i, C.points_from_limbs(c[0].reshape(1, -1))[0])
            groups[b] = C.add(groups.get(b), P) if b in groups else P
        V = sum(c_i * v for c_i, v in zip(ch, vs)) % r
        g, gamma_g = C.points_from_limbs(vk.g.reshape(1, -1))[0], C.points_from_limbs(vk.gamma_g.reshape(1, -1))[0]
        adj = C.add(C.add(C.mul(V, g), C.mul((r - z) % r, w)), C.mul(rv, gamma_g))
        order = sorted(groups, key=lambda b: -1 if b is None else b)
        exp = [groups[b] for b in order] + [C.neg(adj), C.neg(w)]
        assert got == exp, (cname, tamper)
        Qs = [vk.h if b is None else neg_h[b] for b in order] + [vk.h, vk.beta_h]
        assert idx == [0 if b is None else vk.get_shift_power(b) for b in order] + [0, 1]
        want = E.multi_pairing(exp, Qs) == E.ONE
        assert want == (not tamper)
        assert sonic_pc.check(eng, cid, vk, comms, point, vals, proof, chals) == want


def wire_case(eng, keys, compressed):
    """the Sonic verifier key round-trips, and its bytes equal an encoding assembled from pyref's G1 and G2 serializers"""
    from poly_commit_b200 import wire
    cname, cid, vk = keys.cname, keys.id, keys.vk
    C, G2 = pyref.Curve(cname), pyref.G2(cname)
    for bounds in (vk.degree_bounds_and_neg_powers_of_h, None):
        data = wire.sonic_verifier_key_serialize(eng, cid, vk.g, vk.gamma_g, vk.h, vk.beta_h, bounds, vk.supported_degree,
                                                 vk.max_degree, compressed)
        exp = pyref.g1_serialize(C, C.points_from_limbs(np.stack([vk.g, vk.gamma_g])), compressed)
        exp += G2.serialize(vk.h, compressed) + G2.serialize(vk.beta_h, compressed)
        if bounds is None:
            exp += b"\x00"
        else:
            exp += b"\x01" + struct.pack("<Q", len(bounds))
            for b, P in bounds:
                exp += struct.pack("<Q", b) + G2.serialize(P, compressed)
        exp += struct.pack("<QQ", vk.supported_degree, vk.max_degree)
        assert bytes(data) == exp, (cname, compressed, bounds is None)
        d = wire.sonic_verifier_key_deserialize(eng, cid, data, compressed)
        assert (d["g"][0] == vk.g).all() and (d["gamma_g"][0] == vk.gamma_g).all() and not d["g"][1]
        assert d["h"] == vk.h and d["beta_h"] == vk.beta_h and d["degree_bounds_and_neg_powers_of_h"] == bounds
        assert (d["supported_degree"], d["max_degree"], d["consumed"]) == (vk.supported_degree, vk.max_degree, len(data))
    with pytest.raises(ValueError):
        wire.sonic_verifier_key_deserialize(eng, cid, data[:-1], compressed)
    bad = bytearray(data)
    bad[2 * eng.g1_wire_size(cid, compressed) + 2 * G2.size(compressed)] = 2
    with pytest.raises(ValueError):
        wire.sonic_verifier_key_deserialize(eng, cid, bytes(bad), compressed)                # option tag
    inverted = wire.sonic_verifier_key_serialize(eng, cid, vk.g, vk.gamma_g, vk.h, vk.beta_h, None, vk.max_degree + 1,
                                                 vk.max_degree, compressed)
    with pytest.raises(ValueError):
        wire.sonic_verifier_key_deserialize(eng, cid, inverted, compressed)                  # supported_degree > max_degree
    assert wire.sonic_verifier_key_deserialize(eng, cid, inverted, compressed, validate=False)["supported_degree"] == vk.max_degree + 1


def trim_case(eng, pc, keys):
    """trim's key layout and its errors"""
    from poly_commit_b200 import sonic_pc
    ck, vk = keys.ck, keys.vk
    assert ck.enforced_degree_bounds == [10, 20, 33] and ck.max_degree == vk.max_degree == 40 and vk.supported_degree == 36
    assert ck.supported_degree() == 36 and len(ck.shifted_powers_of_g) == 34 and len(ck.powers_of_gamma_g) == 5
    assert {b: len(p) for b, p in ck.shifted_powers_of_gamma_g.items()} == {10: 5, 20: 5, 33: 5}
    assert [b for b, _ in vk.degree_bounds_and_neg_powers_of_h] == [10, 20, 33] and len(vk.prepared) == 5
    assert vk.get_shift_power(20) == 3 and vk.get_shift_power(21) is None
    from poly_commit_b200 import wire
    C = pyref.Curve(keys.cname)
    pts = keys.powers
    pp = wire.universal_params_deserialize(eng, C.id, wire.universal_params_serialize(
        eng, C.id, pts, np.array([0, 1], dtype=np.uint64), pts[:2], keys.h, keys.beta_h, {}))
    with pytest.raises(sonic_pc.TrimmingDegreeTooLarge):
        sonic_pc.trim(eng, C.id, pp, 41, 0)
    with pytest.raises(sonic_pc.UnsupportedDegreeBound):
        sonic_pc.trim(eng, C.id, pp, 30, 0, [31])
    ck2, vk2 = sonic_pc.trim(eng, C.id, pp, 30, 0, [])
    assert ck2.enforced_degree_bounds is None and vk2.degree_bounds_and_neg_powers_of_h is None and len(vk2.prepared) == 2


# ---- host emulation --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cname", PAIRING)
def test_emul_prepared_pairing(emul, pc, cname):
    prepared_case(emul, cname)
    prepared_errors_case(emul, pc, cname)


def test_emul_prepared_honest_bn254(emul, pc):
    honest_bn254_case(emul, pc)


@pytest.fixture(scope="module", params=PAIRING)
def emul_keys(request, emul, pc):
    return SonicKeys(emul, pc, request.param, 40, 36, 3, [20, 33, 10, 20], seed=7)


def test_emul_sonic_check(emul, emul_keys):
    sonic_check_case(emul, emul_keys)


def test_emul_sonic_batch_check(emul, emul_keys):
    sonic_batch_case(emul, emul_keys)


def test_emul_sonic_trim(emul, pc, emul_keys):
    trim_case(emul, pc, emul_keys)


@pytest.mark.parametrize("cname", PAIRING)
def test_emul_sonic_vs_python_verifier(emul, pc, cname):
    python_verifier_case(emul, SonicKeys(emul, pc, cname, 16, 16, 2, [6, 10], seed=9))


@pytest.mark.parametrize("compressed", [True, False])
def test_emul_sonic_verifier_key_wire(emul, emul_keys, compressed):
    wire_case(emul, emul_keys, compressed)


def test_sonic_committer_key_positional_form(emul, pc):
    """CommitterKey(eng, curve, powers, shifted, bounds) commits as trim's key does"""
    from poly_commit_b200 import sonic_pc
    keys = SonicKeys(emul, pc, "bn254", 40, 36, 1, [20, 33], seed=11)
    pp = keys.powers
    ck = sonic_pc.CommitterKey(emul, keys.id, pp[:37], pp[40 - 33:], [33, 20])
    polys = [(util.rand_fr("bn254", 30, 90, mont=True), None), (util.rand_fr("bn254", 18, 91, mont=True), 20)]
    for a, b in zip(sonic_pc.commit(ck, polys), sonic_pc.commit(keys.ck, polys)):
        assert (a[0] == b[0]).all() and a[1] == b[1]


# ---- device ----------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cname", PAIRING)
def test_gpu_prepared_pairing(gpu_engine, pc, cname):
    prepared_case(gpu_engine, cname)
    prepared_errors_case(gpu_engine, pc, cname)
    if cname == "bn254":
        honest_bn254_case(gpu_engine, pc)


@pytest.mark.gpu
@pytest.mark.parametrize("cname", PAIRING)
def test_gpu_sonic_small(gpu_engine, pc, cname):
    keys = SonicKeys(gpu_engine, pc, cname, 40, 36, 3, [20, 33, 10], seed=7)
    sonic_check_case(gpu_engine, keys)
    sonic_batch_case(gpu_engine, keys)
    wire_case(gpu_engine, keys, True)
    python_verifier_case(gpu_engine, SonicKeys(gpu_engine, pc, cname, 16, 16, 2, [6, 10], seed=9))


@pytest.mark.gpu
@pytest.mark.parametrize("cname,lg", [("bls12_381", 20), ("bn254", 16)])
def test_gpu_sonic_at_size(gpu_engine, pc, cname, lg):
    """hiding and a degree bound at full size, through check and batch_check"""
    from poly_commit_b200 import sonic_pc
    n = 1 << lg
    bound = n - 100
    keys = SonicKeys(gpu_engine, pc, cname, n, n, 3, [bound, n // 2], seed=21)
    polys = [(util.rand_fr_fast(cname, n, 22), None), (util.rand_fr_fast(cname, bound + 1, 23), bound),
             (util.rand_fr_fast(cname, n // 2, 24), n // 2)]
    rands = [util.rand_fr(cname, 4, 25, mont=True), util.rand_fr(cname, 3, 26, mont=True), None]
    point = util.rand_fr(cname, 1, 27, mont=True)[0]
    comms, vals, proof, chals = keys.prove(polys, rands, point, 28)
    assert sonic_pc.check(gpu_engine, keys.id, keys.vk, comms, point, vals, proof, chals)
    bad = vals.copy()
    bad[1] = vals[2]
    assert not sonic_pc.check(gpu_engine, keys.id, keys.vk, comms, point, bad, proof, chals)
    polys_d = dict(zip("abc", polys))
    rands_d = dict(zip("abc", rands))
    x, y = util.rand_fr(cname, 2, 29, mont=True)
    query_set = [("a", ("x", x)), ("b", ("x", x)), ("c", ("y", y)), ("b", ("y", y))]
    ch = list(util.rand_fr(cname, 4, 30, mont=True))
    proofs = sonic_pc.batch_open(keys.ck, polys_d, query_set, ch, rands_d)
    comms_d = dict(zip("abc", comms))
    pts = dict(x=x, y=y)
    evaluations = {(lb, pl): keys.value(polys_d[lb][0], pts[pl]) for lb, (pl, _) in query_set}
    rnd = np.stack([util.fr_const(cname, 1), util.rand_fr(cname, 1, 31, mont=True)[0]])
    assert sonic_pc.batch_check(gpu_engine, keys.id, keys.vk, comms_d, query_set, evaluations, proofs, ch, rnd)
    evaluations[("b", "y")] = evaluations[("c", "y")]
    assert not sonic_pc.batch_check(gpu_engine, keys.id, keys.vk, comms_d, query_set, evaluations, proofs, ch, rnd)


@pytest.mark.gpu
@pytest.mark.parametrize("cname", PAIRING)
def test_gpu_prepared_volume(gpu_engine, pc, cname):
    """4096 Sonic-shaped equations (k = 4) against [h, s1 h, s2 h, s3 h] in one call: e(a P, h) e(b P, s1 h) e(c P, s2 h)
    e(d P, s3 h) = 1 with a = -(b s1 + c s2 + d s3), except every 7th, perturbed; GT values equal multi_pairing's; the
    DEVICE_PTRS path equals the host path"""
    eng, C = gpu_engine, pyref.Curve(cname)
    r, count = C.r, 4096
    s = util.rand_fr_ints(cname, 3, 41)
    H, _ = gc.to_limbs(cname, [gc.generator(cname)])
    q = eng.g2_fixed_base_mul(gc.group(pc, cname), H[0], fr_canon(cname, [1] + s))
    prep = eng.g2_prepare(C.id, q)
    b, c, d = (util.rand_fr_ints(cname, count, 42 + j) for j in range(3))
    bad = [i % 7 == 3 for i in range(count)]
    a = [(-(b[i] * s[0] + c[i] * s[1] + d[i] * s[2]) + (1 if bad[i] else 0)) % r for i in range(count)]
    scal = [v for i in range(count) for v in (a[i], b[i], c[i], d[i])]
    g1 = eng.fixed_base_mul(C.id, orc.g1_generator(C.id), fr_canon(cname, scal))
    idx = np.tile(np.arange(4, dtype=np.uint32), count)
    gt, one = eng.multi_pairing_prepared(C.id, g1, prep, idx, 4)
    assert [bool(o) for o in one] == [not x for x in bad]
    plain, plain_one = eng.multi_pairing(C.id, g1[:4 * 64], np.tile(q, (64, 1)), 4)
    assert (gt[:64] == plain).all() and (one[:64] == plain_one).all()
    d1, keep = util.dev_ptr(eng, g1)
    gtd, oned = eng.multi_pairing_prepared(C.id, d1, prep, idx, 4, flags=pc.DEVICE_PTRS, count=count)
    assert (gtd == gt).all() and (oned == one).all()
    dq, keepq = util.dev_ptr(eng, q)
    prep_d = eng.g2_prepare(C.id, dq, n=4, flags=pc.DEVICE_PTRS)
    gt2, _ = eng.multi_pairing_prepared(C.id, g1[:4 * 64], prep_d, idx[:4 * 64], 4)
    assert (gt2 == gt[:64]).all()
    prep.release()
    prep_d.release()
