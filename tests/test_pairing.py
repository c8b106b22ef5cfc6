"""The optimal-ate pairing (pcgpu_multi_pairing, pcgpu_diag_field_op which = 3) and the verifiers built on it (kzg10.check /
batch_check, marlin_pc.check / batch_check, multilinear_pc.check) on BLS12-381 and BN254: one set of case bodies, run on the
host-emulated kernels and, under -m gpu, on the device.

Reference: tests/pairing_ref.py, a definition-level pairing over a flat Fq12 (not the device's tower), itself pinned by the
pairing's defining properties below.  No published GT value exists for these curves in the reference's tests, so the oracle is
pinned by non-degeneracy, order r, bilinearity in both arguments and linearity in G2.
"""
import ctypes

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


# ---- case bodies ---------------------------------------------------------------------------------------------------------
def fq12_ops_case(eng, cname, n=3, seed=0):
    """which = 3 against the flat oracle: products, sums, differences, negations, squares, inverses (0 -> 0), Frobenius and the
    final exponentiation of random elements"""
    E, cid = ref(cname), pyref.Curve(cname).id
    g = util.rng(seed)
    xs = [E.random(g) for _ in range(n)]
    ys = [E.random(g) for _ in range(n)]
    xs[0] = (0,) * 12
    A, B = E.to_limbs(xs), E.to_limbs(ys)
    assert E.from_limbs(A) == xs
    neg = [E.sub((0,) * 12, x) for x in xs]
    for op, exp in ((0, [E.mul(x, y) for x, y in zip(xs, ys)]), (2, [E.add(x, y) for x, y in zip(xs, ys)]),
                    (3, [E.sub(x, y) for x, y in zip(xs, ys)]), (4, neg), (5, [E.inv(x) for x in xs]),
                    (9, [E.mul(x, x) for x in xs]), (10, [E.frob(x) for x in xs])):
        assert E.from_limbs(eng.diag_field_op(cid, 3, op, A, B)) == exp, (cname, op)
    got = E.from_limbs(eng.diag_field_op(cid, 3, 11, A[1:3], B[1:3]))
    assert got == [E.final_exp(x) for x in xs[1:3]], cname


def multi_pairing_case(eng, cname, seed=3):
    """k = 0, 1, 2, 3 against the oracle, with identities in either slot; is_one agrees with the GT value"""
    E, C = ref(cname), pyref.Curve(cname)
    H = gc.generator(cname)
    g = util.rng(seed)
    ks = [int(v) for v in g.integers(2, 1 << 30, size=6)]
    Ps = [C.mul(k, C.g) for k in ks[:3]]
    Qs = [E.G2.mul(k, H) for k in ks[3:]]
    cases = [([], []), ([Ps[0]], [Qs[0]]), ([Ps[0], None], [Qs[0], Qs[1]]), ([Ps[0], Ps[1], Ps[2]], [Qs[0], None, Qs[2]]),
             ([C.neg(Ps[0]), Ps[0]], [Qs[1], Qs[1]])]
    for Ps_, Qs_ in cases:
        k = len(Ps_)
        if k:
            g1, g1i = g1_limbs(cname, Ps_)
            g2, g2i = gc.to_limbs(cname, Qs_)
            gt, one = eng.multi_pairing(C.id, g1, g2, k, g1_inf=g1i, g2_inf=g2i)
        else:
            gt, one = eng.multi_pairing(C.id, None, None, 0, count=2)
        exp = E.multi_pairing(Ps_, Qs_)
        got = E.from_limbs(gt)
        assert all(v == exp for v in got), (cname, k)
        assert list(one) == [int(exp == E.ONE)] * len(got), (cname, k)
    # two equations in one call, outputs one at a time
    g1, _ = g1_limbs(cname, [Ps[0], Ps[1]])
    g2, _ = gc.to_limbs(cname, [Qs[0], Qs[1]])
    gt, _ = eng.multi_pairing(C.id, g1, g2, 1)
    assert E.from_limbs(gt) == [E.pairing(Ps[0], Qs[0]), E.pairing(Ps[1], Qs[1])]
    _, one = eng.multi_pairing(C.id, g1, g2, 2)
    assert list(one) == [0]


def errors_case(eng, pc, cname):
    """Pallas and G2 ids are refused, k > 64 is refused, both outputs NULL is refused, count = 0 is a no-op"""
    C = pyref.Curve(cname)
    g1, _ = g1_limbs(cname, [C.g])
    g2, _ = gc.to_limbs(cname, [gc.generator(cname)])
    for curve, k in ((2, 1), (gc.group(pc, cname), 1), (C.id, 65)):
        with pytest.raises(pc.PcgpuError) as e:
            eng.multi_pairing(curve, np.tile(g1, (k, 1)), np.tile(g2, (k, 1)), k)
        assert e.value.code == -3
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    rc = eng.lib.pcgpu_multi_pairing(eng.ctx, C.id, p(g1), None, p(g2), None, 1, 1, 0, None, None)
    assert rc == -3
    out = np.zeros(1, dtype=np.uint8)
    assert eng.lib.pcgpu_multi_pairing(eng.ctx, C.id, None, None, None, None, 1, 0, 0, None, p(out)) == 0
    with pytest.raises(pc.PcgpuError) as e:
        eng.diag_field_op(2, 3, 0, np.zeros((1, 48), dtype=np.uint64), np.zeros((1, 48), dtype=np.uint64))
    assert e.value.code == -3


class Kzg:
    """KZG10 keys from a known beta: powers_of_g, powers_of_gamma_g, and the verifier key (g, gamma_g, h, beta_h)"""

    def __init__(self, eng, pc, cname, n, seed=1, n_gamma=8):
        C = pyref.Curve(cname)
        self.eng, self.cname, self.id = eng, cname, C.id
        beta = util.rand_fr(cname, 1, 1000 + seed, mont=True)[0]
        pows = orc.fr_powers_canonical(C.id, beta, max(n, n_gamma, 2))
        G = orc.g1_generator(C.id)
        gamma = util.rand_fr(cname, 1, 1500 + seed, mont=False)
        gG = eng.fixed_base_mul(C.id, G, gamma)[0]
        self.powers = eng.fixed_base_mul(C.id, G, pows[:n])
        self.gamma_powers = eng.fixed_base_mul(C.id, gG, pows[:n_gamma])
        H, _ = gc.to_limbs(cname, [gc.generator(cname)])
        beta_h = eng.g2_fixed_base_mul(gc.group(pc, cname), H[0], pows[1:2])[0]
        self.vk = dict(g=G, gamma_g=gG, h=H[0], beta_h=beta_h)
        self.srs = eng.srs_register(C.id, self.powers)
        self.gamma = eng.srs_register(C.id, self.gamma_powers)

    def value(self, coeffs, z):
        return self.eng.fr_div_linear(self.id, coeffs, z)[1]

    def release(self):
        self.srs.release()
        self.gamma.release()


def kzg_check_case(eng, pc, cname, n, seed=5, key=None, fused=False):
    """commit, open, check == true, non-hiding and hiding; false for a wrong value, a wrong point and a swapped proof"""
    from poly_commit_b200 import kzg10
    key = key or Kzg(eng, pc, cname, n, seed)
    cid, vk = key.id, key.vk
    coeffs = util.rand_fr_fast(cname, n, seed)
    other = util.rand_fr(cname, 8, seed + 1, mont=True)
    z, z2 = util.rand_fr(cname, 2, seed + 2, mont=True)
    if fused:
        comm, w = eng.kzg_commit_open(key.srs, coeffs, z)
    else:
        comm = eng.kzg_commit(key.srs, coeffs)
        w = eng.kzg_open(key.srs, coeffs, z)[:2]
    v = key.value(coeffs, z)
    assert kzg10.check(eng, cid, vk, comm, z, v, w)
    assert not kzg10.check(eng, cid, vk, comm, z, eng.fr_mul(cid, v.reshape(1, 4), util.fr_const(cname, 2).reshape(1, 4))[0], w)
    assert not kzg10.check(eng, cid, vk, comm, z2, v, w)
    w_other = eng.kzg_open(key.srs, other, z)[:2]
    assert not kzg10.check(eng, cid, vk, comm, z, v, w_other)
    # hiding
    blind = util.rand_fr(cname, 4, seed + 3, mont=True)
    hc = eng.kzg_commit(key.srs, other, powers_of_gamma_g=key.gamma, blind=blind)
    hw_xy, hw_inf, rv = eng.kzg_open(key.srs, other, z, powers_of_gamma_g=key.gamma, blind=blind)
    hv = key.value(other, z)
    assert kzg10.check(eng, cid, vk, hc, z, hv, (hw_xy, hw_inf), rv)
    assert not kzg10.check(eng, cid, vk, hc, z, hv, (hw_xy, hw_inf), None)


def kzg_batch_case(eng, pc, cname, n, m, seed=7, key=None, batch_open=False):
    """batch_check over m proofs is true, and false with one tampered proof"""
    from poly_commit_b200 import kzg10
    key = key or Kzg(eng, pc, cname, n, seed)
    cid = key.id
    polys = [util.rand_fr_fast(cname, n, seed + 10 + i) for i in range(m)]
    if batch_open:
        z = util.rand_fr(cname, 1, seed, mont=True)[0]
        comms, _, ws, _ = eng.kzg_commit_open_batch(key.srs, polys, z)
        points = np.tile(z, (m, 1))
    else:
        points = util.rand_fr(cname, m, seed, mont=True)
        comms = np.stack([eng.kzg_commit(key.srs, p)[0] for p in polys])
        ws = np.stack([eng.kzg_open(key.srs, p, z)[0] for p, z in zip(polys, points)])
    values = np.stack([key.value(p, z) for p, z in zip(polys, points)])
    rnd = util.rand_fr(cname, m, seed + 1, mont=True)
    rnd[0] = util.fr_const(cname, 1)
    assert kzg10.batch_check(eng, cid, key.vk, comms, points, values, ws, rnd)
    bad = ws.copy()
    bad[m // 2] = ws[(m // 2 + 1) % m] if m > 1 else kzg10.neg_point(cid, ws[0])
    assert not kzg10.batch_check(eng, cid, key.vk, comms, points, values, bad, rnd)


def marlin_case(eng, pc, cname, seed=9):
    """MarlinKZG10: check with a degree bound and hiding is true (and false for a wrong value); batch_check over two points"""
    from poly_commit_b200 import marlin_pc
    C = pyref.Curve(cname)
    max_degree, bounds = 40, [20, 33]
    key = Kzg(eng, pc, cname, max_degree + 1, seed)
    pp = key.powers
    ck = marlin_pc.CommitterKey(eng, C.id, pp, pp[max_degree - bounds[-1]:], bounds, powers_of_gamma_g_xy=key.gamma_powers)
    shift_powers = {b: pp[max_degree - b] for b in bounds}
    polys = [(util.rand_fr(cname, 30, seed=seed + 1, mont=True), None), (util.rand_fr(cname, 18, seed=seed + 2, mont=True), 20),
             (util.rand_fr(cname, 34, seed=seed + 3, mont=True), 33)]
    rands = [dict(rand=util.rand_fr(cname, 4, seed=seed + 4, mont=True)),
             dict(rand=util.rand_fr(cname, 5, seed=seed + 5, mont=True), shifted_rand=util.rand_fr(cname, 5, seed=seed + 6, mont=True)),
             None]
    coms = marlin_pc.commit(ck, polys, rands)
    triples = [(c[0], None if s is None else s[0], b) for (_, b), (c, s) in zip(polys, coms)]
    point, point2 = util.rand_fr(cname, 2, seed=seed + 7, mont=True)
    chals = list(util.rand_fr(cname, 5, seed=seed + 8, mont=True))
    w_xy, w_inf, rv = marlin_pc.open(ck, polys, point, chals, rands)
    vals = np.stack([key.value(c, point) for c, _ in polys])
    assert marlin_pc.check(eng, C.id, key.vk, triples, point, vals, ((w_xy, w_inf), rv), chals, shift_powers)
    bad = vals.copy()
    bad[1] = vals[0]
    assert not marlin_pc.check(eng, C.id, key.vk, triples, point, bad, ((w_xy, w_inf), rv), chals, shift_powers)
    # batch_check: labels a, b at point "x", label c at point "y"; challenges drawn group by group in point-label order
    commitments = dict(zip("abc", triples))
    query_set = [("a", ("x", point)), ("b", ("x", point)), ("c", ("y", point2))]
    ch_x, ch_y = chals[:3], list(util.rand_fr(cname, 2, seed=seed + 9, mont=True))
    proof_x = marlin_pc.open(ck, polys[:2], point, ch_x, rands[:2])
    proof_y = marlin_pc.open(ck, polys[2:], point2, ch_y, rands[2:])
    evaluations = {("a", "x"): vals[0], ("b", "x"): vals[1], ("c", "y"): key.value(polys[2][0], point2)}
    rnd = np.stack([util.fr_const(cname, 1), util.rand_fr(cname, 1, seed=seed + 10, mont=True)[0]])
    proofs = [((proof_x[0], proof_x[1]), proof_x[2]), ((proof_y[0], proof_y[1]), proof_y[2])]
    assert marlin_pc.batch_check(eng, C.id, key.vk, commitments, query_set, evaluations, proofs, ch_x + ch_y, rnd, shift_powers)
    evaluations[("c", "y")] = vals[0]
    assert not marlin_pc.batch_check(eng, C.id, key.vk, commitments, query_set, evaluations, proofs, ch_x + ch_y, rnd, shift_powers)
    key.release()


def mlpc_case(eng, pc, cname, nv, seed=11):
    """MultilinearPC: check is true for an honest proof and false for a wrong value"""
    from poly_commit_b200 import multilinear_pc as mpc
    C = pyref.Curve(cname)
    t = util.rand_fr_ints(cname, nv, seed)
    H, _ = gc.to_limbs(cname, [gc.generator(cname)])
    params = mpc.setup(eng, C.id, t, orc.g1_generator(C.id), H[0])
    ck, vk = mpc.trim(params, nv)
    com = mpc.Committer(eng, C.id, ck)
    evals = util.rand_fr_fast(cname, 1 << nv, seed + 1)
    point = util.rand_fr(cname, nv, seed + 2, mont=True)
    comm = com.commit(evals)
    proofs, pinf, value = com.open(evals, point)
    assert mpc.check(eng, C.id, vk, comm, point, value, (proofs, pinf))
    wrong = eng.fr_mul(C.id, value.reshape(1, 4), util.fr_const(cname, 3).reshape(1, 4))[0]
    assert not mpc.check(eng, C.id, vk, comm, point, wrong, (proofs, pinf))
    com.release()


# ---- oracle ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cname", PAIRING)
def test_oracle_properties(cname):
    E, C = ref(cname), pyref.Curve(cname)
    P, Q = C.g, gc.generator(cname)
    assert E.on_curve(E.untwist(Q)) and E.on_curve(E.untwist(E.G2.mul(12345, Q)))
    e = E.pairing(P, Q)
    assert e != E.ONE and E.pow(e, E.r) == E.ONE
    a, b = 0x1234567, 0x89abcd
    assert E.pairing(C.mul(a, P), E.G2.mul(b, Q)) == E.pow(e, a * b)
    Q1, Q2 = E.G2.mul(5, Q), E.G2.mul(11, Q)
    assert E.pairing(P, E.G2.add(Q1, Q2)) == E.mul(E.pairing(P, Q1), E.pairing(P, Q2))
    assert E.from_tower(E.to_tower(e)) == e


# ---- host emulation --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cname", PAIRING)
def test_emul_fq12_ops(emul, cname):
    fq12_ops_case(emul, cname)


@pytest.mark.parametrize("cname", PAIRING)
def test_emul_multi_pairing(emul, cname):
    multi_pairing_case(emul, cname)


@pytest.mark.parametrize("cname", PAIRING)
def test_emul_errors(emul, pc, cname):
    errors_case(emul, pc, cname)


@pytest.mark.parametrize("cname", PAIRING)
def test_emul_kzg10_check(emul, pc, cname):
    key = Kzg(emul, pc, cname, 64, seed=5)
    kzg_check_case(emul, pc, cname, 64, key=key)
    kzg_batch_case(emul, pc, cname, 64, 3, key=key)
    key.release()


def test_emul_marlin_check(emul, pc):
    marlin_case(emul, pc, "bn254")


def test_emul_multilinear_check(emul, pc):
    mlpc_case(emul, pc, "bn254", 3)


# ---- device ----------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cname", PAIRING)
def test_gpu_field_and_small(gpu_engine, pc, cname):
    fq12_ops_case(gpu_engine, cname, n=6)
    multi_pairing_case(gpu_engine, cname)
    errors_case(gpu_engine, pc, cname)


@pytest.mark.gpu
@pytest.mark.parametrize("cname,lg", [("bls12_381", 20), ("bn254", 16)])
def test_gpu_kzg10_check_at_size(gpu_engine, pc, cname, lg):
    key = Kzg(gpu_engine, pc, cname, 1 << lg, seed=21)
    kzg_check_case(gpu_engine, pc, cname, 1 << lg, seed=22, key=key, fused=True)
    kzg_batch_case(gpu_engine, pc, cname, 1 << 12, 64, seed=23, key=key, batch_open=True)
    key.release()


@pytest.mark.gpu
@pytest.mark.parametrize("cname", PAIRING)
def test_gpu_marlin_check(gpu_engine, pc, cname):
    marlin_case(gpu_engine, pc, cname)


@pytest.mark.gpu
@pytest.mark.parametrize("cname", PAIRING)
def test_gpu_multilinear_check_nv20(gpu_engine, pc, cname):
    mlpc_case(gpu_engine, pc, cname, 20)


@pytest.mark.gpu
@pytest.mark.parametrize("cname", PAIRING)
def test_gpu_volume(gpu_engine, pc, cname):
    """4096 equations e(aP, Q) e(-P, aQ): all one, except every 7th, perturbed; a sample of GT values against the oracle; the
    k = 21 shape; the DEVICE_PTRS path equals the host path"""
    eng, E, C = gpu_engine, ref(cname), pyref.Curve(cname)
    r, count = C.r, 4096
    G = orc.g1_generator(C.id)
    H, _ = gc.to_limbs(cname, [gc.generator(cname)])
    s = util.rand_fr_ints(cname, count, 31)
    t = util.rand_fr_ints(cname, count, 32)
    a = util.rand_fr_ints(cname, count, 33)
    bad = [i % 7 == 3 for i in range(count)]
    g1s = [a[i] * s[i] for i in range(count)] + [r - s[i] for i in range(count)]
    g2s = [t[i] for i in range(count)] + [a[i] * t[i] + (1 if bad[i] else 0) for i in range(count)]
    p1 = eng.fixed_base_mul(C.id, G, fr_canon(cname, g1s))
    q1 = eng.g2_fixed_base_mul(gc.group(pc, cname), H[0], fr_canon(cname, g2s))
    g1 = np.stack([p1[:count], p1[count:]], axis=1).reshape(2 * count, -1)
    g2 = np.stack([q1[:count], q1[count:]], axis=1).reshape(2 * count, -1)
    gt, one = eng.multi_pairing(C.id, g1, g2, 2)
    assert [bool(o) for o in one] == [not b for b in bad]
    for i in (0, 3, 10):
        P0, P1 = C.points_from_limbs(g1[2 * i:2 * i + 2])
        Q0, Q1 = gc.from_limbs(cname, g2[2 * i]), gc.from_limbs(cname, g2[2 * i + 1])
        assert E.from_limbs(gt[i])[0] == E.multi_pairing([P0, P1], [Q0, Q1]), (cname, i)
    # k = 21 (MultilinearPC at nv = 20): 64 equations, one against the oracle
    k, m = 21, 64
    g1k, g2k = g1[: k * m], g2[: k * m]
    gtk, _ = eng.multi_pairing(C.id, g1k, g2k, k)
    Ps = C.points_from_limbs(g1k[:k])
    Qs = [gc.from_limbs(cname, row) for row in g2k[:k]]
    assert E.from_limbs(gtk[0])[0] == E.multi_pairing(Ps, Qs)
    d1, keep1 = util.dev_ptr(eng, g1k)
    d2, keep2 = util.dev_ptr(eng, g2k)
    gtd, oned = eng.multi_pairing(C.id, d1, d2, k, flags=pc.DEVICE_PTRS, count=m)
    assert (gtd == gtk).all()
