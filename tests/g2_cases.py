"""G2 case bodies shared by the host-emulation tests and the device tests (test_g2_msm.py, test_multilinear_pc.py).

References, all independent of the library: oracle/pyref.py's G2 (affine group law in Python integers) for small sizes, and the
trapdoor identity for large ones -- bases B_i = k_i H with known k_i, so sum_i s_i B_i = (sum_i s_i k_i mod r) H, one Python
scalar multiplication.  The bases themselves come from pcgpu_g2_fixed_base_mul and are checked against pyref on a sample.
"""
import json
import os

import numpy as np

from oracle import pyref
from tests import msm_cases, util

PAIRING = ["bls12_381", "bn254"]
SMALL_MAX_N = msm_cases.SMALL_MAX_N
_KATS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "external_kats.json")


def group(pc, cname):
    return pc.binding.G2_OF[pyref.Curve(cname).id]


def generator(cname):
    """the published G2 generator of the curve (external_kats.json), affine ((x0, x1), (y0, y1))"""
    g = json.load(open(_KATS))[cname]["g2_generator"]
    v = {k: int(g[k], 0) for k in ("x_c0", "x_c1", "y_c0", "y_c1")}
    return ((v["x_c0"], v["x_c1"]), (v["y_c0"], v["y_c1"]))


def to_limbs(cname, pts):
    """affine points (None = identity) -> ((n, 4 nq) uint64 Montgomery x.c0 x.c1 y.c0 y.c1, (n,) uint8 identity flags)"""
    C = pyref.Curve(cname)
    out = np.zeros((len(pts), 4 * C.nq), dtype=np.uint64)
    inf = np.zeros(len(pts), dtype=np.uint8)
    for i, P in enumerate(pts):
        if P is None:
            inf[i] = 1
            continue
        for k, c in enumerate((P[0][0], P[0][1], P[1][0], P[1][1])):
            v = c * C.Rq % C.p
            for j in range(C.nq):
                out[i, k * C.nq + j] = (v >> (64 * j)) & 0xFFFFFFFFFFFFFFFF
    return out, inf


def from_limbs(cname, row, is_inf=False):
    C = pyref.Curve(cname)
    row = np.asarray(row, dtype=np.uint64).reshape(-1)
    if is_inf:
        assert not row.any(), "identity written with non-zero coordinates"
        return None
    c = [sum(int(row[k * C.nq + j]) << (64 * j) for j in range(C.nq)) * C.Rq_inv % C.p for k in range(4)]
    if not any(c):
        return None
    return ((c[0], c[1]), (c[2], c[3]))


def neg(cname, P):
    p = pyref.Curve(cname).p
    return None if P is None else (P[0], ((-P[1][0]) % p, (-P[1][1]) % p))


def trapdoor_bases(eng, pc, cname, ks, sample=16, seed=0):
    """B_i = k_i H through pcgpu_g2_fixed_base_mul, `sample` of them (first, last, random) checked against pyref"""
    G = pyref.G2(cname)
    H = generator(cname)
    h_xy, _ = to_limbs(cname, [H])
    ks = [k % G.r for k in ks]
    out = eng.g2_fixed_base_mul(group(pc, cname), h_xy[0], fr_limbs(ks))
    n = len(ks)
    idx = sorted({0, n - 1} | set(util.rng(seed).integers(0, n, size=max(0, sample - 2)).tolist())) if n else []
    for i in idx:
        assert from_limbs(cname, out[i]) == G.mul(ks[i], H), (cname, i)
    return out


def fr_limbs(vals, mont=False, cname=None):
    if mont:
        return pyref.Curve(cname).fr_to_limbs(vals, True)
    a = np.zeros((len(vals), 4), dtype=np.uint64)
    for i, v in enumerate(vals):
        for j in range(4):
            a[i, j] = (v >> (64 * j)) & 0xFFFFFFFFFFFFFFFF
    return a


def msm(eng, pc, cname, bases, scalars, inf=None, mont=False):
    """one G2 MSM through a registered key -> affine point or None"""
    srs = eng.srs_register(group(pc, cname), bases, inf=inf)
    try:
        xy, is_inf = eng.msm(srs, scalars, flags=pc.SCALARS_MONT if mont else 0)
    finally:
        srs.release()
    return from_limbs(cname, xy, is_inf)


def trapdoor_expect(cname, ks, ss):
    G = pyref.G2(cname)
    return G.mul(sum(k * s for k, s in zip(ks, ss)) % G.r, generator(cname))


# ---- cases ---------------------------------------------------------------------------------------------------------------
def fq2_ops_case(eng, cname, n=64, seed=0):
    """pcgpu_diag_field_op which = 2 against Python integers: products, squares, sums, differences, negations and inverses,
    with limb-edge operands and 0 / 1 / p - 1 components (inverse of 0 is 0)"""
    C = pyref.Curve(cname)
    G = pyref.G2(cname)
    p, nq = C.p, C.nq
    g = util.rng(seed)
    edge = [0, 1, p - 1, p - 2, (p - 1) // 2, (1 << 64) - 1, 1 << 64, (1 << (64 * (nq - 1))) - 1, p - (1 << 64)]
    vals = [(a, b) for a in edge for b in edge[:4]] + [(b, a) for a in edge for b in edge[:4]]
    while len(vals) < n:
        vals.append(tuple(int.from_bytes(g.bytes(8 * nq), "little") % p for _ in range(2)))
    vals = vals[:max(n, len(vals))]
    other = vals[1:] + vals[:1]

    def limbs(vs):
        a = np.zeros((len(vs), 2 * nq), dtype=np.uint64)
        for i, (c0, c1) in enumerate(vs):
            for k, c in enumerate((c0, c1)):
                m = c * C.Rq % p
                for j in range(nq):
                    a[i, k * nq + j] = (m >> (64 * j)) & 0xFFFFFFFFFFFFFFFF
        return a

    def back(a):
        return [tuple(sum(int(row[k * nq + j]) << (64 * j) for j in range(nq)) * C.Rq_inv % p for k in range(2)) for row in a]

    A, B = limbs(vals), limbs(other)
    ref = {
        0: [G.mul2(x, y) for x, y in zip(vals, other)],
        9: [G.mul2(x, x) for x in vals],
        2: [((x[0] + y[0]) % p, (x[1] + y[1]) % p) for x, y in zip(vals, other)],
        3: [((x[0] - y[0]) % p, (x[1] - y[1]) % p) for x, y in zip(vals, other)],
        4: [((-x[0]) % p, (-x[1]) % p) for x in vals],
        5: [(0, 0) if x == (0, 0) else G.inv2(x) for x in vals],
    }
    for op, exp in ref.items():
        assert back(eng.diag_field_op(C.id, 2, op, A, B)) == exp, (cname, op)


def generator_kat_case(eng, pc, cname, path):
    """the published generator through the device MSM: [r - 1, 1] . [H, H] = O and [2] . H = pyref's doubling"""
    G = pyref.G2(cname)
    H = generator(cname)
    assert G.on_curve(H)
    hx, _ = to_limbs(cname, [H, H])
    assert msm(eng, pc, cname, hx, fr_limbs([G.r - 1, 1])) is None
    msm_cases.check_geometry(eng, pc, cname, 2, g2=True, small=path == "small")
    assert msm(eng, pc, cname, hx[:1], fr_limbs([2])) == G.add(H, H)
    xy, is_inf = eng.msm_bases(group(pc, cname), hx, fr_limbs([3, 2]))     # unregistered bases
    assert from_limbs(cname, xy, is_inf) == G.mul(5, H)


def edge_case(eng, pc, cname, path, seed=1):
    """n = 0 and 1; edge scalars 0, 1, r - 1, (r +- 1) / 2 and all-(+-2^(c-1)) digits; duplicated, negated and identity bases;
    an exact zero sum; canonical and Montgomery scalars; PCGPU_E_RANGE followed by a correct MSM on the same context"""
    G = pyref.G2(cname)
    r = G.r
    c = msm_cases.msm_pick_c(1) if path == "small" else int(os.environ.get("PCGPU_MSM_C") or msm_cases.msm_pick_c(64))
    half = 1 << (c - 1)
    alt = sum(half << (c * w) for w in range(256 // c)) % r          # every window +2^(c-1) (a carry chain of -2^(c-1) digits)
    ks = [int(v) for v in util.rand_fr_ints(cname, 24, seed)]
    ks[3] = ks[2]                                                     # duplicated base
    ks[5] = (r - ks[4]) % r                                           # negated base
    ks[7] = 0                                                         # identity base (flag)
    bases = trapdoor_bases(eng, pc, cname, ks, sample=4, seed=seed)
    inf = np.zeros(len(ks), dtype=np.uint8)
    inf[7] = 1
    bases[7] = 0
    ss = [0, 1, r - 1, (r - 1) // 2, (r + 1) // 2, alt, r - alt, 2, half, r - half] + \
        [int(v) for v in util.rand_fr_ints(cname, 14, seed + 1)]
    for mont in (False, True):
        for n in (0, 1, 2, 5, len(ks)):
            sc = fr_limbs(ss[:n], mont, cname)
            got = msm(eng, pc, cname, bases[:n], sc, inf=inf[:n], mont=mont)
            assert got == trapdoor_expect(cname, ks[:n], ss[:n]), (cname, path, mont, n)
            msm_cases.check_geometry(eng, pc, cname, n, g2=True, small=path == "small")
    # an exact zero sum: every term cancels against a negated copy
    kz = ks[:8] + [(r - k) % r for k in ks[:8]]
    bz = trapdoor_bases(eng, pc, cname, kz, sample=2, seed=seed)
    sz = ss[:8] * 2
    assert msm(eng, pc, cname, bz, fr_limbs(sz)) is None
    msm_cases.check_geometry(eng, pc, cname, 16, g2=True, small=path == "small")
    # out-of-range scalars, then a good MSM on the same context
    srs = eng.srs_register(group(pc, cname), bases)
    for bad in (r, (1 << 256) - 1):
        sc = fr_limbs([1, bad, 2])
        try:
            eng.msm(srs, sc)
            raise AssertionError("scalar >= r accepted")
        except pc.PcgpuError as e:
            assert e.code == -5, e
    xy, is_inf = eng.msm(srs, fr_limbs(ss[:3]))
    assert from_limbs(cname, xy, is_inf) == trapdoor_expect(cname, ks[:3], ss[:3])
    srs.release()


def random_vs_pyref_case(eng, pc, cname, n, path, seed=2):
    """random bases (k_i H, the k_i forgotten) against pyref's naive MSM"""
    G = pyref.G2(cname)
    ks = util.rand_fr_ints(cname, n, seed)
    bases = trapdoor_bases(eng, pc, cname, ks, sample=4, seed=seed)
    pts = [from_limbs(cname, b) for b in bases]
    ss = util.rand_fr_ints(cname, n, seed + 1)
    exp = None
    for P, s in zip(pts, ss):
        exp = G.add(exp, G.mul(s, P))
    assert msm(eng, pc, cname, bases, fr_limbs(ss)) == exp, (cname, n)
    msm_cases.check_geometry(eng, pc, cname, n, g2=True, small=path == "small")


def fr_ints(arr):
    """(n, 4) uint64 -> Python ints"""
    a = np.asarray(arr, dtype=np.uint64).reshape(-1, 4)
    cols = [[int(v) for v in a[:, j]] for j in range(4)]
    return [c0 | (c1 << 64) | (c2 << 128) | (c3 << 192) for c0, c1, c2, c3 in zip(*cols)]


def trapdoor_case(eng, pc, cname, n, path, skewed=False, seed=3, sample=16, keyed=None):
    """sum s_i (k_i H) = (sum s_i k_i) H at size; skewed: a few distinct scalar values repeated (heavy buckets).
    keyed: (ks, bases) of at least n trapdoor bases to reuse across sizes"""
    r = pyref.Curve(cname).r
    if keyed is None:
        ks = util.rand_fr_ints(cname, n, seed)
        bases = trapdoor_bases(eng, pc, cname, ks, sample=sample, seed=seed)
    else:
        ks, bases = keyed[0][:n], keyed[1][:n]
    if skewed:
        pool = util.rand_fr_ints(cname, 5, seed + 7) + [1, r - 1]
        pick = util.rng(seed + 8).integers(0, len(pool), size=n)
        ss = [pool[int(i)] for i in pick]
    else:
        ss = fr_ints(util.rand_fr(cname, n, seed + 1, mont=False))
    mont = bool(seed & 1)
    assert msm(eng, pc, cname, bases, fr_limbs(ss, mont, cname), mont=mont) == trapdoor_expect(cname, ks, ss), (cname, n, skewed)
    msm_cases.check_geometry(eng, pc, cname, n, g2=True, small=path == "small")


def g2_id_rejected_case(eng, pc, cname):
    """G2 ids are groups, not curves: Fr / G1 entry points reject them; SRS_PRECOMPUTE / SRS_COMB G2 keys are refused"""
    gid = group(pc, cname)
    a = fr_limbs([1, 2])
    for call in (lambda: eng.fr_mul(gid, a, a), lambda: eng.fr_from_mont(gid, a), lambda: eng.ntt(gid, a, 1),
                 lambda: eng.fixed_base_mul(gid, np.zeros(16, dtype=np.uint64), a),
                 lambda: eng.diag_field_op(gid, 0, 0, a, a)):
        try:
            call()
            raise AssertionError("G2 id accepted by a scalar-field / G1 entry point")
        except pc.PcgpuError as e:
            assert e.code == -3, e
    H, _ = to_limbs(cname, [generator(cname)] * 4)
    for fl in (pc.SRS_PRECOMPUTE, pc.SRS_COMB):
        try:
            eng.srs_register(gid, H, flags=fl)
            raise AssertionError("G2 key with tables accepted")
        except pc.PcgpuError as e:
            assert e.code == -3, e
    srs = eng.srs_register(gid, H)
    assert eng.lib.pcgpu_srs_curve(srs.handle) == gid
    try:
        eng.msm_batch(srs, fr_limbs([1] * 4), 4, 1)
        raise AssertionError("G2 key accepted by pcgpu_msm_batch")
    except pc.PcgpuError as e:
        assert e.code == -3, e
    srs.release()
