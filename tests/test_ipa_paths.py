"""The InnerProductArgPC::open halving loop (pcgpu_ipa_*, csrc/ipa.cuh, ipa_*_impl in csrc/impl.cuh) and the inner product
under it (fr_inner_product, csrc/frops.cuh) against references that share nothing with the device: the C oracle's MSMs, folds
and field ops with challenges derived on the host through oracle/pyref.py serialization and hashlib (oracle_ipa_rounds), the
frozen-key identity of csrc/ipa.cuh evaluated on the host from the oracle's own challenges (weight_form_rounds, for 2^18),
Python-integer definitions and closed forms.  Bit-exact everywhere.  The same case bodies run on the host-emulated kernels (CPU,
n <= 2^14) and, with `-m gpu`, on the device at the sizes where the policy picks each path.

Which path a round takes is a pure function of (n, PCGPU_MSM_SMALL, PCGPU_IPA_FREEZE, PCGPU_IPA_GLV, curve); ipa_rounds()
restates it (csrc/impl.cuh ipa_maybe_freeze, ipa_round_lr_impl, ipa_round_fold_impl, msm_small_plan):
  * freeze: at begin and after every explicit fold the key is frozen at its current length n_t when 2 <= n_t <= 4096, unless
    PCGPU_MSM_SMALL=0 or PCGPU_IPA_FREEZE=0; a frozen key is never folded again (its fold multiplies weights);
  * FROZEN round: the one-launch small MSM over the frozen key, M = the frozen length;
  * SMALL round: m = n_t / 2 <= 8192 with the small MSM on: the one-launch kernel, M = m, split 1 below 512 terms, 3 up to
    4096, 6 above;
  * BUCKETS round: otherwise; the context's own MSM is the l commitment over the raw key, n = m;
  * explicit folds: the GLV ladder on the curves with cofactor one (Pallas, BN254) unless PCGPU_IPA_GLV=0, else 256 steps.
Every open case asserts each round's report (Engine.msm_last_geometry) against this, and the report of ipa_finish on a frozen
key; test_round_policy_coverage asserts that the device parameter lists reach every path, split, hand-over and fold.
"""
import ctypes
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from oracle import orc, pyref
from tests import msm_cases, util
from tests.test_hostcheck import oracle_ipa_rounds

SMALL_MAX_N = msm_cases.SMALL_MAX_N           # the largest key that is frozen
SMALL_ROUND_MAX_M = msm_cases.SMALL_WIDE_MAX_N  # the largest commitment of a SMALL round
GLV_CURVES = ("pallas", "bn254")              # cofactor one: the fold runs through the endomorphism
E_BADARG, E_LEN = -3, -4
EXPLICIT_MAX_LOG = 16                         # larger opens are checked through the weight form (explicit folds are slow)

# open rows: (curve, logn, knobs, coeffs, point, key).  coeffs: "rand" (n of them), 0, 1 or "n-3" coefficients; point: "rand",
# 0, 1 or "r-1"; key: "rand" or "dupneg" (duplicated and negated points, within and across the halves)
OPEN_GPU = [
    ("pallas", 15, {}, 0, "rand", "rand"),
    ("bn254", 15, {}, 1, 0, "dupneg"),
    ("bls12_381", 15, {}, "n-3", 1, "rand"),
    ("pallas", 16, {}, "rand", "r-1", "dupneg"),
    ("bn254", 16, {}, "n-3", "rand", "rand"),
    ("bls12_381", 16, {}, 1, "r-1", "dupneg"),
    ("pallas", 14, {"PCGPU_IPA_FREEZE": "0"}, "n-3", "rand", "rand"),
    ("bn254", 14, {"PCGPU_IPA_FREEZE": "0"}, "rand", 1, "rand"),
    ("bls12_381", 14, {"PCGPU_IPA_FREEZE": "0"}, 0, 0, "dupneg"),
    ("pallas", 12, {"PCGPU_MSM_SMALL": "0"}, "rand", 0, "dupneg"),
    ("bn254", 12, {"PCGPU_MSM_SMALL": "0"}, 0, "r-1", "rand"),
    ("bls12_381", 12, {"PCGPU_MSM_SMALL": "0"}, "n-3", "rand", "rand"),
    ("pallas", 12, {}, "rand", 1, "rand"),          # frozen at begin, split 3
    ("bn254", 12, {}, 0, "rand", "rand"),
    ("bls12_381", 12, {}, 1, "rand", "rand"),
    ("pallas", 8, {}, "n-3", "r-1", "rand"),        # frozen at begin, split 1
    ("bn254", 8, {}, "n-3", 0, "dupneg"),
    ("bls12_381", 8, {}, "rand", "rand", "dupneg"),
]
GLV_GPU = [("pallas", 15, {}), ("bn254", 15, {})]
CFG3 = ("pallas", 18)
OPEN_CPU = [
    ("pallas", 14, {}, "rand", "r-1", "dupneg"),    # SMALL split 6 -> SMALL split 3 -> frozen after the fold
    ("bn254", 11, {}, 0, 1, "rand"),
    ("bls12_381", 8, {}, "n-3", 0, "rand"),
    ("bn254", 10, {"PCGPU_IPA_FREEZE": "0"}, 1, "rand", "dupneg"),
    ("bls12_381", 9, {"PCGPU_IPA_FREEZE": "0"}, "rand", "r-1", "rand"),
    ("pallas", 10, {"PCGPU_MSM_SMALL": "0"}, 0, "rand", "rand"),
    ("bn254", 9, {"PCGPU_MSM_SMALL": "0"}, "rand", 0, "dupneg"),
    ("bls12_381", 8, {"PCGPU_MSM_SMALL": "0"}, "n-3", 1, "rand"),
    ("pallas", 9, {}, 1, 0, "rand"),                # frozen at begin, split 3
]
GLV_CPU = [("pallas", 9, {"PCGPU_IPA_FREEZE": "0"}), ("bn254", 8, {"PCGPU_IPA_FREEZE": "0"})]
IP_SIZES = [1, 2, 2047, 2048, 2049, 2050, 4097, (1 << 19) - 1, 1 << 19, (1 << 19) + 1, (1 << 20) + 3]
IP_SIZES_GPU = IP_SIZES + [1 << 22]
CHECK_LOGS_GPU = [0, 1, 12, 13, 18]
CHECK_LOGS_CPU = [0, 1, 12, 13]


def ipa_rounds(n, env, cname):
    """one dict per round of an open of length n under the knobs `env`: n_t, path, M, split (0 for BUCKETS) and the fold
    that ends the round ("glv", "plain" or "weights")"""
    off = lambda k: env.get(k, "")[:1] == "0"   # noqa: E731  (the library's test: the knob's first character is '0')
    small_on = not off("PCGPU_MSM_SMALL")
    freeze_on = small_on and not off("PCGPU_IPA_FREEZE")
    glv = cname in GLV_CURVES and not off("PCGPU_IPA_GLV")
    freeze = lambda nt: nt if freeze_on and 2 <= nt <= SMALL_MAX_N else 0   # noqa: E731
    out, nt, frozen = [], n, freeze(n)
    while nt > 1:
        m = nt // 2
        if frozen:
            path, M = "FROZEN", frozen
        elif small_on and m <= SMALL_ROUND_MAX_M:
            path, M = "SMALL", m
        else:
            path, M = "BUCKETS", m
        out.append(dict(n_t=nt, path=path, M=M, split=0 if path == "BUCKETS" else msm_cases.small_split(M),
                        fold="weights" if frozen else "glv" if glv else "plain"))
        frozen = frozen or freeze(m)
        nt = m
    return out


def handovers(rounds):
    """the transitions an open makes: path changes between rounds, "begin frozen" and "frozen after a fold" """
    out = {(a["path"], b["path"]) for a, b in zip(rounds, rounds[1:]) if a["path"] != b["path"]}
    if rounds and rounds[0]["path"] == "FROZEN":
        out.add("begin frozen")
    if any(a["fold"] != "weights" and b["path"] == "FROZEN" for a, b in zip(rounds, rounds[1:])):
        out.add("frozen after a fold")
    return out


def check_round(eng, pc, cname, rd):
    if rd["path"] == "BUCKETS":
        msm_cases.check_geometry(eng, pc, cname, rd["M"])
    else:
        msm_cases.check_geometry(eng, pc, cname, rd["M"], small=True, small_max=SMALL_ROUND_MAX_M)


# ---------------------------------------------------------------------------------------------------------------------------
# inputs and references
# ---------------------------------------------------------------------------------------------------------------------------
def neg_points(cname, xy):
    C = pyref.Curve(cname)
    return C.points_to_limbs([C.neg(p) for p in C.points_from_limbs(xy)])[0]


def open_inputs(cname, logn, coeffs, point, key, seed):
    """(key, coeffs, point, h') of one open row"""
    C = pyref.Curve(cname)
    n, m = 1 << logn, 1 << (logn - 1)
    comm_key = util.random_points(cname, n, seed=seed)
    if key == "dupneg":
        comm_key[1] = comm_key[0]                       # a duplicate within the left half
        comm_key[m] = comm_key[0]                       # key_r[0] == key_l[0]
        comm_key[3] = neg_points(cname, comm_key[2:3])[0]
        comm_key[m + 3] = neg_points(cname, comm_key[3:4])[0]      # key_r[3] == -key_l[3]
        comm_key[n - 1] = neg_points(cname, comm_key[m - 1:m])[0]  # key_r[m - 1] == -key_l[m - 1]
    nc = {"rand": n, "n-3": n - 3}.get(coeffs, coeffs)
    co = util.rand_fr(cname, nc, seed=seed + 1, mont=True) if nc else np.zeros((0, 4), dtype=np.uint64)
    if point == "rand":
        z = util.rand_fr(cname, 1, seed=seed + 2, mont=True)[0]
    else:
        z = C.fr_to_limbs([{"r-1": C.r - 1}.get(point, point)], True)[0]
    return comm_key, co, z, util.random_points(cname, 1, seed=seed + 3)[0]


def pmap(fn, items):
    with ThreadPoolExecutor(os.cpu_count() or 1) as ex:
        return list(ex.map(fn, items))


def weight_form_rounds(cname, comm_key, coeffs, point, h_prime, round_challenge):
    """the halving loop without a single fold: key_t[i] = sum_{j = i mod n_t} w_t[j] B[j] (csrc/ipa.cuh), so
      l_t = sum_j [(j mod n_t) <  n_t/2] w_t[j] coeffs_t[(j mod n_t) + n_t/2] B[j] + h' <coeffs_t,r, z_t,l>
      r_t = sum_j [(j mod n_t) >= n_t/2] w_t[j] coeffs_t[(j mod n_t) - n_t/2] B[j] + h' <coeffs_t,l, z_t,r>
    each one oracle MSM over the original key; challenges from pyref serialization and hashlib; coeffs_t, z_t from
    orc.fr_axpy.  Same return value as oracle_ipa_rounds."""
    import hashlib
    C = pyref.Curve(cname)
    n = comm_key.shape[0]
    co = np.zeros((n, 4), dtype=np.uint64); co[: coeffs.shape[0]] = coeffs
    z = orc.field_unop("orc_fr_to_mont", C.id, orc.fr_powers_canonical(C.id, point, n))
    w = np.tile(C.fr_to_limbs([1], True), (n, 1))
    j = np.arange(n)
    out = dict(l_vec=[], r_vec=[], l_inf=[], r_inf=[], challenges=[])
    nt = n
    while nt > 1:
        m = nt // 2
        pos = j & (nt - 1)
        right = pos >= m

        def commit(sel, src, ip):
            sc = orc.field_binop("orc_fr_mul", C.id, w[sel], co[src])
            msm, inf = orc.msm(C.id, comm_key[sel], orc.field_unop("orc_fr_from_mont", C.id, sc))
            hp, hinf = orc.g1_mul(C.id, h_prime, orc.field_unop("orc_fr_from_mont", C.id, ip.reshape(1, 4)))
            return orc.g1_sum(C.id, np.stack([msm, hp]), inf=np.array([inf, hinf], dtype=np.uint8))
        sel_l, sel_r = np.nonzero(~right)[0], np.nonzero(right)[0]
        (l, li), (r, ri) = pmap(lambda a: commit(*a), [
            (sel_l, pos[sel_l] + m, orc.fr_inner_product(C.id, co[m:nt], z[:m])),
            (sel_r, pos[sel_r] - m, orc.fr_inner_product(C.id, co[:m], z[m:nt]))])
        for k, v in (("l_vec", l), ("r_vec", r), ("l_inf", li), ("r_inf", ri)):
            out[k].append(v)
        data = int(round_challenge).to_bytes(32, "little") + pyref.g1_serialize(
            C, C.points_from_limbs(np.stack([l, r]), inf=[li, ri]), False)
        ctr = 0
        while True:                                   # compute_random_oracle_challenge (ipa_pc/mod.rs:74-87)
            v = int.from_bytes(hashlib.blake2s(data + ctr.to_bytes(8, "little")).digest(), "little") % (1 << C.r.bit_length())
            if v < C.r:
                break
            ctr += 1
        round_challenge = v
        out["challenges"].append(v)
        co[:m] = orc.fr_axpy(C.id, co[:m], C.fr_to_limbs([pow(v, -1, C.r)], True)[0], co[m:nt])
        z[:m] = orc.fr_axpy(C.id, z[:m], C.fr_to_limbs([v], True)[0], z[m:nt])
        w[right] = orc.field_binop("orc_fr_mul", C.id, w[right], np.tile(C.fr_to_limbs([v], True), (int(right.sum()), 1)))
        nt = m
    out["final_comm_key"] = orc.msm(C.id, comm_key, orc.field_unop("orc_fr_from_mont", C.id, w))[0]
    out["c"] = co[0]
    return out


def compare_open(got, exp, what):
    assert got["challenges"] == exp["challenges"], what
    for t, (a, b, c, d) in enumerate(zip(got["l_vec"], exp["l_vec"], got["r_vec"], exp["r_vec"])):
        assert (a == b).all(), (what, "l", t)
        assert (c == d).all(), (what, "r", t)
    assert len(got["l_vec"]) == len(exp["l_vec"]) == len(exp["challenges"]), what
    assert (got["final_comm_key"] == exp["final_comm_key"]).all(), (what, "final_comm_key")
    assert (got["c"] == exp["c"]).all(), (what, "c")


# ---------------------------------------------------------------------------------------------------------------------------
# case bodies
# ---------------------------------------------------------------------------------------------------------------------------
def checked_open(eng, pc, cname, key, coeffs, point, h_prime, chal, **kw):
    """ipa_pc.open_rounds with every round's path, M and split asserted (the policy under the knobs now in the environment),
    and the report of ipa_finish on a frozen key"""
    from poly_commit_b200 import ipa_pc
    C = pyref.Curve(cname)
    rounds = ipa_rounds(key.shape[0] if kw.get("n") is None else kw["n"], os.environ, cname)
    got = ipa_pc.open_rounds(eng, C.id, key, coeffs, point, h_prime, chal,
                             on_round=lambda t: check_round(eng, pc, cname, rounds[t]), **kw)
    assert len(got["l_vec"]) == len(rounds)
    frozen = [rd["M"] for rd in rounds if rd["path"] == "FROZEN"]
    if frozen:   # final_comm_key = sum_j w[j] B[j]: one more one-launch MSM over the frozen key
        msm_cases.check_geometry(eng, pc, cname, frozen[0], small=True)
    return got


def open_case(eng, pc, cname, logn, knobs, coeffs, point, key, monkeypatch, seed):
    for k, v in knobs.items():
        monkeypatch.setenv(k, v)
    comm_key, co, z, h_prime = open_inputs(cname, logn, coeffs, point, key, seed)
    chal = 0x5eed + seed
    with ThreadPoolExecutor(1) as ex:
        ref = weight_form_rounds if logn > EXPLICIT_MAX_LOG else oracle_ipa_rounds
        oracle = ex.submit(ref, cname, comm_key, co, z, h_prime, chal)    # overlaps the device open
        got = checked_open(eng, pc, cname, comm_key, co, z, h_prime, chal)
        exp = oracle.result()
    compare_open(got, exp, (cname, logn, knobs, coeffs, point, key))
    if coeffs == 0:   # l = r = identity in every round, and the transcript (equal challenges) hashed the infinity flag
        assert all(exp["l_inf"]) and all(exp["r_inf"])
    return comm_key, got


def glv_case(eng, pc, cname, logn, knobs, monkeypatch, seed):
    """the GLV fold and the 256-step fold over the same open: equal to each other and to the oracle"""
    for k, v in knobs.items():
        monkeypatch.setenv(k, v)
    comm_key, co, z, h_prime = open_inputs(cname, logn, "rand", "rand", "rand", seed)
    exp = oracle_ipa_rounds(cname, comm_key, co, z, h_prime, 3)
    for flag in ("1", "0"):       # each equal to the oracle, hence to each other
        monkeypatch.setenv("PCGPU_IPA_GLV", flag)
        rounds = ipa_rounds(1 << logn, dict(knobs, PCGPU_IPA_GLV=flag), cname)
        assert {rd["fold"] for rd in rounds} >= {"glv" if flag == "1" else "plain"}
        compare_open(checked_open(eng, pc, cname, comm_key, co, z, h_prime, 3), exp, (cname, logn, "glv", flag))


def fold_exceptions_case(eng, pc, cname, glv, monkeypatch):
    """one explicit fold key_l + c * key_r (n = 1024, m = 512: lanes in four 128-thread blocks) with the exceptional final
    additions key_l = c * key_r (a doubling) and key_l = -c * key_r (the identity, through xyzz_to_affine_gcd), an identity on
    the left, on the right and on both sides; then random folds to one point, which must be sum_j w[j] B[j] -- every
    lane of every fold carries a distinct random weight, so a wrong lane changes the result"""
    from poly_commit_b200 import params
    C = pyref.Curve(cname)
    monkeypatch.setenv("PCGPU_IPA_FREEZE", "0")
    monkeypatch.setenv("PCGPU_IPA_GLV", "1" if glv else "0")
    n, m = 1024, 512
    key = util.random_points(cname, n, seed=410)
    chals = [C.r - 2, 3] + util.rand_fr_ints(cname, 8, seed=411)
    c0 = chals[0]
    for i, k in ((5, c0), (140, C.r - c0), (300, c0), (401, C.r - c0)):
        key[i] = orc.g1_mul(C.id, key[m + i], C.fr_to_limbs([k], False))[0]
    pts = C.points_from_limbs(key[[140, m + 140]])
    assert C.add(pts[0], C.mul(c0, pts[1])) is None                      # the lane really folds to the identity
    key[270] = 0            # identity on the left
    key[m + 400] = 0        # identity on the right
    key[511] = key[m + 511] = 0
    inf = np.array([0 if p.any() else 1 for p in key], dtype=np.uint8)
    coeffs, z = util.rand_fr(cname, n, seed=412, mont=True), util.rand_fr(cname, 1, seed=413, mont=True)[0]
    st = eng.ipa_begin(C.id, key, coeffs, z)
    for c in chals:
        eng.ipa_round_fold(st, params.fr_mont(C.id, c), params.fr_mont(C.id, pow(c, -1, C.r)))
    assert eng.ipa_len(st) == 1
    got = eng.ipa_finish(C.id, st)[0]
    w = [1] * n
    for t, c in enumerate(chals):
        bit = 1 << (len(chals) - 1 - t)
        w = [x * c % C.r if j & bit else x for j, x in enumerate(w)]
    exp, einf = orc.msm(C.id, key, C.fr_to_limbs(w, False), inf=inf)
    assert einf == 0 and (got == exp).all(), (cname, glv)


def ip_case(eng, cname, n, kind, seed):
    """fr_inner_product of n elements: random operands (against orc.fr_inner_product), every operand r - 1 (n mod r: (r-1)^2 =
    1) or one vector zero"""
    C = pyref.Curve(cname)
    if kind == "rand":
        a, b = util.rand_fr_fast(cname, n, seed), util.rand_fr_fast(cname, n, seed + 1)
        exp = orc.fr_inner_product(C.id, a, b)
    elif kind == "r-1":
        a = b = np.tile(C.fr_to_limbs([C.r - 1], True), (n, 1))
        exp = C.fr_to_limbs([n % C.r], True)[0]
    else:
        a, b = util.rand_fr_fast(cname, n, seed), np.zeros((n, 4), dtype=np.uint64)
        exp = np.zeros(4, dtype=np.uint64)
    assert (eng.fr_inner_product(C.id, a, b) == exp).all(), (cname, n, kind)
    if kind == "zero":
        assert not eng.fr_inner_product(C.id, b, a).any(), (cname, n, "zero first")


def check_final_key_case(eng, pc, cname, log_d, key, seed):
    C = pyref.Curve(cname)
    chals = util.rand_fr_ints(cname, log_d, seed)
    srs = eng.srs_register(C.id, key)
    got = eng.ipa_check_final_key(srs, np.stack([util.fr_const(cname, c) for c in chals]) if log_d else np.zeros((0, 4)))
    msm_cases.check_geometry(eng, pc, cname, 1 << log_d, small=True)
    srs.release()
    co = [1]
    for c in reversed(chals):          # the last challenge on bit 0, the first on the top bit
        co = co + [x * c % C.r for x in co]
    exp = orc.msm(C.id, key[: 1 << log_d], C.fr_to_limbs(co, False))
    assert got[1] == exp[1] and (got[0] == exp[0]).all(), (cname, log_d)


def check_final_key_errors_case(eng, cname):
    C = pyref.Curve(cname)
    key = util.random_points(cname, 8, seed=430)
    srs = eng.srs_register(C.id, key)
    ch = np.stack([util.fr_const(cname, 5 + i) for i in range(27)])
    out, inf = np.zeros(2 * 6, dtype=np.uint64), np.zeros(1, dtype=np.uint8)
    vp = ctypes.c_void_p
    call = lambda k: eng.lib.pcgpu_ipa_check_final_key(eng.ctx, srs.handle, ch.ctypes.data_as(vp), k,   # noqa: E731
                                                       out.ctypes.data_as(vp), inf.ctypes.data_as(vp))
    assert call(4) == E_LEN and call(27) == E_BADARG
    assert call(3) == 0
    srs.release()


def device_ptrs_case(eng, pc, cname, logn, seed):
    """an open with key and coefficients in device buffers (PCGPU_DEVICE_PTRS) gives the proof of the host-buffer open"""
    comm_key, co, z, h_prime = open_inputs(cname, logn, "n-3", "rand", "rand", seed)
    host = checked_open(eng, pc, cname, comm_key, co, z, h_prime, 11)
    kp, keep_k = util.dev_ptr(eng, comm_key)
    cp, keep_c = util.dev_ptr(eng, co)
    dev = checked_open(eng, pc, cname, kp, cp, z, h_prime, 11, n=comm_key.shape[0], n_coeffs=co.shape[0],
                       flags=pc.DEVICE_PTRS)
    compare_open(dev, host, (cname, logn, "device pointers"))
    del keep_k, keep_c


def arena_case(eng, pc, cname, logns, seed):
    """opens of different sizes one after the other on one context (the IPA arena grows, then is reused), each against the
    oracle; a second ipa_begin while an open is active is PCGPU_E_BADARG and leaves the first open intact; ipa_round_lr and
    ipa_round_fold on a length-1 state are PCGPU_E_BADARG"""
    from poly_commit_b200 import binding, ipa_pc
    C = pyref.Curve(cname)
    for i, logn in enumerate(logns):
        comm_key, co, z, h_prime = open_inputs(cname, logn, "rand", "rand", "rand", seed + 10 * i)
        exp = oracle_ipa_rounds(cname, comm_key, co, z, h_prime, 9)
        compare_open(checked_open(eng, pc, cname, comm_key, co, z, h_prime, 9), exp, (cname, logn, i))
    comm_key, co, z, h_prime = open_inputs(cname, 4, "rand", "rand", "rand", seed + 99)
    exp = oracle_ipa_rounds(cname, comm_key, co, z, h_prime, 9)
    st = eng.ipa_begin(C.id, comm_key, co, z)
    with pytest.raises(binding.PcgpuError) as e:
        eng.ipa_begin(C.id, comm_key, co, z)
    assert e.value.code == E_BADARG
    rc, chals, ls = 9, [], []
    while eng.ipa_len(st) > 1:
        l, li, r, ri = eng.ipa_round_lr(C.id, st, h_prime, with_inf=True)
        ls.append(l)
        rc = ipa_pc.compute_random_oracle_challenge(C.id, ipa_pc.round_transcript(eng, C.id, rc, l, li, r, ri))
        chals.append(rc)
        eng.ipa_round_fold(st, ipa_pc._fr_mont(C.id, rc), ipa_pc._fr_mont(C.id, pow(rc, -1, C.r)))
    for call in (lambda: eng.ipa_round_lr(C.id, st, h_prime), lambda: eng.ipa_round_fold(st, ipa_pc._fr_mont(C.id, 2),
                                                                                           ipa_pc._fr_mont(C.id, 2))):
        with pytest.raises(binding.PcgpuError) as e:
            call()
        assert e.value.code == E_BADARG
    fk, c = eng.ipa_finish(C.id, st)
    assert chals == exp["challenges"] and all((a == b).all() for a, b in zip(ls, exp["l_vec"]))
    assert (fk == exp["final_comm_key"]).all() and (c == exp["c"]).all()


# ---------------------------------------------------------------------------------------------------------------------------
# the policy and its coverage
# ---------------------------------------------------------------------------------------------------------------------------
def test_round_policy_coverage():
    """the device parameter lists reach every path, every split, every hand-over and both explicit folds on every curve where
    they exist; the cfg3 open runs all 18 rounds"""
    rows = [(c, lg, k) for c, lg, k, *_ in OPEN_GPU] + [(c, lg, dict(k, PCGPU_IPA_GLV=f)) for c, lg, k in GLV_GPU for f in "01"]
    rows.append((CFG3[0], CFG3[1], {}))
    seen = {c: set() for c in util.CURVE_NAMES}
    for cname, logn, knobs in rows:
        rounds = ipa_rounds(1 << logn, knobs, cname)
        assert len(rounds) == logn
        seen[cname] |= {("path", rd["path"]) for rd in rounds} | {("fold", rd["fold"]) for rd in rounds}
        seen[cname] |= {("split", rd["path"], rd["split"]) for rd in rounds} | set(handovers(rounds))
    want = {("path", p) for p in ("FROZEN", "SMALL", "BUCKETS")} | {("fold", f) for f in ("plain", "weights")}
    want |= {("split", "SMALL", s) for s in (1, 3, 6)} | {("split", "FROZEN", s) for s in (1, 3)}
    want |= {("BUCKETS", "SMALL"), ("SMALL", "FROZEN"), "begin frozen", "frozen after a fold"}
    for cname in util.CURVE_NAMES:
        w = want | ({("fold", "glv")} if cname in GLV_CURVES else set())
        assert not w - seen[cname], (cname, sorted(map(str, w - seen[cname])))
        assert cname in GLV_CURVES or ("fold", "glv") not in seen[cname]
    # the default open of 2^15: BUCKETS (m = 16384) -> SMALL split 6 -> SMALL split 3 -> frozen at 4096 down to m = 1
    assert [(rd["path"], rd["M"], rd["split"]) for rd in ipa_rounds(1 << 15, {}, "pallas")[:4]] == [
        ("BUCKETS", 16384, 0), ("SMALL", 8192, 6), ("SMALL", 4096, 3), ("FROZEN", 4096, 3)]
    # every edge input meets a BUCKETS, a SMALL and a FROZEN round
    for col, values in ((3, (0, 1, "n-3")), (4, (0, 1, "r-1")), (5, ("dupneg",))):
        for v in values:
            paths = {rd["path"] for row in OPEN_GPU if row[col] == v for rd in ipa_rounds(1 << row[1], row[2], row[0])}
            assert paths == {"FROZEN", "SMALL", "BUCKETS"}, (col, v, paths)
    # the CPU rows run a split-6 SMALL round and BUCKETS rounds
    cpu = {(rd["path"], rd["split"]) for c, lg, k, *_ in OPEN_CPU for rd in ipa_rounds(1 << lg, k, c)}
    assert {("SMALL", 6), ("SMALL", 3), ("SMALL", 1), ("FROZEN", 3), ("FROZEN", 1), ("BUCKETS", 0)} <= cpu
    assert all(lg <= 14 for _, lg, *_ in OPEN_CPU) and all(lg <= 10 for _, lg, k, *_ in OPEN_CPU if k.get("PCGPU_MSM_SMALL"))


# ---------------------------------------------------------------------------------------------------------------------------
# host emulation
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emul(pc, hostcheck_path, oracle):
    e = pc.Engine(0, lib_path=hostcheck_path)
    yield e
    e.close()


@pytest.mark.parametrize("cname,logn,knobs,coeffs,point,key", OPEN_CPU)
def test_emul_open(emul, pc, cname, logn, knobs, coeffs, point, key, monkeypatch):
    open_case(emul, pc, cname, logn, knobs, coeffs, point, key, monkeypatch, seed=500 + OPEN_CPU.index(
        (cname, logn, knobs, coeffs, point, key)) * 10)


@pytest.mark.parametrize("cname,logn,knobs", GLV_CPU)
def test_emul_glv_and_plain_fold(emul, pc, cname, logn, knobs, monkeypatch):
    glv_case(emul, pc, cname, logn, knobs, monkeypatch, seed=600)


@pytest.mark.parametrize("cname,glv", [("pallas", True), ("pallas", False), ("bn254", True), ("bn254", False),
                                       ("bls12_381", False)])
def test_emul_fold_exceptions(emul, pc, cname, glv, monkeypatch):
    fold_exceptions_case(emul, pc, cname, glv, monkeypatch)


@pytest.mark.parametrize("n", IP_SIZES)
@pytest.mark.parametrize("cname", util.CURVE_NAMES)
def test_emul_inner_product_shapes(emul, cname, n):
    for kind in ("rand", "r-1", "zero"):
        ip_case(emul, cname, n, kind, seed=n % 1000)


@pytest.mark.parametrize("cname", util.CURVE_NAMES)
def test_emul_check_final_key(emul, pc, cname):
    key = util.random_points(cname, 1 << max(CHECK_LOGS_CPU), seed=420)
    for log_d in CHECK_LOGS_CPU:
        check_final_key_case(emul, pc, cname, log_d, key, seed=421 + log_d)
    check_final_key_errors_case(emul, cname)


def test_emul_device_ptrs(emul, pc):
    device_ptrs_case(emul, pc, "bn254", 8, seed=700)


def test_emul_arena_reuse(pc, hostcheck_path, oracle):
    e = pc.Engine(0, lib_path=hostcheck_path)
    try:
        arena_case(e, pc, "pallas", (9, 3, 9), seed=710)
    finally:
        e.close()


# ---------------------------------------------------------------------------------------------------------------------------
# the device
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cname,logn,knobs,coeffs,point,key", OPEN_GPU)
def test_gpu_open(gpu_engine, pc, cname, logn, knobs, coeffs, point, key, monkeypatch):
    open_case(gpu_engine, pc, cname, logn, knobs, coeffs, point, key, monkeypatch, seed=800 + OPEN_GPU.index(
        (cname, logn, knobs, coeffs, point, key)) * 10)


@pytest.mark.gpu
@pytest.mark.parametrize("cname,logn,knobs", GLV_GPU)
def test_gpu_glv_and_plain_fold(gpu_engine, pc, cname, logn, knobs, monkeypatch):
    glv_case(gpu_engine, pc, cname, logn, knobs, monkeypatch, seed=900)


@pytest.mark.gpu
def test_gpu_cfg3_open_2p18_pallas(gpu_engine, pc, monkeypatch):
    """BASELINE.json cfg3: InnerProductArgPC open, degree 2^18 - 1, Pallas: all 18 rounds against the weight form, the
    verifier's recomputed key (check_poly.compute_coeffs() + cm_commit, ipa_pc/mod.rs:760-766) equal to final_comm_key"""
    from poly_commit_b200 import ipa_pc
    cname, logn = CFG3
    comm_key, got = open_case(gpu_engine, pc, cname, logn, {}, "rand", "rand", "rand", monkeypatch, seed=40)
    vk = ipa_pc.check_final_key(gpu_engine, pyref.Curve(cname).id, comm_key, got["challenges"])
    assert vk[1] == 0 and (vk[0] == got["final_comm_key"]).all()


@pytest.mark.gpu
@pytest.mark.parametrize("cname,glv", [("pallas", True), ("pallas", False), ("bn254", True), ("bn254", False),
                                       ("bls12_381", False)])
def test_gpu_fold_exceptions(gpu_engine, pc, cname, glv, monkeypatch):
    fold_exceptions_case(gpu_engine, pc, cname, glv, monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("n", IP_SIZES_GPU)
@pytest.mark.parametrize("cname", util.CURVE_NAMES)
def test_gpu_inner_product_shapes(gpu_engine, cname, n):
    for kind in ("rand", "r-1", "zero"):
        ip_case(gpu_engine, cname, n, kind, seed=n % 1000)


@pytest.mark.gpu
@pytest.mark.parametrize("cname", util.CURVE_NAMES)
def test_gpu_check_final_key(gpu_engine, pc, cname):
    key = util.random_points(cname, 1 << max(CHECK_LOGS_GPU), seed=420)
    for log_d in CHECK_LOGS_GPU:
        check_final_key_case(gpu_engine, pc, cname, log_d, key, seed=421 + log_d)
    check_final_key_errors_case(gpu_engine, cname)


@pytest.mark.gpu
@pytest.mark.parametrize("cname", ["pallas", "bls12_381"])
def test_gpu_device_ptrs(gpu_engine, pc, cname):
    device_ptrs_case(gpu_engine, pc, cname, 16, seed=700)


@pytest.mark.gpu
def test_gpu_arena_reuse(pc, oracle):
    e = pc.Engine(0)
    try:
        arena_case(e, pc, "pallas", (15, 3, 15), seed=710)
    finally:
        e.close()
