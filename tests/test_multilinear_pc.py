"""MultilinearPC (XZZPD19, multilinear_pc/mod.rs): pcgpu_mlpc_register / pcgpu_mlpc_open and poly_commit_b200.multilinear_pc,
against a Python-integer transcription of the reference's setup and open, on the host-emulated kernels and on the device.

The G2 keys are trapdoor keys: every base is k H with a known k (built by pcgpu_g2_fixed_base_mul, sampled against pyref),
so a transcribed proof  sum_x q[x >> 1] H_i[x]  is  (sum_x q[x >> 1] k_i[x]) H, one Python scalar multiplication.  For an
honest key from a known t the closed forms hold as well: proof i = q_i(t_{i+1}, ..., t_{nv-1}) h, commit = p(t) g and the
returned value is p(point)."""
import importlib

import numpy as np
import pytest

from oracle import pyref
from tests import g2_cases as gc
from tests import util


# ---- the reference, transcribed in Python integers ---------------------------------------------------------------------
def ref_eq_extension(t, r):
    dim = len(t)
    res = []
    for i in range(dim):
        poly = []
        for x in range(1 << dim):
            xi = 1 if (x >> i) & 1 else 0
            ti_xi = t[i] * xi
            poly.append((ti_xi + ti_xi - xi - t[i] + 1) % r)
        res.append(poly)
    return res


def ref_remove_dummy_variable(poly, pad):
    if pad == 0:
        return list(poly)
    nv = (len(poly) - 1).bit_length() - pad
    return [poly[x << pad] for x in range(1 << nv)]


def ref_pp_powers(t, r):
    """setup :39-59"""
    nv = len(t)
    eq = ref_eq_extension(t, r)
    eq_arr = []
    base = eq.pop()
    for i in reversed(range(nv)):
        eq_arr.insert(0, ref_remove_dummy_variable(base, i))
        if i != 0:
            mul = eq.pop()
            base = [a * b % r for a, b in zip(base, mul)]
    out = []
    for i in range(nv):
        out.extend(eq_arr[i][x] for x in range(1 << (nv - i)))
    return out


def ref_open(r, evals, point):
    """open :131-168 with the MSM left symbolic: per level the scalars q[x >> 1] (over 2^k bases) and the final r[0]"""
    nv = len(point)
    rr = list(evals)
    levels = []
    for i in range(nv):
        k = nv - i
        x = point[i]
        q = [(rr[2 * b + 1] - rr[2 * b]) % r for b in range(1 << (k - 1))]
        rr = [(rr[2 * b] * (1 - x) + rr[2 * b + 1] * x) % r for b in range(1 << (k - 1))]
        levels.append([q[j >> 1] for j in range(1 << k)])
    return levels, rr[0]


def mle_eval(vals, pts, r):
    """the multilinear extension of `vals` at pts (variable 0 = the lowest index bit)"""
    v = list(vals)
    for x in pts:
        v = [(v[2 * b] * (1 - x) + v[2 * b + 1] * x) % r for b in range(len(v) // 2)]
    return v[0]


def mlpc_module(pc):
    return importlib.import_module(pc.__name__ + ".multilinear_pc")


# ---- cases -------------------------------------------------------------------------------------------------------------
def make_key(eng, pc, cname, nv, kind, seed):
    """levels of trapdoor exponents k_i (2^(nv-i) each) and their G2 points.  kind: 'random' (not an honest key),
    'double' (H[2b+1] = H[2b]), 'cancel' (H[2b+1] = -H[2b]), 'identity' (every 5th base the identity, by flag)"""
    r = pyref.Curve(cname).r
    ks, flags = [], []
    for i in range(nv):
        k = util.rand_fr_ints(cname, 1 << (nv - i), seed + i)
        if kind == "double":
            k = [k[j & ~1] for j in range(len(k))]
        elif kind == "cancel":
            k = [k[j] if j % 2 == 0 else (r - k[j - 1]) % r for j in range(len(k))]
        f = np.zeros(len(k), dtype=np.uint8)
        if kind == "identity":
            for j in range(0, len(k), 5):
                k[j] = 0
                f[j] = 1
        ks.append(k)
        flags.append(f)
    flat = [v for k in ks for v in k]
    pts = gc.trapdoor_bases(eng, pc, cname, flat, sample=8, seed=seed)
    levels, start = [], 0
    for k in ks:
        levels.append(pts[start:start + len(k)])
        start += len(k)
    return ks, levels, flags


def open_case(eng, pc, cname, nv, kind="random", seed=0, evals=None, point=None, device_ptrs=False):
    C = pyref.Curve(cname)
    r = C.r
    G = pyref.G2(cname)
    H = gc.generator(cname)
    ks, levels, flags = make_key(eng, pc, cname, nv, kind, seed)
    key = eng.mlpc_register(C.id, levels, inf=flags if kind == "identity" else None)
    ev = evals if evals is not None else util.rand_fr_ints(cname, 1 << nv, seed + 100)
    pt = point if point is not None else util.rand_fr_ints(cname, nv, seed + 200)
    ev_l = C.fr_to_limbs(ev, True)
    flags_arg = 0
    if device_ptrs:
        ptr, owner = util.dev_ptr(eng, ev_l)
        ev_arg, flags_arg = ptr, pc.DEVICE_PTRS
    else:
        ev_arg = ev_l
    proofs, pinf, value = eng.mlpc_open(key, ev_arg, C.fr_to_limbs(pt, True), n=1 << nv, flags=flags_arg)
    key.release()
    scal, val = ref_open(r, ev, pt)
    assert C.fr_from_limbs(value, True)[0] == val == mle_eval(ev, pt, r)
    for i in range(nv):
        exp = G.mul(sum(s * k for s, k in zip(scal[i], ks[i])) % r, H)
        assert gc.from_limbs(cname, proofs[i], pinf[i]) == exp, (cname, nv, kind, i)
    return proofs, pinf


def naive_case(eng, pc, cname, nv, seed=5):
    """small nv: the proofs against pyref's naive G2 MSM over the (unfolded) key points"""
    C = pyref.Curve(cname)
    G = pyref.G2(cname)
    ks, levels, _ = make_key(eng, pc, cname, nv, "random", seed)
    ev = util.rand_fr_ints(cname, 1 << nv, seed + 1)
    pt = util.rand_fr_ints(cname, nv, seed + 2)
    key = eng.mlpc_register(C.id, levels)
    proofs, pinf, _ = eng.mlpc_open(key, C.fr_to_limbs(ev, True), C.fr_to_limbs(pt, True))
    key.release()
    scal, _ = ref_open(C.r, ev, pt)
    for i in range(nv):
        exp = None
        for s, row in zip(scal[i], levels[i]):
            exp = G.add(exp, G.mul(s, gc.from_limbs(cname, row)))
        assert gc.from_limbs(cname, proofs[i], pinf[i]) == exp


def honest_case(eng, pc, cname, nv, seed=7, device_ptrs=False):
    """setup / trim / commit / open through poly_commit_b200.multilinear_pc with a known t: proof i = q_i(t_{i+1}, ..) h,
    commit = p(t) g, value = p(point)"""
    mlpc = mlpc_module(pc)
    C = pyref.Curve(cname)
    r = C.r
    G2 = pyref.G2(cname)
    H = gc.generator(cname)
    t = gc.fr_ints(util.rand_fr(cname, nv + 1, seed, mont=False))
    h_xy, _ = gc.to_limbs(cname, [H])
    g_xy, _ = C.points_to_limbs([C.g])
    params = mlpc.setup(eng, C.id, t, g_xy[0], h_xy[0])
    ck, vk = mlpc.trim(params, nv)
    tt = t[1:]
    assert len(ck["powers_of_h"]) == nv and ck["powers_of_h"][0].shape[0] == 1 << nv
    for j in (0, (1 << nv) - 1):    # the key itself: powers_of_h[0][x] = eq(t, x) h
        assert gc.from_limbs(cname, ck["powers_of_h"][0][j]) == G2.mul(mlpc.pp_powers(tt, r)[j], H)
    assert C.points_from_limbs(vk["g_mask_random"][-1:])[0] == C.mul(t[-1], C.g)
    com = mlpc.Committer(eng, C.id, ck)
    ev_l = util.rand_fr(cname, 1 << nv, seed + 1, mont=True)
    ev = C.fr_from_limbs(ev_l, True)
    pt = gc.fr_ints(util.rand_fr(cname, nv, seed + 2, mont=False))
    cxy, cinf = com.commit(ev_l)
    assert C.points_from_limbs(cxy.reshape(1, -1), [cinf])[0] == C.mul(mle_eval(ev, tt, r), C.g)
    if device_ptrs:
        ptr, owner = util.dev_ptr(eng, ev_l)
        proofs, pinf, value = eng.mlpc_open(com.h_key, ptr, C.fr_to_limbs(pt, True), n=1 << nv, flags=pc.DEVICE_PTRS)
    else:
        proofs, pinf, value = com.open(ev_l, C.fr_to_limbs(pt, True))
    com.release()
    assert C.fr_from_limbs(value, True)[0] == mle_eval(ev, pt, r)
    rr = ev
    for i in range(nv):
        x = pt[i]
        q = [(rr[2 * b + 1] - rr[2 * b]) % r for b in range(len(rr) // 2)]
        rr = [(rr[2 * b] + x * qb) % r for b, qb in enumerate(q)]
        assert gc.from_limbs(cname, proofs[i], pinf[i]) == G2.mul(mle_eval(q, tt[i + 1:], r), H), (cname, nv, i)


def errors_case(eng, pc, cname):
    C = pyref.Curve(cname)
    ks, levels, _ = make_key(eng, pc, cname, 3, "random", 30)
    key = eng.mlpc_register(C.id, levels)
    pt = C.fr_to_limbs([1, 2, 3], True)
    for n in (7, 9, 0):
        ev = C.fr_to_limbs(list(range(max(n, 1))), True)
        with pytest.raises(pc.PcgpuError) as e:
            eng.mlpc_open(key, ev, pt, n=n)
        assert e.value.code == -4
    key.release()
    for bad in (lambda: eng.mlpc_register(C.id, []),                       # nv = 0
                lambda: eng.mlpc_register(pc.PALLAS, levels),              # no G2
                lambda: eng.mlpc_register(gc.group(pc, cname), levels)):   # a group id is not a curve here
        with pytest.raises(pc.PcgpuError) as e:
            bad()
        assert e.value.code == -3
    with pytest.raises(pc.PcgpuError) as e:
        pc.binding.Engine.mlpc_open(eng, pc.binding.MlpcKey(eng, None, C.id, 3), C.fr_to_limbs([0] * 8, True), pt)
    assert e.value.code == -3


# ---- host emulation ----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emul(pc, hostcheck_path):
    e = pc.Engine(0, lib_path=hostcheck_path)
    yield e
    e.close()


@pytest.mark.parametrize("cname", gc.PAIRING)
def test_emul_pp_powers_match_reference(pc, cname):
    r = pyref.Curve(cname).r
    for nv in range(1, 8):
        t = util.rand_fr_ints(cname, nv, nv)
        assert mlpc_module(pc).pp_powers(t, r) == ref_pp_powers(t, r)
        assert mlpc_module(pc).eq_extension(t, r) == ref_eq_extension(t, r)


@pytest.mark.parametrize("cname", gc.PAIRING)
@pytest.mark.parametrize("nv", range(1, 9))
def test_emul_open_random_key(emul, pc, cname, nv):
    open_case(emul, pc, cname, nv, "random", seed=nv)


@pytest.mark.parametrize("cname", gc.PAIRING)
@pytest.mark.parametrize("kind", ["double", "cancel", "identity"])
def test_emul_open_exceptional_keys(emul, pc, cname, kind):
    for nv in (1, 4, 6):
        open_case(emul, pc, cname, nv, kind, seed=40 + nv)


@pytest.mark.parametrize("cname", gc.PAIRING)
def test_emul_open_special_polynomials(emul, pc, cname):
    r = pyref.Curve(cname).r
    nv = 5
    proofs, pinf = open_case(emul, pc, cname, nv, evals=[12345] * (1 << nv), seed=50)      # constant: every proof is O
    assert pinf.all() and not proofs.any()
    ev = [util.rand_fr_ints(cname, 1, 51 + (x >> 1))[0] for x in range(1 << nv)]        # independent of variable 0
    proofs, pinf = open_case(emul, pc, cname, nv, evals=ev, seed=52)
    assert pinf[0] == 1
    open_case(emul, pc, cname, nv, point=[0, 1, 0, 1, r - 1], seed=53)
    open_case(emul, pc, cname, nv, point=[1] * nv, seed=54, device_ptrs=True)


@pytest.mark.parametrize("cname", gc.PAIRING)
def test_emul_open_vs_naive_msm(emul, pc, cname):
    naive_case(emul, pc, cname, 4)


@pytest.mark.parametrize("cname", gc.PAIRING)
def test_emul_honest_setup_commit_open(emul, pc, cname):
    honest_case(emul, pc, cname, 6)


@pytest.mark.parametrize("cname", gc.PAIRING)
def test_emul_errors(emul, pc, cname):
    errors_case(emul, pc, cname)


# ---- device ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cname", gc.PAIRING)
def test_gpu_honest_nv16_nv20(gpu_engine, pc, cname):
    honest_case(gpu_engine, pc, cname, 16, seed=60)
    honest_case(gpu_engine, pc, cname, 20, seed=61, device_ptrs=True)


@pytest.mark.gpu
@pytest.mark.parametrize("cname", gc.PAIRING)
def test_gpu_random_key_nv10(gpu_engine, pc, cname):
    open_case(gpu_engine, pc, cname, 10, "random", seed=70)
    open_case(gpu_engine, pc, cname, 10, "cancel", seed=71, device_ptrs=True)
    naive_case(gpu_engine, pc, cname, 5, seed=72)
    errors_case(gpu_engine, pc, cname)
