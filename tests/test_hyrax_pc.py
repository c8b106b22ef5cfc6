"""HyraxPC on the device (pcgpu_hyrax_commit / _open / _check, poly_commit_b200.hyrax): one set of case bodies, run on the
host-emulated kernels and, under -m gpu, on the H100.

References: tests/hyrax_ref.py (a pure-Python HyraxPC over oracle/pyref.py: proofs compared byte for byte), pcgpu_msm_batch on
the host-transposed block, the C oracle (orc.msm, orc.fr_row_mul) and an independent fold of the multilinear polynomial.
"""
import ctypes

import numpy as np
import pytest

from oracle import orc, pyref
from tests import hyrax_ref as ref
from tests import util

CURVES = util.CURVE_NAMES


@pytest.fixture(scope="module")
def emul(pc, hostcheck_path):
    e = pc.Engine(0, lib_path=hostcheck_path)
    yield e
    e.close()


class Keys:
    """dim + 1 independent points k_i G as com_key || h (setup's hash-to-curve is checked separately), registered with comb
    tables"""

    def __init__(self, eng, cname, nv, seed=1):
        from poly_commit_b200 import hyrax
        self.eng, self.cname, self.nv = eng, cname, nv
        self.C = pyref.Curve(cname)
        self.dim = 1 << (nv // 2)
        self.xy = util.random_points(cname, self.dim + 1, seed)
        pts = self.C.points_from_limbs(self.xy)
        self.com_key, self.h = pts[:self.dim], pts[self.dim]
        self.ck = hyrax.CommitterKey(eng, self.C.id, self.xy[:self.dim], self.xy[self.dim])


def mont(C, vals):
    return C.fr_to_limbs(list(vals), True)


def ints(C, limbs):
    return C.fr_from_limbs(np.asarray(limbs, dtype=np.uint64).reshape(-1, 4), True)


def point_bytes(C, P):
    xy, inf = C.points_to_limbs([P])
    return xy[0], bool(inf[0])


def same_point(C, got, P):
    exp_xy, exp_inf = point_bytes(C, P)
    return bool(got[1]) == exp_inf and (np.asarray(got[0], dtype=np.uint64) == exp_xy).all()


def draws(C, n, seed):
    return util.rand_fr_ints(C.name, n, seed) if n else []


def challenge_fn(C, seed, log=None):
    cs = draws(C, 64, seed)

    def f(j, com_eval, com_d, com_b):
        if log is not None:
            log.append((j, com_eval, com_d, com_b))
        return mont(C, [cs[j]])[0]
    return f, cs


# ---- commit ---------------------------------------------------------------------------------------------------------------
def commit_case(eng, cname, nv, seed=3):
    """row commitments equal hyrax_ref's and pcgpu_msm_batch's over the host-transposed block; device-pointer evals agree"""
    from poly_commit_b200 import hyrax
    from poly_commit_b200.binding import DEVICE_PTRS
    k = Keys(eng, cname, nv, seed)
    C, dim = k.C, k.dim
    ev, rnd = draws(C, dim * dim, seed + 1), draws(C, dim, seed + 2)
    rows, inf, st = hyrax.commit_resident(k.ck, mont(C, ev), mont(C, rnd))
    exp, _ = ref.commit(C, k.com_key, k.h, ev, rnd)
    assert all(same_point(C, (rows[i], inf[i]), exp[i]) for i in range(dim))
    rows_b, inf_b, _ = hyrax.commit(k.ck, mont(C, ev), mont(C, rnd))
    assert (rows_b == rows).all() and (inf_b == inf).all()
    e_ptr, e_keep = util.dev_ptr(eng, mont(C, ev))
    r_ptr, r_keep = util.dev_ptr(eng, mont(C, rnd))
    rows_d, inf_d, st_d = eng.hyrax_commit(k.ck.srs, nv, e_ptr, r_ptr, flags=DEVICE_PTRS)
    assert (rows_d == rows).all() and (inf_d == inf).all()
    st.release()
    st.release()
    st_d.release()


# ---- open -----------------------------------------------------------------------------------------------------------------
def open_case(eng, cname, nv, count, point=None, zero=False, seed=5):
    """every proof field, lt || r_lt and eval bit-exact against hyrax_ref; eval against an independent fold; the challenge
    callback sees com_eval, com_d, com_b in polynomial order"""
    from poly_commit_b200 import hyrax
    k = Keys(eng, cname, nv, seed)
    C, dim = k.C, k.dim
    point = draws(C, nv, seed + 1) if point is None else point
    polys, states = [], []
    for j in range(count):
        ev = [0] * (dim * dim) if zero else draws(C, dim * dim, seed + 10 + j)
        rnd = draws(C, dim, seed + 20 + j)
        _, _, st = hyrax.commit_resident(k.ck, mont(C, ev), mont(C, rnd))
        polys.append((ev, rnd))
        states.append(st)
    blinds = [draws(C, dim + 3, seed + 30 + j) for j in range(count)]
    log = []
    chal, cs = challenge_fn(C, seed + 40, log)
    proofs = hyrax.open(k.ck, states, mont(C, point), mont(C, [b for bl in blinds for b in bl]), chal)
    _, _, lt, _ = eng.hyrax_open(k.ck.srs, states, mont(C, point), mont(C, [b for bl in blinds for b in bl]), nv=nv)
    assert [e[0] for e in log] == list(range(count))
    for j, ((ev, rnd), p) in enumerate(zip(polys, proofs)):
        mat = ref.flat_to_matrix_column_major(ev, dim, dim)
        exp = ref.open_one(C, k.com_key, k.h, mat, rnd, point, blinds[j], cs[j])
        for key in ("com_eval", "com_d", "com_b"):
            assert same_point(C, p[key], exp[key]), (cname, nv, j, key)
            assert same_point(C, log[j][1 + ("com_eval", "com_d", "com_b").index(key)], exp[key])
        assert (p["z"] == mont(C, exp["z"])).all()
        assert (p["z_d"] == mont(C, [exp["z_d"]])[0]).all() and (p["z_b"] == mont(C, [exp["z_b"]])[0]).all()
        assert (lt[j] == mont(C, exp["lt"] + [exp["r_lt"]])).all()
        assert ints(C, p["eval"]) == [exp["eval"]] == [ref.mle_eval(ev, point, C.r)]
        assert ref.check_one(C, k.com_key, k.h, ref.commit(C, k.com_key, k.h, ev, rnd)[0], point, exp, cs[j])
    for st in states:
        st.release()


# ---- check ----------------------------------------------------------------------------------------------------------------
class Batch:
    """count honest proofs at one point, through the device open"""

    def __init__(self, eng, cname, nv, count, seed=7, zero_row=False):
        from poly_commit_b200 import hyrax
        self.k = k = Keys(eng, cname, nv, seed)
        C, dim = k.C, k.dim
        self.point = draws(C, nv, seed + 1)
        self.row_coms, states = [], []
        for j in range(count):
            ev = draws(C, dim * dim, seed + 10 + j)
            rnd = draws(C, dim, seed + 20 + j)
            if zero_row and j == 0:     # row 0 of T all zero with r_0 = 0: an identity row commitment
                for c in range(dim):
                    ev[c * dim] = 0
                rnd[0] = 0
            rows, inf, st = hyrax.commit_resident(k.ck, mont(C, ev), mont(C, rnd))
            self.row_coms.append((rows, inf))
            states.append(st)
        if zero_row:
            assert self.row_coms[0][1][0] == 1
        blinds = mont(C, draws(C, count * (dim + 3), seed + 30))
        chal, self.cs = challenge_fn(C, seed + 40)
        self.proofs = hyrax.open(k.ck, states, mont(C, self.point), blinds, chal)
        self.ch = mont(C, self.cs[:count])
        for st in states:
            st.release()

    def check(self, row_coms=None, point=None, proofs=None, ch=None):
        from poly_commit_b200 import hyrax
        C = self.k.C
        return list(hyrax.check(self.k.ck, self.row_coms if row_coms is None else row_coms,
                                mont(C, self.point if point is None else point), self.proofs if proofs is None else proofs,
                                self.ch if ch is None else ch))


def check_case(eng, cname, nv, count=3, seed=7):
    """honest proofs are true; each tampering in proof 1 makes only proof 1 false; a tampered point makes every proof false"""
    import copy
    b = Batch(eng, cname, nv, count, seed)
    C, dim = b.k.C, b.k.dim
    assert b.check() == [True] * count
    other = point_bytes(C, C.mul(5, C.g))
    one = mont(C, [1])[0]

    def bump(x):
        return (mont(C, [ints(C, x)[0] + 1])[0]).reshape(np.asarray(x).shape)

    tampers = {
        "com_eval": lambda p: p.update(com_eval=other),
        "com_d": lambda p: p.update(com_d=other),
        "com_b": lambda p: p.update(com_b=other),
        "z[0]": lambda p: p["z"].__setitem__(0, bump(p["z"][0])),
        "z[dim-1]": lambda p: p["z"].__setitem__(dim - 1, bump(p["z"][dim - 1])),
        "z_d": lambda p: p.update(z_d=bump(p["z_d"])),
        "z_b": lambda p: p.update(z_b=bump(p["z_b"])),
    }
    exp = [True] * count
    exp[1] = False
    for name, f in tampers.items():
        proofs = copy.deepcopy(b.proofs)
        f(proofs[1])
        assert b.check(proofs=proofs) == exp, (cname, name)
    rc = [(r.copy(), i.copy()) for r, i in b.row_coms]
    rc[1][0][dim // 2] = other[0]
    assert b.check(row_coms=rc) == exp
    ch = b.ch.copy()
    ch[1] = one if not (ch[1] == one).all() else mont(C, [2])[0]
    assert b.check(ch=ch) == exp
    pt = list(b.point)
    if pt:
        pt[0] = (pt[0] + 1) % C.r
        assert b.check(point=pt) == [False] * count


def identity_row_case(eng, cname, nv=4):
    b = Batch(eng, cname, nv, 2, seed=11, zero_row=True)
    assert b.check() == [True, True]


def bucket_check_case(eng, cname, monkeypatch):
    """PCGPU_MSM_SMALL=0: t_prime through the bucket pipeline one proof at a time gives the same answers"""
    b = Batch(eng, cname, 4, 2, seed=13)
    monkeypatch.setenv("PCGPU_MSM_SMALL", "0")
    assert b.check() == [True, True]
    proofs = [dict(p) for p in b.proofs]
    proofs[0]["com_d"] = proofs[1]["com_d"]
    assert b.check(proofs=proofs) == [False, True]


# ---- errors and handles ---------------------------------------------------------------------------------------------------
def errors_case(eng, pc, cname):
    """odd nv and a key without comb tables: BADARG; a key of the wrong length and a state of another nv: LEN; a state of another
    curve: BADARG; an input not below r: RANGE; *out cleared on failure"""
    from poly_commit_b200 import hyrax
    k = Keys(eng, cname, 2, 17)
    C, dim = k.C, k.dim
    lib, ctx = eng.lib, eng.ctx
    ev, rnd = mont(C, draws(C, 4, 1)), mont(C, draws(C, 2, 2))

    def raw_commit(srs, nv, e, r, flags=0):
        h = ctypes.c_void_p(0x1234)
        out = np.zeros((max(1 << (nv // 2), 1), k.xy.shape[1]), dtype=np.uint64)
        rc = lib.pcgpu_hyrax_commit(ctx, srs.handle, nv, e.ctypes.data, r.ctypes.data, flags, out.ctypes.data, None, ctypes.byref(h))
        return rc, h.value

    assert raw_commit(k.ck.srs, 3, ev, rnd) == (-3, None)                            # InvalidNumberOfVariables
    assert raw_commit(k.ck.srs, 4, mont(C, draws(C, 16, 3)), mont(C, draws(C, 4, 4))) == (-4, None)   # key of dim + 1 != 5
    plain = eng.srs_register(C.id, k.xy)
    assert raw_commit(plain, 2, ev, rnd) == (-3, None)                               # no comb tables
    assert raw_commit(k.ck.srs, 2, ev, rnd, flags=1) == (-3, None)                   # unknown flag
    bad = ev.copy()
    bad[2] = C.fr_to_limbs([0], False)[0]
    r_l = [(C.r >> (64 * j)) & (2**64 - 1) for j in range(4)]
    bad[2] = np.array(r_l, dtype=np.uint64)
    assert raw_commit(k.ck.srs, 2, bad, rnd) == (-5, None)                           # not below r
    with pytest.raises(pc.PcgpuError) as e:
        eng.hyrax_commit(k.ck.srs, 2, ev, np.array([r_l, r_l], dtype=np.uint64))
    assert e.value.code == -5
    _, _, st = hyrax.commit_resident(k.ck, ev, rnd)
    k4 = Keys(eng, cname, 4, 19)
    _, _, st4 = hyrax.commit_resident(k4.ck, mont(C, draws(C, 16, 5)), mont(C, draws(C, 4, 6)))
    blinds = mont(C, draws(C, dim + 3, 7))
    for states, nv, code in (([st4], 2, -4), ([st, st4], 2, -4)):                   # MismatchedNumVars
        with pytest.raises(pc.PcgpuError) as e:
            eng.hyrax_open(k.ck.srs, states, mont(C, draws(C, nv, 8)), np.tile(blinds, (len(states), 1)), nv=nv)
        assert e.value.code == code
    with pytest.raises(pc.PcgpuError) as e:                                          # open with an odd point length
        eng.hyrax_open(k.ck.srs, [st], mont(C, draws(C, 3, 8)), blinds, nv=3)
    assert e.value.code == -3
    with pytest.raises(pc.PcgpuError) as e:                                          # a point element not below r
        eng.hyrax_open(k.ck.srs, [st], np.array([r_l, r_l], dtype=np.uint64), blinds, nv=2)
    assert e.value.code == -5
    other = "pallas" if cname != "pallas" else "bn254"
    ko = Keys(eng, other, 2, 21)
    with pytest.raises(pc.PcgpuError) as e:                                          # a state of another curve
        eng.hyrax_open(ko.ck.srs, [st], mont(C, draws(C, 2, 8)), blinds, nv=2)
    assert e.value.code == -3
    with pytest.raises(pc.PcgpuError) as e:                                          # check with a key of the wrong length
        eng.hyrax_check(k4.ck.srs, 2, 1, k.xy[:2], mont(C, draws(C, 2, 8)), k.xy[:3], mont(C, draws(C, 4, 9)), mont(C, [1]))
    assert e.value.code == -4
    with pytest.raises(pc.PcgpuError) as e:                                          # a challenge not below r
        eng.hyrax_check(k.ck.srs, 2, 1, k.xy[:2], mont(C, draws(C, 2, 8)), k.xy[:3], mont(C, draws(C, 4, 9)),
                        np.array([r_l], dtype=np.uint64))
    assert e.value.code == -5
    st.release()
    st4.release()
    plain.release()


def setup_case(eng, pc, cname):
    """setup's points are the reference's hash-to-curve generators, h the last; BLS12-381 raises"""
    from poly_commit_b200 import hyrax
    C = pyref.Curve(cname)
    if cname == "bls12_381":
        with pytest.raises(ValueError):
            hyrax.setup(eng, C.id, 2)
        return
    with pytest.raises(ValueError):
        hyrax.setup(eng, C.id, 3)
    pp = hyrax.setup(eng, C.id, 2)
    exp = pyref.sample_generators(C, hyrax.PROTOCOL_NAME, 3)
    assert C.points_from_limbs(pp.com_key_xy) == exp[:2] and C.points_from_limbs(pp.h_xy) == [exp[2]]
    ck, vk = hyrax.trim(eng, pp)
    assert ck is vk and ck.dim == 2


# ---- host emulation --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cname", CURVES)
@pytest.mark.parametrize("nv", [0, 2, 4, 6])
def test_emul_hyrax_commit(emul, cname, nv):
    commit_case(emul, cname, nv)


@pytest.mark.parametrize("cname", CURVES)
def test_emul_hyrax_open(emul, cname):
    open_case(emul, cname, 4, 1)
    open_case(emul, cname, 2, 3)
    open_case(emul, cname, 0, 1)


def test_emul_hyrax_open_edges(emul):
    C = pyref.Curve("bn254")
    open_case(emul, "bn254", 4, 1, point=[0, 1, 1, 0])
    open_case(emul, "bn254", 4, 3, point=[1, 0, 0, 1], zero=True)
    open_case(emul, "pallas", 4, 1, point=[0, 0, 0, 0], zero=True)
    assert C.r > 1


@pytest.mark.parametrize("cname", CURVES)
def test_emul_hyrax_check(emul, cname):
    check_case(emul, cname, 4)


def test_emul_hyrax_check_nv0_and_identity_row(emul):
    check_case(emul, "bn254", 0, count=2)
    identity_row_case(emul, "pallas")


def test_emul_hyrax_check_bucket_path(emul, monkeypatch):
    bucket_check_case(emul, "bn254", monkeypatch)


@pytest.mark.parametrize("cname", CURVES)
def test_emul_hyrax_errors(emul, pc, cname):
    errors_case(emul, pc, cname)
    setup_case(emul, pc, cname)


def test_emul_row_mul_split_path(emul):
    """a tall matrix takes the row product's split path (row_mul_plan: 8 spans of 32 rows) and matches the oracle"""
    cname = "bn254"
    C = pyref.Curve(cname)
    for rows, cols in ((256, 3), (255, 2), (2048, 1)):
        v, m = util.rand_fr(cname, rows, 1, True), util.rand_fr(cname, rows * cols, 2, True)
        assert (emul.fr_row_mul(C.id, v, m, rows, cols) == orc.fr_row_mul(C.id, v, m, rows, cols)).all()


# ---- H100 -------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cname", CURVES)
def test_gpu_hyrax_small(gpu_engine, pc, cname, monkeypatch):
    for nv in (0, 2, 4, 6):
        commit_case(gpu_engine, cname, nv)
    open_case(gpu_engine, cname, 4, 3)
    open_case(gpu_engine, cname, 4, 1, point=[0, 1, 1, 0], zero=True)
    check_case(gpu_engine, cname, 4)
    identity_row_case(gpu_engine, cname)
    errors_case(gpu_engine, pc, cname)
    setup_case(gpu_engine, pc, cname)
    bucket_check_case(gpu_engine, cname, monkeypatch)


def at_size_case(eng, cname, nv, count, seed=31):
    """commit + open + check at full size; proof fields against the C oracle"""
    from poly_commit_b200 import hyrax
    C = pyref.Curve(cname)
    dim = 1 << (nv // 2)
    xy = util.random_points(cname, dim + 1, seed)
    ck = hyrax.CommitterKey(eng, C.id, xy[:dim], xy[dim])
    point_c = util.rand_fr(cname, nv, seed + 1, False)
    point = util.rand_fr(cname, nv, seed + 1, True)
    evs = [util.rand_fr_fast(cname, dim * dim, seed + 10 + j) for j in range(count)]
    rnds = [util.rand_fr(cname, dim, seed + 20 + j, True) for j in range(count)]
    commits = [hyrax.commit_resident(ck, e, r) for e, r in zip(evs, rnds)]
    blinds = util.rand_fr(cname, count * (dim + 3), seed + 30, True)
    ch = util.rand_fr(cname, count, seed + 40, True)
    proofs = hyrax.open(ck, [c[2] for c in commits], point, blinds, lambda j, *pts: ch[j])
    _, _, lt, _ = eng.hyrax_open(ck.srs, [c[2] for c in commits], point, blinds, nv=nv)
    l_c, _ = ref.tensors([int(x) for x in C.fr_from_limbs(point_c, False)], C.r)
    l_m = mont(C, l_c)
    canon = lambda a: orc.field_unop("orc_fr_from_mont", C.id, np.ascontiguousarray(a, dtype=np.uint64).reshape(-1, 4))
    bl = blinds.reshape(count, dim + 3, 4)
    for j in range(count):
        mat = hyrax.flat_to_matrix_column_major(evs[j], dim, dim)
        block = np.concatenate([mat, rnds[j].reshape(dim, 1, 4)], axis=1).reshape(-1, 4)
        assert (lt[j] == orc.fr_row_mul(C.id, l_m, block, dim, dim + 1)).all()
        for row in (0, dim // 2, dim - 1):                                           # row commitments
            exp = orc.msm(C.id, xy, canon(block.reshape(dim, dim + 1, 4)[row]))
            assert (commits[j][0][row] == exp[0]).all()
        exp_d = orc.msm(C.id, xy, canon(bl[j, 1:dim + 2]))                           # com_d = [d | r_d]
        assert (proofs[j]["com_d"][0] == exp_d[0]).all()
    ok = hyrax.check(ck, [(c[0], c[1]) for c in commits], point, proofs, ch)
    assert list(ok) == [True] * count
    proofs[count - 1]["z"][0] = proofs[count - 1]["z"][1]
    assert list(hyrax.check(ck, [(c[0], c[1]) for c in commits], point, proofs, ch)) == [True] * (count - 1) + [False]
    for c in commits:
        c[2].release()


@pytest.mark.gpu
def test_gpu_hyrax_cfg4(gpu_engine):
    at_size_case(gpu_engine, "bn254", 22, 2)


@pytest.mark.gpu
@pytest.mark.parametrize("cname", ["bls12_381", "pallas"])
def test_gpu_hyrax_nv20(gpu_engine, cname):
    at_size_case(gpu_engine, cname, 20, 1)


@pytest.mark.gpu
def test_gpu_hyrax_device_ptrs(gpu_engine):
    """commit, open and check with every PCGPU_DEVICE_PTRS argument on the device give the host path's results"""
    from poly_commit_b200 import hyrax
    from poly_commit_b200.binding import DEVICE_PTRS
    eng, cname, nv, count = gpu_engine, "bn254", 8, 2
    k = Keys(eng, cname, nv, 41)
    C, dim = k.C, k.dim
    evs = [util.rand_fr(cname, dim * dim, 50 + j, True) for j in range(count)]
    rnds = [util.rand_fr(cname, dim, 60 + j, True) for j in range(count)]
    host = [hyrax.commit_resident(k.ck, e, r) for e, r in zip(evs, rnds)]
    keep, dev = [], []
    for e, r in zip(evs, rnds):
        (ep, eo), (rp, ro) = util.dev_ptr(eng, e), util.dev_ptr(eng, r)
        keep += [eo, ro]
        dev.append(eng.hyrax_commit(k.ck.srs, nv, ep, rp, flags=DEVICE_PTRS))
    for h, d in zip(host, dev):
        assert (h[0] == d[0]).all() and (h[1] == d[1]).all()
    point = util.rand_fr(cname, nv, 70, True)
    blinds = util.rand_fr(cname, count * (dim + 3), 71, True)
    ch = util.rand_fr(cname, count, 72, True)
    coms, inf, lt, ev = eng.hyrax_open(k.ck.srs, [d[2] for d in dev], point, blinds, nv=nv)
    bp, bo = util.dev_ptr(eng, blinds)
    lt_buf = eng.buffer(count * (dim + 1))
    coms_d, inf_d, _, ev_d = eng.hyrax_open(k.ck.srs, [d[2] for d in dev], point, bp, nv=nv, flags=DEVICE_PTRS, out_lt=lt_buf.ptr())
    assert (coms == coms_d).all() and (inf == inf_d).all() and (ev == ev_d).all()
    assert (lt_buf.read().reshape(lt.shape) == lt).all()
    proofs = hyrax.open(k.ck, [d[2] for d in dev], point, blinds, lambda j, *pts: ch[j])
    rc_xy = np.concatenate([d[0] for d in dev])
    rc_inf = np.concatenate([d[1] for d in dev])
    zs = np.concatenate([np.concatenate([p["z"], p["z_d"].reshape(1, 4), p["z_b"].reshape(1, 4)]) for p in proofs])
    pxy = np.array([[p[key][0] for key in ("com_eval", "com_d", "com_b")] for p in proofs], dtype=np.uint64).reshape(-1, rc_xy.shape[1])
    (xp, xo), (ip, io), (zp, zo) = util.dev_ptr(eng, rc_xy), util.dev_ptr(eng, rc_inf), util.dev_ptr(eng, zs)
    ok = eng.hyrax_check(k.ck.srs, nv, count, xp, point, pxy, zp, ch, row_coms_inf=ip, flags=DEVICE_PTRS)
    assert list(ok) == [True] * count
    for d in dev + host:
        d[2].release()
    lt_buf.release()


@pytest.mark.gpu
def test_gpu_hyrax_check_64(gpu_engine):
    """64 proofs in one check, every 7th tampered; the same batch nine times over in one call"""
    b = Batch(gpu_engine, "bn254", 8, 64, seed=43)
    proofs = [dict(p) for p in b.proofs]
    for j in range(0, 64, 7):
        proofs[j]["z_b"] = proofs[(j + 1) % 64]["z_b"]
    assert b.check(proofs=proofs) == [j % 7 != 0 for j in range(64)]
    # 576 proofs: 1152 small-MSM problems, more than one launch takes (SMALL_MAX_PROB = 1024)
    reps = 9
    got = b.check(row_coms=b.row_coms * reps, proofs=proofs * reps, ch=np.tile(b.ch, (reps, 1)))
    assert got == [j % 7 != 0 for j in range(64)] * reps


@pytest.mark.gpu
def test_gpu_row_mul_split_cfg4(gpu_engine):
    """pcgpu_fr_row_mul at the cfg4 shape (2^11 rows x (2^11 + 1) columns: the split path) against the oracle"""
    cname = "bn254"
    C = pyref.Curve(cname)
    rows, cols = 2048, 2049
    v, m = util.rand_fr(cname, rows, 81, True), util.rand_fr_fast(cname, rows * cols, 82)
    assert (gpu_engine.fr_row_mul(C.id, v, m, rows, cols) == orc.fr_row_mul(C.id, v, m, rows, cols)).all()
