"""The handles that outlive a call -- pcgpu_srs, pcgpu_mlpc, pcgpu_brakedown, pcgpu_ipa -- and the Python objects that own them
(poly_commit_b200/binding.py _Handle):
  * every creator sets *out to NULL whenever out is non-null, whatever it returns: on a null context, on an argument check
    and on a failure after the handle was allocated; the context then serves a good register and its MSM, open or encode,
    bit-exact against the oracle;
  * an IPA state belongs to the context that began it: round_lr, round_fold and finish through another context are
    PCGPU_E_BADARG and leave the open intact; opens on two contexts, interleaved round by round, are independent;
  * every Python handle can be released twice, and released or collected after Engine.close(); the IPA calls refuse a curve
    other than the state's.
The same case bodies run on the host-emulated library (CPU) and, with `-m gpu`, on libpcgpu.so."""
import ctypes
import gc
from itertools import zip_longest

import numpy as np
import pytest

from oracle import orc, pyref
from tests import util
from tests import test_multilinear_pc as mlpc_cases
from tests.test_brakedown import _lc, bref, params_for
from tests.test_hostcheck import oracle_ipa_rounds
from tests.test_ipa_paths import compare_open, open_inputs

E_BADARG = -3
SENTINEL = 0x5E471E1
_vp = ctypes.c_void_p


def _p(a):
    return None if a is None else a.ctypes.data_as(_vp)


def expect_refused(cases):
    """every call(out) returns PCGPU_E_BADARG and leaves NULL in *out, which held a sentinel"""
    for what, call in cases:
        out = _vp(SENTINEL)
        rc = call(ctypes.byref(out))
        assert rc == E_BADARG and out.value is None, (what, rc, out.value)


# ---------------------------------------------------------------------------------------------------------------------------
# creators
# ---------------------------------------------------------------------------------------------------------------------------
def srs_case(eng, pc, cname):
    C = pyref.Curve(cname)
    lib, g2 = eng.lib, pc.binding.G2_OF[C.id]
    g2_bases = np.zeros((4, pc.binding.affine_limbs(g2)), dtype=np.uint64)
    expect_refused([
        ("null context", lambda out: lib.pcgpu_srs_register(None, C.id, _p(g2_bases), None, 4, 0, out)),
        ("null bases", lambda out: lib.pcgpu_srs_register(eng.ctx, C.id, None, None, 4, 0, out)),
        ("G2 key with PRECOMPUTE", lambda out: lib.pcgpu_srs_register(eng.ctx, g2, _p(g2_bases), None, 4, pc.SRS_PRECOMPUTE, out)),
    ])
    bases = util.random_points(cname, 40, seed=1)
    scalars = util.rand_fr(cname, 40, seed=2, mont=False)
    srs = eng.srs_register(C.id, bases)
    got = eng.msm(srs, scalars)
    srs.release()
    exp = orc.msm(C.id, bases, scalars)
    assert got[1] == exp[1] and (got[0] == exp[0]).all()


def mlpc_case(eng, pc, cname):
    C = pyref.Curve(cname)
    lib = eng.lib
    level = np.zeros((4, pc.binding.affine_limbs(pc.binding.G2_OF[C.id])), dtype=np.uint64)
    levels = (_vp * 2)(_p(level), None)
    expect_refused([
        ("null context", lambda out: lib.pcgpu_mlpc_register(None, C.id, 2, levels, None, 0, out)),
        ("nv = 0", lambda out: lib.pcgpu_mlpc_register(eng.ctx, C.id, 0, levels, None, 0, out)),
        ("null level", lambda out: lib.pcgpu_mlpc_register(eng.ctx, C.id, 2, levels, None, 0, out)),
    ])
    mlpc_cases.open_case(eng, pc, cname, 3, seed=40)     # register + open against the reference


def brakedown_case(eng, pc, cname):
    C = pyref.Curve(cname)
    p = params_for(cname, 128)                             # one level
    lib, L = eng.lib, len(p["a_dims"])
    mats = [[np.ascontiguousarray(x, dtype=np.uint64) for x in mat] for mat in p["a_mats"] + p["b_mats"]]
    ad = np.ascontiguousarray(np.asarray(p["a_dims"], dtype=np.uint64).reshape(-1))
    bd = np.ascontiguousarray(np.asarray(p["b_dims"], dtype=np.uint64).reshape(-1))
    P, Cc, V = ((_vp * (2 * L))(*[_p(x[k]) for x in mats]) for k in range(3))
    reg = lambda ctx, m: lambda out: lib.pcgpu_brakedown_register(ctx, C.id, m, p["m_ext"], L, _p(ad), _p(bd), P, Cc, V, 0, out)  # noqa: E731
    expect_refused([
        ("null context", reg(None, p["m"])),
        ("m = 0", reg(eng.ctx, 0)),
        ("a_dims[0] != m", reg(eng.ctx, p["m"] + 1)),
    ])
    code = _lc().brakedown_register(eng, p)
    mat = util.rand_fr_fast(cname, 3 * p["m"], seed=41).reshape(3, p["m"], 4)
    got = eng.brakedown_encode(code, mat)
    code.release()
    assert (got == bref.c_encode(mat, p, C.r)).all()


def ipa_rounds(eng, cname, st, h_prime, chal):
    """ipa_pc.open_rounds one round at a time: yields None after each round, then the open's result"""
    from poly_commit_b200 import ipa_pc
    C = pyref.Curve(cname)
    got = dict(l_vec=[], r_vec=[], challenges=[])
    while eng.ipa_len(st) > 1:
        l, li, r, ri = eng.ipa_round_lr(C.id, st, h_prime, with_inf=True)
        got["l_vec"].append(l)
        got["r_vec"].append(r)
        chal = ipa_pc.compute_random_oracle_challenge(C.id, ipa_pc.round_transcript(eng, C.id, chal, l, li, r, ri))
        got["challenges"].append(chal)
        eng.ipa_round_fold(st, ipa_pc._fr_mont(C.id, chal), ipa_pc._fr_mont(C.id, pow(chal, -1, C.r)))
        yield None
    got["final_comm_key"], got["c"] = eng.ipa_finish(C.id, st)
    yield got


def run_opens(*opens):
    """runs (eng, cname, st, h_prime, chal) opens interleaved round by round -> their results"""
    gens = [ipa_rounds(*o) for o in opens]
    last = [None] * len(gens)
    for step in zip_longest(*gens):
        last = [s if s is not None else x for s, x in zip(step, last)]
    return last


def ipa_case(eng, pc, cname):
    C = pyref.Curve(cname)
    lib = eng.lib
    key, co, z, h_prime = open_inputs(cname, 5, "rand", "rand", "rand", seed=50)
    st = eng.ipa_begin(C.id, key, co, z)
    begin = lambda ctx, n: lambda out: lib.pcgpu_ipa_begin(ctx, C.id, _p(key), n, _p(co), co.shape[0] if n == 32 else 0, _p(z), 0, out)  # noqa: E731
    expect_refused([
        ("null context", begin(None, 32)),
        ("n not a power of two", begin(eng.ctx, 3)),
        ("a second open on the context", begin(eng.ctx, 32)),
    ])
    compare_open(run_opens((eng, cname, st, h_prime, 7))[0], oracle_ipa_rounds(cname, key, co, z, h_prime, 7), "first open")


def ipa_context_case(a, b, pc, cname):
    """an open begun on a: b's round_lr, round_fold and finish are refused and change nothing; then opens on a and b at once"""
    from poly_commit_b200 import ipa_pc
    C = pyref.Curve(cname)
    key, co, z, h_prime = open_inputs(cname, 6, "rand", "rand", "rand", seed=60)
    st = a.ipa_begin(C.id, key, co, z)
    one = ipa_pc._fr_mont(C.id, 1)
    for call in (lambda: b.ipa_round_lr(C.id, st, h_prime), lambda: b.ipa_round_fold(st, one, one),
                 lambda: b.ipa_finish(C.id, st)):
        with pytest.raises(pc.PcgpuError) as e:
            call()
        assert e.value.code == E_BADARG
    assert st.handle is not None and a.ipa_len(st) == 64
    compare_open(run_opens((a, cname, st, h_prime, 8))[0], oracle_ipa_rounds(cname, key, co, z, h_prime, 8), "open on a")
    key2, co2, z2, h2 = open_inputs(cname, 5, "n-3", "rand", "dupneg", seed=70)
    sa, sb = a.ipa_begin(C.id, key, co, z), b.ipa_begin(C.id, key2, co2, z2)   # a's next open, and one on b
    got_a, got_b = run_opens((a, cname, sa, h_prime, 9), (b, cname, sb, h2, 10))
    compare_open(got_a, oracle_ipa_rounds(cname, key, co, z, h_prime, 9), "interleaved on a")
    compare_open(got_b, oracle_ipa_rounds(cname, key2, co2, z2, h2, 10), "interleaved on b")


# ---------------------------------------------------------------------------------------------------------------------------
# Python handles
# ---------------------------------------------------------------------------------------------------------------------------
def make_handles(eng, pc):
    """one object of each of the five handle kinds on eng"""
    C = pyref.Curve("bn254")
    key, co, z, _ = open_inputs("bn254", 3, "rand", "rand", "rand", seed=80)
    _, levels, _ = mlpc_cases.make_key(eng, pc, "bn254", 2, "random", 81)
    return [eng.srs_register(C.id, key), eng.mlpc_register(C.id, levels), _lc().brakedown_register(eng, params_for("bn254", 16)),
            eng.buffer(4), eng.ipa_begin(C.id, key, co, z)]


def python_handles_case(new_engine, pc):
    eng = new_engine()
    hs = make_handles(eng, pc)
    assert [type(h).__name__ for h in hs] == ["Srs", "MlpcKey", "BrakedownCode", "DeviceBuffer", "IpaState"]
    st = hs[-1]
    h_prime = util.random_points("bn254", 1, seed=82)[0]
    for call in (lambda: eng.ipa_round_lr(pc.PALLAS, st, h_prime), lambda: eng.ipa_finish(pc.BLS12_381, st)):
        with pytest.raises(ValueError):
            call()
    assert st.handle is not None and eng.ipa_len(st) == 8
    for h in hs:
        h.release()
        h.release()
    hs = make_handles(eng, pc)         # the released IPA state let the context begin again
    eng.close()
    for h in hs:
        h.release()
        h.release()
    eng = new_engine()
    hs = make_handles(eng, pc)
    eng.close()
    del hs
    gc.collect()


# ---------------------------------------------------------------------------------------------------------------------------
# the host-emulated library
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def emul_engines(pc, hostcheck_path, oracle):
    engs = []

    def new():
        engs.append(pc.Engine(0, lib_path=hostcheck_path))
        return engs[-1]
    yield new
    for e in engs:
        e.close()


def test_emul_creators(emul_engines, pc):
    eng = emul_engines()
    srs_case(eng, pc, "bn254")
    mlpc_case(eng, pc, "bls12_381")
    brakedown_case(eng, pc, "pallas")
    ipa_case(eng, pc, "pallas")


def test_emul_ipa_context(emul_engines, pc):
    ipa_context_case(emul_engines(), emul_engines(), pc, "bn254")


def test_emul_python_handles(emul_engines, pc):
    python_handles_case(emul_engines, pc)


# ---------------------------------------------------------------------------------------------------------------------------
# the device
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def gpu_engines(pc, oracle):
    engs = []

    def new():
        engs.append(pc.Engine(0))
        return engs[-1]
    yield new
    for e in engs:
        e.close()


@pytest.mark.gpu
def test_gpu_creators(gpu_engines, pc):
    eng = gpu_engines()
    srs_case(eng, pc, "bls12_381")
    mlpc_case(eng, pc, "bn254")
    brakedown_case(eng, pc, "bn254")
    ipa_case(eng, pc, "bls12_381")


@pytest.mark.gpu
def test_gpu_ipa_context(gpu_engines, pc):
    ipa_context_case(gpu_engines(), gpu_engines(), pc, "pallas")


@pytest.mark.gpu
def test_gpu_python_handles(gpu_engines, pc):
    python_handles_case(gpu_engines, pc)
