"""The bucket pipeline's paths on an H100 at the sizes where they are taken, against the C oracle (bit-exact).  Every case
states the path it covers and asserts it from Engine.msm_last_geometry (tests/msm_cases.py restates the policy), so a change
of the window picker or of the pair kernel's occupancy that moves a case off its path fails the case instead of silently
dropping the coverage.

  * the default policy (no knobs) for all three curves up to 2^20 terms, raw bases and window-folded tables, uniform and
    skewed Montgomery scalars -- the 2^20 rows must run batched-affine pair rounds;
  * forced pair rounds at 2^17 + 1 with a full and a 1/16 wave of pair threads (chains of several hundred slots per thread);
  * exceptional pairs (P + P, P + (-P), identity operands) at every chain position, and an exact sum of zero;
  * more heavy buckets than the heavy-bucket kernel's grid; the two-level reduction (c = 18, 19); batch mode (pair kernels
    at half a wave on sibling streams).
"""
import numpy as np
import pytest

from oracle import orc, pyref
from tests import msm_cases, util
from tests.test_gpu_parity import gpu_srs

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng(gpu_engine):
    return gpu_engine


def _mixture(cname, n, seed):
    """the randomised sweep's scalar mixture (zeros, 1, r-1, 16-bit values, uniform), canonical"""
    C = pyref.Curve(cname)
    sc = util.rand_fr(cname, n, seed=seed, mont=False)
    kind = util.rng(seed + 1).integers(0, 8, size=n)
    sc[kind == 0] = 0
    sc[kind == 1] = C.fr_to_limbs([1], False)[0]
    sc[kind == 2] = C.fr_to_limbs([C.r - 1], False)[0]
    small = kind == 3
    sc[small, 1:] = 0
    sc[small, 0] &= np.uint64(0xFFFF)
    return sc


DEFAULT_ROWS = [("bn254", (1 << 16) + 3), ("bn254", (1 << 18) + 1), ("bn254", (1 << 20) + 1),
                ("pallas", (1 << 16) + 3), ("pallas", (1 << 18) + 1), ("pallas", (1 << 20) + 1),
                ("bls12_381", (1 << 18) + 1)]


@pytest.mark.parametrize("cname,n", DEFAULT_ROWS)
def test_default_policy(eng, pc, cname, n, monkeypatch):
    """no knobs: the geometry the picker chooses, raw and folded, uniform canonical and skewed Montgomery scalars"""
    for k in ("PCGPU_MSM_SMALL", "PCGPU_MSM_C", "PCGPU_SRS_C", "PCGPU_MSM_AFFINE_ROUNDS", "PCGPU_MSM_AFFINE_TDIV", "PCGPU_MSM_L"):
        monkeypatch.delenv(k, raising=False)
    C = pyref.Curve(cname)
    bases = gpu_srs(eng, cname, n, seed=n % 97)
    uni = util.rand_fr(cname, n, seed=600 + n % 97, mont=False)
    mix = _mixture(cname, n, seed=700 + n % 97)
    exp = [orc.msm(C.id, bases, uni), orc.msm(C.id, bases, mix)]
    mix_m = orc.field_unop("orc_fr_to_mont", C.id, mix)
    for fold in (False, True):
        srs = eng.srs_register(C.id, bases, flags=pc.SRS_PRECOMPUTE if fold else 0)
        for (sc, flags), e in zip(((uni, 0), (mix_m, pc.SCALARS_MONT)), exp):
            got = eng.msm(srs, sc, flags=flags)
            g = msm_cases.check_geometry(eng, pc, cname, n, folded_c=msm_cases.srs_precompute_window(n) if fold else None,
                                         depth=n > (1 << 20))
            print(f"geometry {cname} n={n} {'folded' if fold else 'raw'} flags={flags}: {g}")
            assert got[1] == e[1] and (got[0] == e[0]).all(), (cname, n, fold, flags)
            assert g["heavy"] is not None
        srs.release()


@pytest.mark.parametrize("cname", util.CURVE_NAMES)
def test_forced_depth(eng, pc, cname, monkeypatch):
    """PCGPU_MSM_AFFINE_ROUNDS 1 / 3 / 5 x PCGPU_MSM_AFFINE_TDIV 1 / 16 at 2^17 + 1 terms, raw bases and folded tables (c = 14)"""
    n = (1 << 17) + 1
    assert msm_cases.srs_precompute_window(n) == 14
    msm_cases.forced_depth_case(eng, pc, cname, gpu_srs(eng, cname, n, seed=31), monkeypatch, seed=610)


@pytest.mark.parametrize("cname", util.CURVE_NAMES)
@pytest.mark.parametrize("rounds,tdiv", [(3, 16), (None, None)])
def test_exceptional_pairs_at_depth(eng, pc, cname, rounds, tdiv, monkeypatch):
    """2^17 bases drawn from 40 points and their negations, 1/64 identities, scalars from {1, r-1, 2, ...}: forced R = 3 with
    a 1/16 wave, and the default policy; plain and with an exact sum of zero"""
    msm_cases.exceptional_case(eng, pc, cname, 1 << 17, monkeypatch, rounds=rounds, tdiv=tdiv, seed=620)


@pytest.mark.parametrize("cname", ["bn254", "bls12_381"])
def test_heavy_buckets_past_the_grid_stride(eng, pc, cname, monkeypatch):
    """2^17 + 1 terms whose scalars take 128 distinct values: thousands of heavy buckets for 64 heavy-bucket blocks"""
    n = (1 << 17) + 1
    msm_cases.heavy_case(eng, pc, cname, gpu_srs(eng, cname, n, seed=32), 128, monkeypatch, seed=630)


@pytest.mark.parametrize("cname", ["bn254", "pallas"])
@pytest.mark.parametrize("c", [18, 19])
def test_two_level_reduction(eng, pc, cname, c, monkeypatch):
    """c = 18 / 19 (row / column bucket reduction) at 2^18 terms, raw bases (PCGPU_MSM_C) and folded tables (PCGPU_SRS_C)"""
    monkeypatch.setenv("PCGPU_MSM_C", str(c))
    monkeypatch.setenv("PCGPU_SRS_C", str(c))
    n = 1 << 18
    C = pyref.Curve(cname)
    bases = gpu_srs(eng, cname, n, seed=33)
    sc = util.rand_fr(cname, n, seed=640 + c, mont=False)
    sc[5] = C.fr_to_limbs([C.r - 1], False)[0]
    sc[7] = C.fr_to_limbs([1 << (c - 1)], False)[0]
    exp = orc.msm(C.id, bases, sc)
    for fold in (False, True):
        srs = eng.srs_register(C.id, bases, flags=pc.SRS_PRECOMPUTE if fold else 0)
        got = eng.msm(srs, sc)
        msm_cases.check_geometry(eng, pc, cname, n, folded_c=c if fold else None)
        assert got[1] == exp[1] and (got[0] == exp[0]).all(), (cname, c, fold)
        srs.release()


@pytest.mark.parametrize("cname", ["bn254", "pallas"])
def test_batch_mode(eng, pc, cname, monkeypatch):
    """kzg_commit_batch (four polynomials in flight) and kzg_commit_open_batch (two commit / open pairs in flight, pair kernels
    at half a wave: tdiv = 2) for 5 polynomials of 2^18 + 1 coefficients, each against the oracle's commit and open"""
    for k in ("PCGPU_MSM_AFFINE_ROUNDS", "PCGPU_MSM_AFFINE_TDIV", "PCGPU_BATCH_TDIV", "PCGPU_COMMIT_OPEN_WAYS"):
        monkeypatch.delenv(k, raising=False)
    C = pyref.Curve(cname)
    n = (1 << 18) + 1
    bases = gpu_srs(eng, cname, n, seed=34)
    srs = eng.srs_register(C.id, bases, flags=pc.SRS_PRECOMPUTE)
    polys = [util.rand_fr_fast(cname, n, seed=650 + i) for i in range(5)]
    z = util.rand_fr(cname, 1, seed=656, mont=True)[0]
    exp = []
    for p in polys:
        rc, cxy, cinf = orc.kzg_commit(C.id, bases, p)
        rc2, wxy, winf, _ = orc.kzg_open(C.id, bases, p, z)
        assert rc == 0 and rc2 == 0
        exp.append((cxy, cinf, wxy, winf))
    got, inf = eng.kzg_commit_batch(srs, polys)
    for i, e in enumerate(exp):
        assert (got[i] == e[0]).all() and inf[i] == e[1], i
    c, ci, w, wi = eng.kzg_commit_open_batch(srs, polys, z)
    g = msm_cases.check_geometry(eng, pc, cname, n, folded_c=msm_cases.srs_precompute_window(n), tdiv=2)
    assert g["R"] >= 1, g            # the half-wave pair kernels actually ran
    for i, e in enumerate(exp):
        assert (c[i] == e[0]).all() and ci[i] == e[1] and (w[i] == e[2]).all() and wi[i] == e[3], i
    srs.release()
