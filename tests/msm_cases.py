"""MSM case bodies shared by the host-emulation tests (test_hostcheck.py, small n) and the device tests (test_gpu_msm_paths.py,
sizes where the pair rounds run at depth on an H100), plus the restatement of the library's path policy that every case
asserts through Engine.msm_last_geometry: a case whose geometry differs from the one it claims to cover fails, so coverage
cannot silently move to another path when the picker or the pair kernel's occupancy changes.

The policy restated here (csrc/msm.cuh msm_pick_c / msm_geometry, csrc/srs.cuh srs_precompute_window, csrc/impl.cuh
msm_device_planes, msm_run):
  * window-folded tables (SRS_PRECOMPUTE, n >= 4096): c = the registration's window, G = W table groups, one bucket set;
  * raw bases: c = clamp(floor(log2 n) - 4, 8, 16) or PCGPU_MSM_C, G = 1, S = W bucket sets;
  * W = ceil(bits(r) / c); entries = n * W; buckets TB = S * 2^(c-1);
  * affine rounds R: add one while R < 8, (entries / TB) >> R >= 4 and entries >> (R + 1) >= 16 * wave, where wave is one
    resident wave of the pair kernel; PCGPU_MSM_AFFINE_ROUNDS overrides;
  * pair threads T = wave, or with a divisor tdiv > 1 (batch mode, PCGPU_MSM_AFFINE_TDIV) ceil(wave / tdiv / 128) * 128.
"""
import os

import numpy as np

from oracle import orc, pyref
from tests import util

SRS_PRECOMPUTE_MIN_N = 1 << 12
HEAVY_BUCKET_TASKS = 8          # csrc/msm.cuh: a bucket with more accumulate tasks than this goes to MsmHeavyBucketBody
HEAVY_GRID = 64                 # blocks of MsmHeavyBucketBody (grid-strided over the heavy list)
DEPTH_SLOTS = 32                # a "depth" case gives every pair-round thread at least this many round-0 slots


def on_gpu(eng):
    return os.path.basename(eng.lib._name) != "libpcgpu_hostcheck.so"


def msm_pick_c(n):
    return min(16, max(8, max(n, 1).bit_length() - 1 - 4))


def srs_precompute_window(n):
    if os.environ.get("PCGPU_SRS_C"):
        return int(os.environ["PCGPU_SRS_C"])
    lg = max(n, 1).bit_length() - 1
    return 17 if lg >= 18 else 14 if lg >= 15 else 12


def policy_rounds(entries, tb, wave):
    avg, r = entries // tb, 0
    while r < 8 and (avg >> r) >= 4 and (entries >> (r + 1)) >= 16 * wave:
        r += 1
    return r


def pair_threads(wave, tdiv):
    t = min(wave, 1 << 20)
    return t if tdiv == 1 else (t // tdiv + 127) // 128 * 128


def check_geometry(eng, pc, cname, n, folded_c=None, tdiv=1, depth=False):
    """asserts that the last MSM on `eng` took the bucket pipeline with the documented geometry for n terms.  folded_c: the
    window the SRS_PRECOMPUTE tables were registered with (None: raw bases).  tdiv: the pair-round divisor expected without
    a PCGPU_MSM_AFFINE_TDIV knob.  depth: the pair rounds must run and give every thread >= DEPTH_SLOTS round-0 slots."""
    g = eng.msm_last_geometry()
    bits = pyref.Curve(cname).r.bit_length()
    assert g["path"] == pc.binding.MSM_PATH_BUCKETS and g["n"] == n, g
    if folded_c is not None and n >= SRS_PRECOMPUTE_MIN_N:
        c = folded_c
        G = -(-bits // c)
    else:
        c = int(os.environ.get("PCGPU_MSM_C") or msm_pick_c(n))
        G = 1
    W = -(-bits // c)
    assert (g["c"], g["W"], g["G"]) == (c, W, G), g
    entries = n * W
    assert g["entries"] == entries, g
    S = -(-W // G)
    knob = os.environ.get("PCGPU_MSM_AFFINE_ROUNDS")
    R = int(knob) if knob else policy_rounds(entries, S << (c - 1), g["wave"])
    assert g["R"] == R, (g, R)
    if R:
        td = int(os.environ.get("PCGPU_MSM_AFFINE_TDIV") or tdiv)
        assert (g["T"], g["tdiv"]) == (pair_threads(g["wave"], td), td), g
    else:
        assert g["T"] == 0, g
    if depth:
        assert R >= 1 and entries // (2 * g["T"]) >= DEPTH_SLOTS, g
    return g


def _assert_point(got, exp, what):
    assert got[1] == exp[1] and (got[0] == exp[0]).all(), what


def forced_depth_case(eng, pc, cname, bases, monkeypatch, rounds=(1, 3, 5), tdivs=(1, 16), folded=(False, True), seed=1):
    """uniform scalars through forced pair rounds: every (rounds, tdiv, raw / folded) combination against one oracle MSM.
    With tdiv = 16 each thread walks a chain of many slots, and the slot count differs by one between threads."""
    C = pyref.Curve(cname)
    n = bases.shape[0]
    sc = util.rand_fr(cname, n, seed=seed, mont=False)
    exp = orc.msm(C.id, bases, sc)
    monkeypatch.setenv("PCGPU_MSM_SMALL", "0")
    for fold in folded:
        srs = eng.srs_register(C.id, bases, flags=pc.SRS_PRECOMPUTE if fold else 0)
        for r in rounds:
            for td in tdivs:
                monkeypatch.setenv("PCGPU_MSM_AFFINE_ROUNDS", str(r))
                monkeypatch.setenv("PCGPU_MSM_AFFINE_TDIV", str(td))
                got = eng.msm(srs, sc)
                check_geometry(eng, pc, cname, n, folded_c=srs_precompute_window(n) if fold else None,
                               depth=td > 1 or not on_gpu(eng))
                _assert_point(got, exp, (cname, n, fold, r, td))
        srs.release()


def exceptional_inputs(cname, n, seed, identity=False):
    """n bases drawn from a few dozen distinct points and their negations, about 1/64 of them identity (inf flag), with
    scalars from a small set (1, r-1, 2, ...): every bucket holds copies of the same points, so each pair round meets P + P,
    P + (-P) and identity operands at every chain position.  identity=True: the second half repeats the first with negated
    bases and the same scalars, so the exact sum is the identity."""
    C = pyref.Curve(cname)
    k = 40
    pts = util.random_points(cname, k, seed=seed)
    neg = C.points_to_limbs([C.neg(p) for p in C.points_from_limbs(pts)])[0]
    pool = np.concatenate([pts, neg])
    g = util.rng(seed)
    m = n // 2 if identity else n
    idx = g.integers(0, 2 * k, size=m)
    inf = (g.integers(0, 64, size=m) == 0).astype(np.uint8)
    vals = C.fr_to_limbs([1, C.r - 1, 2, C.r - 2, 3, 0x10001, (C.r - 1) // 2, 1 << 200], False)
    sc = vals[g.integers(0, len(vals), size=m)]
    if identity:
        idx = np.concatenate([idx, (idx + k) % (2 * k)])
        inf = np.concatenate([inf, inf])
        sc = np.concatenate([sc, sc])
    return np.ascontiguousarray(pool[idx]), inf, np.ascontiguousarray(sc)


def exceptional_case(eng, pc, cname, n, monkeypatch, rounds=None, tdiv=None, seed=7):
    """exceptional_inputs through the pair rounds (forced rounds / tdiv, or the default policy when None), plain and the
    identity-sum variant, against the oracle."""
    C = pyref.Curve(cname)
    monkeypatch.setenv("PCGPU_MSM_SMALL", "0")
    if rounds is not None:
        monkeypatch.setenv("PCGPU_MSM_AFFINE_ROUNDS", str(rounds))
    if tdiv is not None:
        monkeypatch.setenv("PCGPU_MSM_AFFINE_TDIV", str(tdiv))
    for identity in (False, True):
        bases, inf, sc = exceptional_inputs(cname, n, seed, identity)
        srs = eng.srs_register(C.id, bases, inf=inf)
        got = eng.msm(srs, sc)
        check_geometry(eng, pc, cname, bases.shape[0], depth=rounds is not None and ((tdiv or 1) > 1 or not on_gpu(eng)))
        exp = orc.msm(C.id, bases, sc, inf=inf)
        _assert_point(got, exp, (cname, n, rounds, tdiv, identity))
        if identity:
            assert got[1] == 1 and not got[0].any()
        srs.release()


def expected_heavy_buckets(cname, values, counts, c, W, S, R, L):
    """number of buckets the heavy-bucket kernel reduces for scalars `values` (canonical ints) repeated `counts` times:
    the signed-digit recoding of msm.cuh (range halving, carries), R pair rounds halving every bucket (rounding up), then
    more than HEAVY_BUCKET_TASKS tasks of L entries."""
    C = pyref.Curve(cname)
    half, size = 1 << (c - 1), {}
    for v, m in zip(values, counts):
        k = C.r - v if v > (C.r - 1) // 2 else v
        carry = 0
        for w in range(W):
            d = ((k >> (w * c)) & ((1 << c) - 1)) + carry
            carry = 1 if d > half else 0
            mag = (1 << c) - d if d > half else d
            if mag:
                key = (w % S, mag - 1)
                size[key] = size.get(key, 0) + m
    heavy = 0
    for cnt in size.values():
        for _ in range(R):
            cnt = (cnt + 1) // 2
        heavy += -(-cnt // L) > HEAVY_BUCKET_TASKS
    return heavy


def heavy_case(eng, pc, cname, bases, n_values, monkeypatch, seed=11, L=32):
    """scalars drawn from n_values distinct values: more than HEAVY_GRID buckets exceed HEAVY_BUCKET_TASKS, so the heavy-bucket
    kernel's blocks loop over the list.  Asserts the reported count against the recoding restated in Python."""
    C = pyref.Curve(cname)
    n = bases.shape[0]
    monkeypatch.setenv("PCGPU_MSM_SMALL", "0")
    if L != 32:
        monkeypatch.setenv("PCGPU_MSM_L", str(L))
    vals = util.rand_fr_ints(cname, n_values, seed)
    pick = util.rng(seed + 1).integers(0, n_values, size=n)
    sc = C.fr_to_limbs([vals[i] for i in pick], False)
    srs = eng.srs_register(C.id, bases)
    got = eng.msm(srs, sc)
    g = check_geometry(eng, pc, cname, n)
    _assert_point(got, orc.msm(C.id, bases, sc), (cname, n, n_values))
    exp_heavy = expected_heavy_buckets(cname, vals, np.bincount(pick, minlength=n_values), g["c"], g["W"],
                                       -(-g["W"] // g["G"]), g["R"], L)
    assert exp_heavy > HEAVY_GRID and g["heavy"] == exp_heavy, (g, exp_heavy)
    srs.release()
