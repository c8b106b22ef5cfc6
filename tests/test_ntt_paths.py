"""The four-step NTT of csrc/ntt.cuh (pcgpu_ntt, pcgpu_ntt_batch, pcgpu_ntt_pass, pcgpu_ntt_pass1_peer and the row encoding of
pcgpu_lincode_commit) against references that share nothing with it: the C oracle's recursive radix-2 transform (orc.fr_ntt),
Horner evaluation at w^j with w taken from the published two-adic roots (tests/golden/external_kats.json), and closed forms.
The same case bodies run on the host-emulated kernels (CPU, logn <= 16 and one logn 21 transform) and, with `-m gpu`, on the
device at every logn 1 ... 22.

Which launch shape runs is a pure function of (logn, count) -- no SM-count query, no environment knob -- so ntt_shapes() below
restates it exactly (csrc/ntt.cuh ntt_split, ntt_build_plan, ntt_launch, ntt_run, ntt_run_batch):
  * logn <= 11: one block pass of M = 2^logn.  Otherwise four-step, N1 = 2^m1 with m1 = ceil(logn / 2), N2 = 2^m2 with
    m2 = floor(logn / 2): pass 1 transforms the N2 columns (M = N1) and applies the step-2 twiddle w_N^(k1 n2), pass 2 the N1
    rows (M = N2);
  * the step-2 twiddle reads one full table w_N^e for 12 <= logn <= 20; for 21 and 22 it is hi[e >> 10] * lo[e & 1023];
  * block width: a launch of fewer than 4096 blocks uses 128 threads; from 4096 blocks up, M <= 256 uses 32 threads (16 blocks
    per SM), M <= 512 uses 64 (8 per SM) and larger M 128;
  * pcgpu_ntt_batch launches `count` blocks for single-pass rows; for four-step rows count * N2 blocks in pass 1 and then
    count * N1 blocks in pass 2.  pcgpu_ntt is the count = 1 case, so it never has more than 2048 blocks per pass.
Host emulation runs every block serially whatever its width, so only the device runs the 32- and 64-thread shapes.  On the
device every case also asserts its kernel count (Engine.launch_count() around one call, after a call that built the plan).
"""
import ctypes
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from oracle import orc, pyref
from tests import util
from tests.external_cases import published_root

MAX_LOG_BLOCK = 11        # csrc/ntt.cuh NTT_MAX_LOG_BLOCK: longest single block pass
LO_BITS = 10              # NTT_LO_BITS: the hi * lo split of the step-2 exponent
FULL_TABLE_MAX_LOG = 20   # NTT_FULL_TABLE_MAX_LOG: largest logn with one full step-2 table
MAX_LOG = 2 * MAX_LOG_BLOCK
NARROW_GRID = 4096        # ntt_launch: grids this large run narrow blocks when M allows
E_BADARG = -3

# the parameter lists; test_shape_policy_coverage asserts that the device lists reach every launch shape
SWEEP_GPU = list(range(1, MAX_LOG + 1))
SWEEP_CPU = list(range(1, 17))
CLOSED_FORM_LOGS = (11, 12, 20, 21, 22)
HILO_CPU = ("bls12_381", 21)
BATCH_GPU = [(1, 5000), (5, 8191), (8, 4096), (8, 4095), (9, 4096), (9, 4097), (10, 4096), (12, 64), (12, 63), (17, 16),
             (18, 8), (15, 128), (21, 2), (22, 2)]
# emulation runs blocks serially whatever their width, so only the shapes up to 2^20 elements run there
BATCH_CPU = [(logn, count) for logn, count in BATCH_GPU if count << logn <= 1 << 20]
PASSES_GPU = [(21, 8), (22, 8)]
PASSES_CPU = [(13, 8), (14, 8)]


def split(logn):
    if logn <= MAX_LOG_BLOCK:
        return logn, 0
    return (logn + 1) // 2, logn // 2


def block_width(M, nblocks):
    if nblocks < NARROW_GRID:
        return 128
    if M <= 256:
        return 32
    if M <= 512:
        return 64
    return 128


def ntt_shapes(logn, count=1):
    """the launches of pcgpu_ntt (count = 1) or pcgpu_ntt_batch (count rows), in order: dicts of kind ("single", "pass1",
    "pass2"), M, blocks, threads and twiddle (the step-2 table pass 1 reads: "full" or "hilo"; None for the other kinds)"""
    m1, m2 = split(logn)
    if m2 == 0:
        launches = [("single", 1 << m1, count, None)]
    else:
        tw = "full" if logn <= FULL_TABLE_MAX_LOG else "hilo"
        launches = [("pass1", 1 << m1, count << m2, tw), ("pass2", 1 << m2, count << m1, None)]
    return [dict(kind=k, M=M, blocks=b, threads=block_width(M, b), twiddle=tw) for k, M, b, tw in launches]


def pmap(fn, items):
    """fn over items on every core (the oracle's ctypes calls release the GIL)"""
    with ThreadPoolExecutor(os.cpu_count() or 1) as ex:
        return list(ex.map(fn, items))


def domain_w(cname, logn):
    """w = root^(2^(s - logn)) from the PUBLISHED 2^s-th root of unity: owes nothing to the oracle's domain generator"""
    _, s, root = published_root(cname)
    return pow(root, 1 << (s - logn), pyref.Curve(cname).r)


def scale(cname, a, k):
    """k * a elementwise (a Montgomery, k a Python int)"""
    C = pyref.Curve(cname)
    a = np.ascontiguousarray(a, dtype=np.uint64)
    return orc.fr_axpy(C.id, np.zeros_like(a), C.fr_to_limbs([k], True)[0], a)


def inverse_from_forward(cname, fwd):
    """ifft(y)[k] = N^-1 * fft(y)[-k mod N], from the forward transform fft(y) of the same zero-padded y"""
    N = fwd.shape[0]
    return scale(cname, np.concatenate([fwd[:1], fwd[:0:-1]]), pow(N, -1, pyref.Curve(cname).r))


def check_launches(eng, delta, logn, count=1, what=""):
    if util.on_gpu(eng):
        assert delta == len(ntt_shapes(logn, count)), (what, logn, count, delta)


def run_ntt(eng, pc, cname, x, logn, n_in, inverse=False, device=False):
    """one pcgpu_ntt of x[:n_in] -> (output, kernels launched); device: operands in device buffers (PCGPU_DEVICE_PTRS)"""
    cid = pyref.Curve(cname).id
    if not device:
        l0 = eng.launch_count()
        out = eng.ntt(cid, x[:n_in], logn, n_in=n_in, inverse=inverse)
        return out, eng.launch_count() - l0
    xb, ob = eng.buffer(n_in), eng.buffer(1 << logn)
    xb.write(x[:n_in])
    l0 = eng.launch_count()
    eng.ntt(cid, xb.ptr(), logn, n_in=n_in, inverse=inverse, flags=pc.DEVICE_PTRS, out=ob.ptr())
    delta = eng.launch_count() - l0
    out = ob.read()
    xb.release()
    ob.release()
    return out, delta


# ---------------------------------------------------------------------------------------------------------------------------
# case bodies
# ---------------------------------------------------------------------------------------------------------------------------
def sweep_input(cname, logn):
    """the random coefficients of the sweep at (cname, logn) and the length of the full comparison, N - 3"""
    N = 1 << logn
    return util.rand_fr_fast(cname, N, seed=7000 + 100 * pyref.Curve(cname).id + logn), (N - 3 if N > 3 else N)


def const_case(eng, cname, logn, c):
    """p = c (n_in = 1): every output of the forward transform is c, every output of the inverse c / N"""
    C = pyref.Curve(cname)
    for inverse in (False, True):
        got = eng.ntt(C.id, C.fr_to_limbs([c], True), logn, inverse=inverse)
        want = c * pow(1 << logn, -1, C.r) % C.r if inverse else c
        assert (got == C.fr_to_limbs([want], True)[0]).all(), (cname, logn, inverse)


def horner_case(cname, logn, coeffs, got, seed):
    """got[j] == p(w^j) at j = 0, 1, N/2, N - 1 and 60 random j, p the polynomial of `coeffs`"""
    C = pyref.Curve(cname)
    N, w = 1 << logn, domain_w(cname, logn)
    js = sorted({0, 1, N // 2, N - 1} | set(util.rng(seed).integers(0, N, size=60).tolist()))
    zs = C.fr_to_limbs([pow(w, j, C.r) for j in js], True)
    p = np.ascontiguousarray(coeffs)
    exp = pmap(lambda z: orc.fr_eval(C.id, p, z), list(zs))
    for j, e in zip(js, exp):
        assert (got[j] == e).all(), (cname, logn, len(p), j)


def closed_form_case(eng, pc, cname, logn):
    """transforms whose result is known without any transform: every coefficient r - 1 (each butterfly's add and sub at the
    reduction edge), X^k -> w^(jk) for k = 1, N/2, N - 1, and the inverses of the all-ones and of the (w^j) evaluations"""
    C = pyref.Curve(cname)
    N, w = 1 << logn, domain_w(cname, logn)
    one = C.fr_to_limbs([1], True)[0]
    pw = orc.field_unop("orc_fr_to_mont", C.id, orc.fr_powers_canonical(C.id, C.fr_to_limbs([w], True)[0], N))   # w^j, j < N
    assert C.fr_from_limbs(pw[[1, N // 2]], True) == [w, C.r - 1]

    def fwd(x, inverse=False):
        out, launches = run_ntt(eng, pc, cname, x, logn, x.shape[0], inverse)
        check_launches(eng, launches, logn, what=("closed form", cname, inverse))
        return out

    def unit(k, v):
        e = np.zeros((N, 4), dtype=np.uint64)
        e[k] = v
        return e
    rm1 = np.tile(C.fr_to_limbs([C.r - 1], True), (N, 1))
    assert (fwd(rm1) == unit(0, C.fr_to_limbs([-N], True)[0])).all(), "all r - 1, forward"
    assert (fwd(rm1, True) == unit(0, rm1[0])).all(), "all r - 1, inverse"
    for k in (1, N // 2, N - 1):
        xk = np.zeros((k + 1, 4), dtype=np.uint64)
        xk[k] = one
        assert (fwd(xk) == pw[(np.arange(N, dtype=np.int64) * k) % N]).all(), ("X^k", k)
    assert (fwd(np.tile(one, (N, 1)), True) == unit(0, one)).all(), "inverse of all ones"
    assert (fwd(pw, True) == unit(1, one)).all(), "inverse of the evaluations of X"


def sweep_case(eng, pc, cname, logn, closed=False):
    """one (curve, logn) of the pcgpu_ntt sweep, both directions: the constant closed form (it builds the two plans), the full
    comparison at n_in = N - 3 and the inverse of that zero-padded vector, Horner samples at n_in = N2 - 1, N2 + 1 and N/2 + 1
    (n_in < N2 leaves only row k1 = 0 of every column live; N2 + 1 crosses into row 1).  logn 22 runs as bench.py calls it:
    device pointers in and out, n_in = 2^22 - 3."""
    C = pyref.Curve(cname)
    N, N2 = 1 << logn, 1 << split(logn)[1]
    x, n_full = sweep_input(cname, logn)
    with ThreadPoolExecutor(1) as ex:
        oracle = ex.submit(orc.fr_ntt, C.id, np.ascontiguousarray(x[:n_full]), logn)   # overlaps the device calls below
        const_case(eng, cname, logn, util.rand_fr_ints(cname, 1, seed=logn)[0])
        device = logn == MAX_LOG
        got, launches = run_ntt(eng, pc, cname, x, logn, n_full, device=device)
        check_launches(eng, launches, logn, what=(cname, "forward"))
        inv, launches = run_ntt(eng, pc, cname, x, logn, n_full, inverse=True, device=device)
        check_launches(eng, launches, logn, what=(cname, "inverse"))
        exp = oracle.result()
    assert (got == exp).all(), (cname, logn, "forward")
    assert (inv == inverse_from_forward(cname, exp)).all(), (cname, logn, "inverse")
    for n_in in sorted({N2 - 1, N2 + 1, N // 2 + 1} - {0}):
        y, launches = run_ntt(eng, pc, cname, x, logn, n_in)
        check_launches(eng, launches, logn, what=(cname, "horner", n_in))
        horner_case(cname, logn, x[:n_in], y, seed=logn + n_in)
    if closed:
        closed_form_case(eng, pc, cname, logn)


def plan_cache_case(eng, pc, logns):
    """after the sweep: one plan per (curve, logn, direction) in the context's cache (the constant transform builds any the
    sweep did not), then the first three transforms of the sweep again"""
    cells = [(cname, logn) for cname in util.CURVE_NAMES for logn in logns]
    for cname, logn in cells:
        const_case(eng, cname, logn, 5)
    for logn in logns[:3]:
        cname = util.CURVE_NAMES[0]
        x, n_full = sweep_input(cname, logn)
        exp = orc.fr_ntt(pyref.Curve(cname).id, x[:n_full], logn)
        assert (run_ntt(eng, pc, cname, x, logn, n_full)[0] == exp).all(), (logn, "forward after the sweep")
        assert (run_ntt(eng, pc, cname, x, logn, n_full, inverse=True)[0] == inverse_from_forward(cname, exp)).all()
    return 2 * len(cells)


def batch_case(eng, cname, logn, count, seed):
    """pcgpu_ntt_batch of `count` partial rows (n_in < N, so i_valid and in_row_stride matter), both directions, each checked
    row against orc.fr_ntt; every row unless that is more than 2^22 elements of oracle work, else the first, the last and 16
    random rows"""
    C = pyref.Curve(cname)
    N = 1 << logn
    n_in = N - N // 4 - 1 if N >= 8 else N // 2
    rows = util.rand_fr_fast(cname, count * n_in, seed=seed).reshape(count, n_in, 4)
    if count * N <= 1 << 22:
        idx = list(range(count))
    else:
        idx = sorted({0, count - 1} | set(util.rng(seed).integers(0, count, size=16).tolist()))
    with ThreadPoolExecutor(1) as ex:
        oracle = ex.submit(pmap, lambda r: orc.fr_ntt(C.id, rows[r], logn), idx)
        for inverse in (False, True):
            eng.ntt(C.id, rows[0], logn, inverse=inverse)          # builds the plan
        got = {}
        for inverse in (False, True):
            l0 = eng.launch_count()
            got[inverse] = eng.ntt_batch(C.id, rows, logn, inverse=inverse)
            check_launches(eng, eng.launch_count() - l0, logn, count, what=(cname, "batch", inverse))
        exp = oracle.result()
    for r, e in zip(idx, exp):
        assert (got[False][r] == e).all(), (cname, logn, count, "forward", r)
        assert (got[True][r] == inverse_from_forward(cname, e)).all(), (cname, logn, count, "inverse", r)


def lincode_rows_case(eng, cname, n_rows, n_cols, log_ext, seed):
    """the row encoding inside pcgpu_lincode_commit: every row of `ext` against orc.fr_ntt (the hashes and the tree are
    checked against hashlib by test_lincode_hash.py)"""
    C = pyref.Curve(cname)
    mat = util.rand_fr_fast(cname, n_rows * n_cols, seed=seed).reshape(n_rows, n_cols, 4)
    ext = eng.lincode_commit(C.id, mat, log_ext)["ext"]
    exp = pmap(lambda r: orc.fr_ntt(C.id, mat[r], log_ext), range(n_rows))
    for r in range(n_rows):
        assert (ext[r] == exp[r]).all(), (cname, n_rows, n_cols, log_ext, r)


def sharded_passes_case(eng, cname, logn, world, seed):
    """pcgpu_ntt_pass: every rank's slice of pass 1 (which = 1, columns [r * cols, (r + 1) * cols): the step-2 exponent takes
    the slice's offset), the all-to-all done on the host, every rank's pass 2; reassembled, both directions equal pcgpu_ntt"""
    C = pyref.Curve(cname)
    m1, m2 = split(logn)
    assert eng.ntt_split(logn) == (m1, m2)
    N1, N2 = 1 << m1, 1 << m2
    cols, rows = N2 // world, N1 // world
    n_in = (1 << logn) - 77
    x = util.rand_fr_fast(cname, n_in, seed=seed)
    xb = eng.buffer(n_in)
    xb.write(x)
    for inverse in (False, True):
        exp = eng.ntt(C.id, x, logn, inverse=inverse)         # also builds the plan the passes use
        parts = []
        for r in range(world):
            a = eng.buffer(N1 * cols)
            l0 = eng.launch_count()
            eng.ntt_pass(C.id, logn, 1, r * cols, cols, xb.ptr(), n_in, a.ptr(), inverse=inverse)
            assert not util.on_gpu(eng) or eng.launch_count() - l0 == 1
            parts.append(a.read().reshape(N1, cols, 4))
            a.release()
        outs = []
        for r in range(world):
            rb, o = eng.buffer(rows * N2), eng.buffer(N2 * rows)
            rb.write(np.concatenate([p[r * rows:(r + 1) * rows] for p in parts], axis=1))    # [k1 - r * rows][n2]
            eng.ntt_pass(C.id, logn, 2, r * rows, rows, rb.ptr(), rows * N2, o.ptr(), inverse=inverse)
            outs.append(o.read().reshape(N2, rows, 4))                                      # [k2][k1 - r * rows]
            rb.release()
            o.release()
        got = np.stack(outs, 1).reshape(-1, 4)
        assert (got == exp).all(), (cname, logn, world, inverse)
    xb.release()


def pass1_peer_case(eng, cname, logn, world, seed):
    """pcgpu_ntt_pass1_peer with every rank's row buffer on this one device: each rank's columns stored straight into the
    owners' rows, then pass 2 per rank; reassembled, both directions equal pcgpu_ntt"""
    C = pyref.Curve(cname)
    m1, m2 = split(logn)
    N1, N2 = 1 << m1, 1 << m2
    cols, rows = N2 // world, N1 // world
    n_in = (1 << logn) - 5
    x = util.rand_fr_fast(cname, n_in, seed=seed)
    xb = eng.buffer(n_in)
    xb.write(x)
    for inverse in (False, True):
        bufs = [eng.buffer(rows * N2) for _ in range(world)]
        for r in range(world):
            eng.ntt_pass1_peer(C.id, logn, r * cols, cols, xb.ptr(), n_in, [b.ptr() for b in bufs], inverse=inverse)
        outs = []
        for r in range(world):
            o = eng.buffer(N2 * rows)
            eng.ntt_pass(C.id, logn, 2, r * rows, rows, bufs[r].ptr(), rows * N2, o.ptr(), inverse=inverse)
            outs.append(o.read().reshape(N2, rows, 4))
            o.release()
        for b in bufs:
            b.release()
        got = np.stack(outs, 1).reshape(-1, 4)
        assert (got == eng.ntt(C.id, x, logn, inverse=inverse)).all(), (cname, logn, world, inverse)
    xb.release()


def errors_case(eng, cname):
    """logn 0 and 23 are PCGPU_E_BADARG on pcgpu_ntt, pcgpu_ntt_batch, pcgpu_ntt_pass and pcgpu_ntt_split; pcgpu_ntt_pass is
    PCGPU_E_BADARG at every single-pass logn.  After each error the context still computes a correct transform."""
    C = pyref.Curve(cname)
    L, ctx, vp = eng.lib, eng.ctx, ctypes.c_void_p
    x = util.rand_fr_fast(cname, 16, seed=91)
    out = np.zeros((16, 4), dtype=np.uint64)
    px, po = x.ctypes.data_as(vp), out.ctypes.data_as(vp)
    good = {inv: (orc.fr_ntt(C.id, x, 4) if not inv else inverse_from_forward(cname, orc.fr_ntt(C.id, x, 4))) for inv in (0, 1)}

    def still_good(what):
        for inv in (0, 1):
            assert (eng.ntt(C.id, x, 4, inverse=bool(inv)) == good[inv]).all(), what
    m1, m2 = ctypes.c_uint32(), ctypes.c_uint32()
    for logn in (0, MAX_LOG + 1):
        for flags in (0, 8):
            assert L.pcgpu_ntt(ctx, C.id, px, 1, logn, flags, po) == E_BADARG, ("ntt", logn, flags)
            still_good(("ntt", logn))
            assert L.pcgpu_ntt_batch(ctx, C.id, px, 1, 1, logn, flags, po) == E_BADARG, ("ntt_batch", logn, flags)
            still_good(("ntt_batch", logn))
            for which in (1, 2):
                assert L.pcgpu_ntt_pass(ctx, C.id, logn, flags, which, 0, 1, px, 1, po) == E_BADARG, ("ntt_pass", logn, which)
                still_good(("ntt_pass", logn))
        assert L.pcgpu_ntt_split(logn, ctypes.byref(m1), ctypes.byref(m2)) == E_BADARG
    for logn in range(1, MAX_LOG_BLOCK + 1):
        for which in (1, 2):
            assert L.pcgpu_ntt_pass(ctx, C.id, logn, 0, which, 0, 1, px, 1, po) == E_BADARG, ("single-pass ntt_pass", logn)
    still_good("single-pass ntt_pass")
    assert not out.any()


# ---------------------------------------------------------------------------------------------------------------------------
# the policy and its coverage
# ---------------------------------------------------------------------------------------------------------------------------
def test_shape_policy_coverage(emul):
    """the device parameter lists reach every launch shape; ntt_shapes agrees with the library's own split"""
    for logn in range(1, MAX_LOG + 1):
        assert emul.ntt_split(logn) == split(logn), logn
        for s in ntt_shapes(logn):
            assert s["blocks"] <= 2048 and s["threads"] == 128, (logn, s)     # pcgpu_ntt never narrows its blocks
    batch = {(s["kind"], s["threads"]) for logn, count in BATCH_GPU for s in ntt_shapes(logn, count)}
    missing = {(k, t) for k in ("single", "pass1", "pass2") for t in (128, 64, 32)} - batch
    assert not missing, f"ntt_batch shapes no case runs: {sorted(missing)}"
    single = {(s["twiddle"], inverse, cname) for cname in util.CURVE_NAMES for logn in SWEEP_GPU for inverse in (False, True)
              for s in ntt_shapes(logn) if s["kind"] == "pass1"}
    missing = {(tw, inverse, cname) for tw in ("full", "hilo") for inverse in (False, True) for cname in util.CURVE_NAMES} - single
    assert not missing, f"ntt twiddle modes no case runs: {sorted(missing)}"
    assert {s["twiddle"] for logn, count in BATCH_GPU for s in ntt_shapes(logn, count)} >= {"full", "hilo"}
    assert HILO_CPU[1] > FULL_TABLE_MAX_LOG                                    # the emulated run also reads hi * lo
    # DESIGN section 4's Ligero 2^20 shape: 128 rows x 2^15, both passes 32 threads wide
    assert [(s["blocks"], s["threads"]) for s in ntt_shapes(15, 128)] == [(16384, 32), (32768, 32)]


# ---------------------------------------------------------------------------------------------------------------------------
# host emulation
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emul(pc, hostcheck_path, oracle):
    e = pc.Engine(0, lib_path=hostcheck_path)
    yield e
    e.close()


@pytest.fixture(scope="module")
def emul_sweep(pc, hostcheck_path, oracle):
    """a fresh context for the sweep: its plan cache fills up as the sweep goes"""
    e = pc.Engine(0, lib_path=hostcheck_path)
    yield e
    e.close()


@pytest.mark.parametrize("logn", SWEEP_CPU)
@pytest.mark.parametrize("cname", util.CURVE_NAMES)
def test_emul_ntt_sweep(emul_sweep, pc, cname, logn):
    sweep_case(emul_sweep, pc, cname, logn, closed=logn in CLOSED_FORM_LOGS)


def test_emul_ntt_hilo(emul_sweep, pc):
    """one transform with the hi * lo step-2 twiddle, against the oracle"""
    cname, logn = HILO_CPU
    x, n_full = sweep_input(cname, logn)
    got, _ = run_ntt(emul_sweep, pc, cname, x, logn, n_full)
    assert (got == orc.fr_ntt(pyref.Curve(cname).id, x[:n_full], logn)).all()


def test_emul_ntt_plan_cache(emul_sweep, pc):
    plan_cache_case(emul_sweep, pc, SWEEP_CPU)


@pytest.mark.parametrize("logn,count", BATCH_CPU)
def test_emul_ntt_batch_shapes(emul, logn, count):
    batch_case(emul, util.CURVE_NAMES[BATCH_GPU.index((logn, count)) % 3], logn, count, seed=8000 + 64 * logn + count)


def test_emul_lincode_commit_rows(emul):
    lincode_rows_case(emul, "bls12_381", 64, 1000, 12, seed=81)


@pytest.mark.parametrize("logn,world", PASSES_CPU)
@pytest.mark.parametrize("cname", util.CURVE_NAMES)
def test_emul_sharded_passes(emul, cname, logn, world):
    sharded_passes_case(emul, cname, logn, world, seed=82 + logn)


@pytest.mark.parametrize("cname", util.CURVE_NAMES)
def test_emul_pass1_peer(emul, cname):
    pass1_peer_case(emul, cname, 13, 8, seed=83)


@pytest.mark.parametrize("cname", util.CURVE_NAMES)
def test_emul_errors(emul, cname):
    errors_case(emul, cname)


# ---------------------------------------------------------------------------------------------------------------------------
# the device
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gpu_sweep(pc, oracle):
    """a fresh context on cuda:0 for the sweep"""
    e = pc.Engine(0)
    yield e
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("logn", SWEEP_GPU)
@pytest.mark.parametrize("cname", util.CURVE_NAMES)
def test_gpu_ntt_sweep(gpu_sweep, pc, cname, logn):
    sweep_case(gpu_sweep, pc, cname, logn, closed=logn in CLOSED_FORM_LOGS)


@pytest.mark.gpu
def test_gpu_ntt_plan_cache(gpu_sweep, pc):
    assert plan_cache_case(gpu_sweep, pc, SWEEP_GPU) > 100


@pytest.mark.gpu
@pytest.mark.parametrize("logn,count", BATCH_GPU)
def test_gpu_ntt_batch_shapes(gpu_engine, logn, count):
    batch_case(gpu_engine, util.CURVE_NAMES[BATCH_GPU.index((logn, count)) % 3], logn, count, seed=8000 + 64 * logn + count)


@pytest.mark.gpu
def test_gpu_lincode_commit_rows_2p20_shape(gpu_engine):
    """the Ligero shape of a 2^20-coefficient polynomial (DESIGN section 4): 128 rows of 8192 coefficients -> 2^15"""
    lincode_rows_case(gpu_engine, "bls12_381", 128, 8192, 15, seed=84)


@pytest.mark.gpu
@pytest.mark.parametrize("logn,world", PASSES_GPU)
@pytest.mark.parametrize("cname", util.CURVE_NAMES)
def test_gpu_sharded_passes(gpu_engine, cname, logn, world):
    sharded_passes_case(gpu_engine, cname, logn, world, seed=82 + logn)


@pytest.mark.gpu
@pytest.mark.parametrize("cname", util.CURVE_NAMES)
def test_gpu_pass1_peer(gpu_engine, cname):
    pass1_peer_case(gpu_engine, cname, MAX_LOG, 8, seed=83)


@pytest.mark.gpu
@pytest.mark.parametrize("cname", util.CURVE_NAMES)
def test_gpu_errors(gpu_engine, cname):
    errors_case(gpu_engine, cname)
