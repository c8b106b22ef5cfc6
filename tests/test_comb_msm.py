"""The fixed-base comb behind pcgpu_msm_batch over PCGPU_SRS_COMB tables (HyraxPC::commit's row loop, hyrax/mod.rs:233-242) and
the Hyrax open's pcgpu_fr_row_mul, against the C oracle.  The same case bodies run on the host-emulated kernels (CPU) and, with
`-m gpu`, on the device.

The comb runs three kernels of csrc/srs.cuh that no other path uses: CombTableBody (d * 2^(c w) * G_j for d = 1 .. 2^(c-1),
built in chunks of COMB_CHUNK entries that each start from a double-and-add), CombAccumulateBody (signed-digit lookups with
load_scalar's range-halving flip and mixed XYZZ additions over one segment of a row) and CombRowSumBody (the row's segment
partials summed with xyzz_add).  Every case forces the window with PCGPU_COMB_C (read at registration) and asserts, through
Engine.msm_last_geometry, the window and segmentation it exercised.  The policy restated here (csrc/impl.cuh msm_batch_impl):
  * W = ceil(BITS / c), BITS = the bit length of r: 255 for BLS12-381 and Pallas, 254 for BN254;
  * seg_len = 64 for count >= 4096 rows; below that it halves from 64 while it is above 8 and count * ceil(n / seg_len) is
    below 65536; each row is cut into ceil(n / seg_len) segments, and entries = count * segments accumulate tasks.
"""
import numpy as np
import pytest

from oracle import orc, pyref
from tests import util

COMB_CHUNK = 256                 # csrc/srs.cuh: table entries one CombTableBody thread builds
SEG_TASKS = 65536                # csrc/impl.cuh: seg_len halves while a batch has fewer accumulate tasks than this
E_LEN, E_RANGE = -4, -5


def fr_bits(cname):
    return pyref.Curve(cname).r.bit_length()


def comb_windows(cname, c):
    return -(-fr_bits(cname) // c)


def seg_len(n, count):
    s = 64
    if count < 4096:
        while s > 8 and count * -(-n // s) < SEG_TASKS:
            s //= 2
    return s


def check_geometry(eng, pc, cname, n, count, c):
    """asserts that the last batch on `eng` ran the comb with window c and the documented segmentation; returns seg_len"""
    g = eng.msm_last_geometry()
    s = seg_len(n, count)
    exp = dict.fromkeys(pc.binding.GEOM_FIELDS, 0)
    exp.update(path=pc.binding.MSM_PATH_COMB, n=n, c=c, W=comb_windows(cname, c), split=s, entries=count * -(-n // s))
    assert g == exp, (g, exp)
    return s


def limbs(vals):
    """python ints (not reduced) -> (n, 4) uint64 raw limbs"""
    out = np.zeros((len(vals), 4), dtype=np.uint64)
    for i, v in enumerate(vals):
        for j in range(4):
            out[i, j] = (v >> (64 * j)) & (2**64 - 1)
    return out


def register_comb(eng, pc, monkeypatch, cname, bases, c, inf=None):
    monkeypatch.setenv("PCGPU_COMB_C", str(c))
    return eng.srs_register(pyref.Curve(cname).id, bases, inf=inf, flags=pc.SRS_COMB)


def expected_rows(cname, bases, rows, inf=None):
    """one oracle MSM per row of canonical scalars (rows: (count, n, 4))"""
    cid = pyref.Curve(cname).id
    n = rows.shape[1]
    return [orc.msm(cid, bases[:n], rows[r], inf=None if inf is None else inf[:n], nthreads=1 if n < 256 else 0)
            for r in range(rows.shape[0])]


def assert_rows(got, inf, exp, what):
    for r, e in enumerate(exp):
        assert inf[r] == e[1] and (got[r] == e[0]).all(), (what, r)


ALL_ROWS = 64   # check_rows compares up to this many rows one by one


def check_rows(cname, bases, canon, got, inf, what):
    """every row against the oracle for small batches; for large ones, the first, middle and last rows and a random sample
    one by one, and the sum of all row results against the MSM of the column sums (a wrong row shows up in the sum)"""
    count, n = canon.shape[:2]
    if count <= ALL_ROWS:
        assert_rows(got, inf, expected_rows(cname, bases, canon), what)
        return
    C = pyref.Curve(cname)
    idx = sorted({0, 1, count // 2, count - 2, count - 1} | set(util.rng(count + n).integers(0, count, size=11).tolist()))
    assert_rows(got[idx], inf[idx], expected_rows(cname, bases, canon[idx]), what)
    one = np.tile(util.fr_const(cname, 1), (count, 1))
    colsum = orc.fr_row_mul(C.id, one, canon.reshape(-1, 4), count, n)   # Montgomery 1 times canonical values: column sums
    tot = orc.g1_sum(C.id, got, inf)
    exp = orc.msm(C.id, bases[:n], colsum)
    assert tot[1] == exp[1] and (tot[0] == exp[0]).all(), (what, "sum of all rows")


# ---------------------------------------------------------------------------------------------------------------------------
# case bodies
# ---------------------------------------------------------------------------------------------------------------------------
def edge_values(cname, c):
    """the scalars where the comb's digit recoding goes wrong first, canonical"""
    C = pyref.Curve(cname)
    r, W, half = C.r, comb_windows(cname, c), (C.r - 1) // 2

    def capped(digit):   # every window holds `digit`, as many windows as keep the scalar <= (r - 1) / 2 (no flip)
        s = 0
        for w in range(W):
            if s + (digit << (c * w)) > half:
                break
            s += digit << (c * w)
        return s
    top = capped(1 << (c - 1))                        # every digit is +2^(c-1): the last table entry of every window
    carry = capped((1 << (c - 1)) + 1)                # every digit is negative and carries into the next window
    vals = [0, 1, 2, r - 1, r - 2, half, half + 1, top, r - top, carry, r - carry,
            sum((1 << (c - 1)) << (c * w) for w in range(W)) % r, sum(((1 << (c - 1)) + 1) << (c * w) for w in range(W)) % r,
            1 << 253, r - (1 << 253)]
    assert all(0 <= v < r for v in vals)
    return vals


def sweep_bases(cname, k, seed):
    """k random points, then a copy of P0, -P1 and an identity base (inf flag set over P2's coordinates): n = k + 3"""
    C = pyref.Curve(cname)
    pts = util.random_points(cname, k, seed=seed)
    neg = C.points_to_limbs([C.neg(C.points_from_limbs(pts[1:2])[0])])[0]
    bases = np.concatenate([pts, pts[0:1], neg, pts[2:3]])
    inf = np.zeros(k + 3, dtype=np.uint8)
    inf[k + 2] = 1
    return bases, inf


def window_sweep_case(eng, pc, cname, c, k, monkeypatch, seed=0):
    """every edge value in every term, the edge values rotated across the terms, uniform rows and a row that sums to the
    identity through the duplicated and the negated base; canonical and Montgomery input"""
    C = pyref.Curve(cname)
    bases, inf = sweep_bases(cname, k, seed=100 + seed)
    n = k + 3
    vals = edge_values(cname, c)
    rows = [[v] * n for v in vals] + [[vals[(j + i) % len(vals)] for i in range(n)] for j in range(len(vals))]
    rows += [util.rand_fr_ints(cname, n, seed=200 + seed + j) for j in range(2)]
    u = util.rand_fr_ints(cname, 3, seed=300 + seed)
    ident = [0] * n
    ident[0], ident[k], ident[1], ident[k + 1], ident[k + 2] = u[0], C.r - u[0], u[1], u[1], u[2]
    rows.append(ident)
    canon = np.stack([limbs(row) for row in rows])
    count = canon.shape[0]
    exp = expected_rows(cname, bases, canon, inf)
    assert exp[-1][1] == 1
    srs = register_comb(eng, pc, monkeypatch, cname, bases, c, inf=inf)
    mont = orc.field_unop("orc_fr_to_mont", C.id, canon.reshape(-1, 4)).reshape(canon.shape)
    for sc, flags in ((canon, 0), (mont, pc.SCALARS_MONT)):
        got, oinf = eng.msm_batch(srs, sc, n, count, flags=flags)
        check_geometry(eng, pc, cname, n, count, c)
        assert_rows(got, oinf, exp, (cname, c, flags))
        assert oinf[-1] == 1 and not got[-1].any()
    srs.release()


def table_sweep_rows(cname, c, n_bases, count):
    """row k gives base i the digit d = ((k + 7 i) mod 2^(c-1)) + 1 in every window below the top: with count >= 2^(c-1) rows
    every entry of those windows is read for every base.  Rows alternate between the scalar and r minus it, and the pattern
    flips after 2^(c-1) rows, so with 2^c rows each of those entries is read with both signs."""
    C = pyref.Curve(cname)
    W, half_d, half = comb_windows(cname, c), 1 << (c - 1), (C.r - 1) // 2
    rows = []
    for k in range(count):
        row = []
        for i in range(n_bases):
            d = (k + 7 * i) % half_d + 1
            s = sum(d << (c * w) for w in range(W - 1))
            assert s <= half, (c, k, i)          # digits below the top window never reach the range-halving threshold
            row.append(C.r - s if (k + k // half_d) % 2 else s)
        rows.append(row)
    return rows


def exceptional_case(eng, pc, cname, c, monkeypatch, big=False):
    """rows whose accumulator meets +-the next table entry (CombAccumulateBody's xyzz_madd doubling and cancellation
    branches), and rows whose second segment repeats or negates the first (CombRowSumBody's xyzz_add P = Q and P = -Q)"""
    C = pyref.Curve(cname)
    r = C.r
    G = util.random_points(cname, 1, seed=40 + c)
    G2 = C.points_to_limbs([C.mul(2, C.points_from_limbs(G)[0])])[0]
    Gc = C.points_to_limbs([C.mul(1 << c, C.points_from_limbs(G)[0])])[0]
    # madd: [G, G, 2G, G, 2^c G]
    bases = np.concatenate([G, G, G2, G, Gc])
    rows = [[1, 1, 0, 0, 0], [1, r - 1, 0, 0, 0], [1, 1, 1, 0, 0], [1, 1, r - 1, 0, 0], [1, 1, r - 2, 0, 0],
            [0, 0, 0, 1 << c, 1], [0, 0, 0, 1 << c, r - 1], [0, 0, 0, r - (1 << c), 1], [5, 7, r - 6, 0, 0]]
    canon = np.stack([limbs(row) for row in rows])
    exp = expected_rows(cname, bases, canon)
    assert [e[1] for e in exp] == [0, 1, 0, 1, 0, 0, 1, 1, 1]
    srs = register_comb(eng, pc, monkeypatch, cname, bases, c)
    got, oinf = eng.msm_batch(srs, canon, 5, len(rows))
    check_geometry(eng, pc, cname, 5, len(rows), c)
    assert_rows(got, oinf, exp, (cname, c, "madd"))
    srs.release()
    # row sum: count rows of n = 2 * seg_len terms over bases B || B; the second segment holds the first one's scalars (P = Q),
    # their negations (P = -Q: the row is the identity) or fresh scalars
    count = 4096 if big else 4
    s = seg_len(2 * 64 if big else 16, count)
    n = 2 * s
    assert seg_len(n, count) == s
    half_b = util.random_points(cname, s, seed=50 + c)
    bases = np.concatenate([half_b, half_b])
    rows = []
    for j in range(count):
        a = util.rand_fr_ints(cname, s, seed=60 + j) if j < 8 else [((j * 7919 + i) * 2654435761) % r for i in range(s)]
        second = a if j % 3 == 0 else [(r - v) % r for v in a] if j % 3 == 1 else util.rand_fr_ints(cname, s, seed=9000 + j)
        rows.append(a + second)
    canon = np.stack([limbs(row) for row in rows])
    srs = register_comb(eng, pc, monkeypatch, cname, bases, c)
    got, oinf = eng.msm_batch(srs, canon, n, count)
    assert check_geometry(eng, pc, cname, n, count, c) == s
    check_rows(cname, bases, canon, got, oinf, (cname, c, "row sum", s))
    assert oinf[1::3].all() and not got[1::3].any() and not oinf[0::3].any()
    srs.release()


def shape_case(eng, pc, cname, c, shapes, monkeypatch, seed=70):
    """rows x row lengths around the segment boundaries, over a key longer than every row (n < srs.n: a prefix of the key)"""
    C = pyref.Curve(cname)
    n_key = max(n for _, n in shapes) + 1
    bases = util.random_points(cname, n_key, seed=seed)
    srs = register_comb(eng, pc, monkeypatch, cname, bases, c)
    for count, n in shapes:
        sc = util.rand_fr(cname, count * n, seed=seed + 7 * count + n, mont=False).reshape(count, n, 4)
        got, oinf = eng.msm_batch(srs, sc, n, count)
        check_geometry(eng, pc, cname, n, count, c)
        check_rows(cname, bases, sc, got, oinf, (cname, count, n))
    srs.release()


def error_case(eng, pc, cname, c, monkeypatch, seed=80):
    """PCGPU_E_LEN for n > srs.n, empty batches, n = 0 (the per-row path: identities), PCGPU_E_RANGE for an unreduced
    canonical scalar followed by a correct batch on the same context, and device-resident scalars"""
    C = pyref.Curve(cname)
    n, count = 9, 3
    bases = util.random_points(cname, n, seed=seed)
    srs = register_comb(eng, pc, monkeypatch, cname, bases, c)
    sc = util.rand_fr(cname, count * (n + 1), seed=seed + 1, mont=False).reshape(count, n + 1, 4)
    with pytest.raises(pc.PcgpuError) as ei:
        eng.msm_batch(srs, sc, n + 1, count)
    assert ei.value.code == E_LEN
    got, oinf = eng.msm_batch(srs, sc, n, 0)
    assert got.shape[0] == 0 and oinf.shape[0] == 0
    got, oinf = eng.msm_batch(srs, sc, 0, count)
    assert oinf.all() and not got.any()
    assert eng.msm_last_geometry()["path"] == pc.binding.MSM_PATH_NONE
    sc = np.ascontiguousarray(sc[:, :n])
    exp = expected_rows(cname, bases, sc)
    for bad in (C.r, 2**256 - 1):
        b = sc.copy()
        b[count - 1, n - 1] = limbs([bad])[0]
        with pytest.raises(pc.PcgpuError) as ei:
            eng.msm_batch(srs, b, n, count)
        assert ei.value.code == E_RANGE, bad
        got, oinf = eng.msm_batch(srs, sc, n, count)
        check_geometry(eng, pc, cname, n, count, c)
        assert_rows(got, oinf, exp, (cname, "after E_RANGE", hex(bad)))
    mont = orc.field_unop("orc_fr_to_mont", C.id, sc.reshape(-1, 4))
    for arr, flags in ((sc, 0), (mont, pc.SCALARS_MONT)):
        ptr, keep = util.dev_ptr(eng, np.ascontiguousarray(arr))
        got, oinf = eng.msm_batch(srs, ptr, n, count, flags=flags | pc.DEVICE_PTRS)
        check_geometry(eng, pc, cname, n, count, c)
        assert_rows(got, oinf, exp, (cname, "device pointers", flags))
        del keep
    srs.release()


def row_mul_case(eng, cname, rows_list, cols_list, seed=90):
    """pcgpu_fr_row_mul (Matrix::row_mul, utils.rs:127-146) against the oracle: uniform operands, every operand r - 1 (the
    largest inputs fr_dot2 sees) and a zero matrix, at odd and even row counts (the unpaired last row)"""
    C = pyref.Curve(cname)
    top = limbs([C.r - 1])[0]
    for rows in rows_list:
        for cols in cols_list:
            v = util.rand_fr_fast(cname, rows, seed=seed + rows)
            m = util.rand_fr_fast(cname, rows * cols, seed=seed + rows + cols)
            for what, vv, mm in (("uniform", v, m), ("r-1", np.tile(top, (rows, 1)), np.tile(top, (rows * cols, 1))),
                                 ("zero matrix", v, np.zeros_like(m))):
                got = eng.fr_row_mul(C.id, vv, mm, rows, cols)
                exp = orc.fr_row_mul(C.id, vv, mm, rows, cols)
                assert (got == exp).all(), (cname, rows, cols, what)
                if what == "zero matrix":
                    assert not got.any()


# ---------------------------------------------------------------------------------------------------------------------------
# host emulation (CPU): the same kernel bodies, serially; tables kept near 10^5 entries
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emul(pc, hostcheck_path):
    e = pc.Engine(0, lib_path=hostcheck_path)
    yield e
    e.close()


@pytest.mark.parametrize("cname", util.CURVE_NAMES)
@pytest.mark.parametrize("c", [4, 5, 8, 10])
def test_emul_window_sweep(emul, pc, cname, c, monkeypatch):
    window_sweep_case(emul, pc, cname, c, 4, monkeypatch)


@pytest.mark.parametrize("cname", util.CURVE_NAMES)
def test_emul_exceptional_additions(emul, pc, cname, monkeypatch):
    exceptional_case(emul, pc, cname, 5, monkeypatch)


def test_emul_shapes(emul, pc, monkeypatch):
    shape_case(emul, pc, "bn254", 4, [(count, n) for count in (1, 2) for n in (1, 7, 8, 9, 63, 64, 65)] + [(4096, 1)],
               monkeypatch)


@pytest.mark.parametrize("cname", util.CURVE_NAMES)
def test_emul_errors_and_device_pointers(emul, pc, cname, monkeypatch):
    error_case(emul, pc, cname, 6, monkeypatch)


@pytest.mark.parametrize("cname", util.CURVE_NAMES)
def test_emul_row_mul(emul, cname):
    row_mul_case(emul, cname, (1, 2, 3, 8), (1, 31))


# ---------------------------------------------------------------------------------------------------------------------------
# device
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cname", util.CURVE_NAMES)
@pytest.mark.parametrize("c", list(range(4, 17)))
def test_gpu_window_sweep(gpu_engine, pc, cname, c, monkeypatch):
    """every window width 4 .. 16 (tables <= 0.5 GB)"""
    window_sweep_case(gpu_engine, pc, cname, c, 7, monkeypatch, seed=c)


TABLE_SWEEP = [("bn254", 10), ("bn254", 12), ("bn254", 16), ("bls12_381", 10), ("bls12_381", 12), ("pallas", 10),
               ("pallas", 12)]


@pytest.mark.gpu
@pytest.mark.parametrize("cname,c", TABLE_SWEEP)
def test_gpu_table_sweep(gpu_engine, pc, cname, c, monkeypatch):
    """every entry of the windows below the top read for 8 bases, so every CombTableBody chunk start d = 256 q + 1 and chunk
    end d = 256 q is read: 2^c rows at c = 10 / 12 (each entry with both signs), 2^(c-1) = 32768 rows at c = 16 (signs
    alternating by row; this also runs the count >= 4096 segmentation)"""
    eng = gpu_engine
    nb = 8
    count = (1 << c) if c <= 12 else 1 << (c - 1)
    assert (1 << (c - 1)) > COMB_CHUNK
    bases = util.random_points(cname, nb, seed=110 + c)
    rows = table_sweep_rows(cname, c, nb, count)
    canon = np.stack([limbs(row) for row in rows])
    srs = register_comb(eng, pc, monkeypatch, cname, bases, c)
    got, oinf = eng.msm_batch(srs, canon, nb, count)
    check_geometry(eng, pc, cname, nb, count, c)
    srs.release()
    assert_rows(got, oinf, expected_rows(cname, bases, canon), (cname, c))


@pytest.mark.gpu
@pytest.mark.parametrize("cname", util.CURVE_NAMES)
@pytest.mark.parametrize("c", [5, 11, 16])
def test_gpu_exceptional_additions(gpu_engine, pc, cname, c, monkeypatch):
    """the madd and row-sum exceptional branches, including 4096 rows of 128 terms (seg_len = 64)"""
    exceptional_case(gpu_engine, pc, cname, c, monkeypatch, big=c == 11)


@pytest.mark.gpu
def test_gpu_shapes(gpu_engine, pc, monkeypatch):
    """count 1, 2, 4095, 4096, 4097 x n 1, 7, 8, 9, 63, 64, 65 (seg_len 8 below 4096 rows, 64 from there), and 3000 rows of
    700 terms (seg_len 32)"""
    shapes = [(count, n) for count in (1, 2, 4095, 4096, 4097) for n in (1, 7, 8, 9, 63, 64, 65)] + [(3000, 700)]
    assert seg_len(700, 3000) == 32
    shape_case(gpu_engine, pc, "bn254", 8, shapes, monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("cname", util.CURVE_NAMES)
def test_gpu_errors_and_device_pointers(gpu_engine, pc, cname, monkeypatch):
    error_case(gpu_engine, pc, cname, 12, monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("cname", util.CURVE_NAMES)
def test_gpu_row_mul(gpu_engine, cname):
    row_mul_case(gpu_engine, cname, (1, 2, 3, 2047, 2048), (1, 31, 2049))


# cfg4 at size: (curve, log2 rows, forced window).  The tables are sized by the shape (5.9 GB for BN254 at c = 12, 1.3 GB
# for BLS12-381 at c = 10) and built once per curve.
CFG4 = [("bn254", 11, 12), ("pallas", 10, 10), ("bls12_381", 10, 10)]


@pytest.fixture(scope="module", params=CFG4, ids=[p[0] for p in CFG4])
def cfg4(request, gpu_engine, pc):
    cname, logd, c = request.param
    C = pyref.Curve(cname)
    dim = 1 << logd
    bases = util.random_points(cname, dim + 1, seed=120 + logd)        # com_key || h
    mat = util.rand_fr_fast(cname, dim * (dim + 1), seed=121 + logd).reshape(dim, dim + 1, 4)   # evaluations || r_i
    mat[3] = 0                                                         # a zero row commits to the identity
    with pytest.MonkeyPatch.context() as mp:
        comb = register_comb(gpu_engine, pc, mp, cname, bases, c)
    got, inf = gpu_engine.msm_batch(comb, mat, dim + 1, dim, flags=pc.SCALARS_MONT)
    geom = gpu_engine.msm_last_geometry()
    comb.release()
    yield dict(cname=cname, C=C, dim=dim, c=c, bases=bases, mat=mat, got=got, inf=inf, geom=geom)


@pytest.mark.gpu
def test_gpu_cfg4_rows(gpu_engine, pc, cfg4):
    """every row against the same row through the per-row MSM path (a registration without comb tables), 8 rows against the
    oracle"""
    d = cfg4
    C, dim = d["C"], d["dim"]
    g = d["geom"]
    s = seg_len(dim + 1, dim)
    assert (g["path"], g["n"], g["c"], g["W"], g["split"], g["entries"]) == \
        (pc.binding.MSM_PATH_COMB, dim + 1, d["c"], comb_windows(d["cname"], d["c"]), s, dim * -(-(dim + 1) // s)), g
    assert s == (64 if dim == 2048 else 16)
    plain = gpu_engine.srs_register(C.id, d["bases"])
    ref, rinf = gpu_engine.msm_batch(plain, d["mat"], dim + 1, dim, flags=pc.SCALARS_MONT)
    plain.release()
    assert (d["inf"] == rinf).all() and (d["got"] == ref).all()
    assert d["inf"][3] == 1 and d["inf"].sum() == 1
    for r in (0, 1, 3, 17, dim // 2, dim - 65, dim - 2, dim - 1):
        exp = orc.msm(C.id, d["bases"], orc.field_unop("orc_fr_from_mont", C.id, d["mat"][r]))
        assert d["inf"][r] == exp[1] and (d["got"][r] == exp[0]).all(), r


@pytest.mark.gpu
def test_gpu_cfg4_hyrax_identity_and_row_mul(gpu_engine, cfg4):
    """sum_i l_i C_i = commit(l^T M) + h <l, r> over all rows (the verifier's t_prime, hyrax/mod.rs:498-504), and the open's
    l^T M (hyrax/mod.rs:347) in every column against the oracle"""
    from poly_commit_b200 import hyrax
    d = cfg4
    C, dim, mat = d["C"], d["dim"], d["mat"]
    l = util.rand_fr_fast(d["cname"], dim, seed=130)
    lt = gpu_engine.fr_row_mul(C.id, l, mat.reshape(-1, 4), dim, dim + 1)      # l^T M || <l, r>
    assert (lt == orc.fr_row_mul(C.id, l, mat.reshape(-1, 4), dim, dim + 1)).all()
    assert (lt[dim] == gpu_engine.fr_inner_product(C.id, l, np.ascontiguousarray(mat[:, dim]))).all()
    t_prime, tinf = hyrax.check_t_prime(gpu_engine, C.id, d["got"], l, d["inf"])
    exp = orc.msm(C.id, d["bases"], orc.field_unop("orc_fr_from_mont", C.id, lt))
    assert (t_prime == exp[0]).all() and tinf == exp[1]
