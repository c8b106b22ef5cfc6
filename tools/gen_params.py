#!/usr/bin/env python3
"""Generate field/curve constants for the device headers (32-bit limbs) and the
C oracle (64-bit limbs) from the primes themselves, so no limb is typed by hand.

Parameters are the public curve parameters that ark-bls12-381 / ark-bn254 /
ark-pallas 0.5.0 instantiate (un-vendored crates; SURVEY.md section 8c lists
them and how they were verified arithmetically).  Conventions follow ark-ff:
Montgomery radix R = 2^(64*ceil(bits/64)), little-endian limbs.

Outputs (both committed):
  poly-commit_b200/csrc/params_gen.cuh
  oracle/params_gen.h
"""
import os, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CURVES = {
    # name: (p, r, b, Gx, Gy, fr_generator, two_adicity)
    "bls12_381": dict(
        p=0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffaaab,
        r=0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001,
        b=4,
        gx=0x17f1d3a73197d7942695638c4fa9ac0fc3688c4f9774b905a14e3a3f171bac586c55e83ff97a1aeffb3af00adb22c6bb,
        gy=0x08b3f481e3aaa0f1a09e30ed741d8ae4fcf5e095d5d00af600db18cb2c04b3edd03cc744a2888ae40caa232946c5e7e1,
        fr_gen=7, two_adicity=32),
    "bn254": dict(
        p=21888242871839275222246405745257275088696311157297823662689037894645226208583,
        r=21888242871839275222246405745257275088548364400416034343698204186575808495617,
        b=3, gx=1, gy=2, fr_gen=5, two_adicity=28),
    "pallas": dict(
        p=0x40000000000000000000000000000000224698fc094cf91b992d30ed00000001,
        r=0x40000000000000000000000000000000224698fc0994a8dd8c46eb2100000001,
        b=5, gx=-1, gy=2, fr_gen=5, two_adicity=32),
}


def limbs(x, n, w):
    m = (1 << w) - 1
    return [(x >> (w * i)) & m for i in range(n)]


def fmt(ls, w):
    d = w // 4
    suf = "u" if w == 32 else "ull"
    return ", ".join(f"0x{v:0{d}x}{suf}" for v in ls)


def field_consts(mod):
    n64 = (mod.bit_length() + 63) // 64
    R = 1 << (64 * n64)
    return dict(n64=n64, n32=2 * n64, mod=mod, R=R % mod, R2=R * R % mod,
                m0_32=(-pow(mod, -1, 1 << 32)) % (1 << 32),
                m0_64=(-pow(mod, -1, 1 << 64)) % (1 << 64),
                bits=mod.bit_length())


def ec_mul(k, P, p):
    """affine double-and-add on y^2 = x^3 + b (a = 0); None is the identity (generator-time checks only)"""
    def add(A, B):
        if A is None: return B
        if B is None: return A
        if A[0] == B[0]:
            if (A[1] + B[1]) % p == 0: return None
            lam = 3 * A[0] * A[0] * pow(2 * A[1], -1, p) % p
        else:
            lam = (B[1] - A[1]) * pow(B[0] - A[0], -1, p) % p
        x = (lam * lam - A[0] - B[0]) % p
        return (x, (lam * (A[0] - x) - A[1]) % p)
    R = None
    while k:
        if k & 1: R = add(R, P)
        P = add(P, P)
        k >>= 1
    return R


def sqrt_consts(p):
    """constants for y = sqrt(a) in Fq: p = 3 (mod 4) -> a^((p+1)/4); otherwise Tonelli-Shanks with p - 1 = 2^s t."""
    if p % 4 == 3:
        return dict(ts=0, s=1, exp=(p + 1) // 4, root=0)
    s, t = 0, p - 1
    while t % 2 == 0:
        s, t = s + 1, t // 2
    g = 2
    while pow(g, (p - 1) // 2, p) != p - 1:
        g += 1
    return dict(ts=1, s=s, exp=(t - 1) // 2, root=pow(g, t, p))


def glv_consts(c):
    """GLV data for y^2 = x^3 + b: phi(x, y) = (zeta x, y) acts as multiplication by lambda on the order-r group.
    Returns zeta (mod p), lambda (mod r) and a reduced lattice basis (a1, b1), (a2, b2) of {(a, b): a + b lambda = 0 mod r}
    with a1 b2 - a2 b1 = +r (extended Euclid on (r, lambda), stopped around sqrt(r))."""
    p, r = c["p"], c["r"]
    G = (c["gx"] % p, c["gy"] % p)
    g = 2
    while pow(g, (p - 1) // 3, p) == 1:
        g += 1
    z0 = pow(g, (p - 1) // 3, p)
    l0 = pow(c["fr_gen"], (r - 1) // 3, r)
    assert l0 != 1 and pow(l0, 3, r) == 1
    pick = None
    for zeta in (z0, z0 * z0 % p):
        for lam in (l0, l0 * l0 % r):
            if ec_mul(lam, G, p) == (zeta * G[0] % p, G[1]):
                pick = (zeta, lam)
    assert pick is not None
    zeta, lam = pick
    # r_i = s_i r + t_i lam
    rows = [(r, 1, 0), (lam, 0, 1)]
    while rows[-1][0] != 0:
        q = rows[-2][0] // rows[-1][0]
        rows.append(tuple(x - q * y for x, y in zip(rows[-2], rows[-1])))
    sq = int(r ** 0.5)
    l = max(i for i, row in enumerate(rows) if row[0] >= sq)
    v1 = (rows[l + 1][0], -rows[l + 1][2])
    cand = [(rows[l][0], -rows[l][2]), (rows[l + 2][0], -rows[l + 2][2])]
    v2 = min(cand, key=lambda v: v[0] * v[0] + v[1] * v[1])
    for a, b in (v1, v2):
        assert (a + b * lam) % r == 0
    det = v1[0] * v2[1] - v2[0] * v1[1]
    if det < 0:
        v2 = (-v2[0], -v2[1]); det = -det
    assert det == r and max(abs(x) for x in v1 + v2) < 1 << 128
    return dict(zeta=zeta, lam=lam, v1=v1, v2=v2)


BLS_X = 0xd201000000010000          # |z| of BLS12-381 (z is negative); ark-bls12-381 `Config::X`
BN_U = 4965661367192848881          # u of BN254 (positive); the optimal-ate loop runs over 6u + 2


def fq2_mul(a, b, p):
    return ((a[0] * b[0] - a[1] * b[1]) % p, (a[0] * b[1] + a[1] * b[0]) % p)


def fq2_pow(a, e, p):
    acc = (1, 0)
    for bit in bin(e)[2:]:
        acc = fq2_mul(acc, acc, p)
        if bit == "1":
            acc = fq2_mul(acc, a, p)
    return acc


def pairing_consts(cname, c):
    """Constants of the optimal-ate pairing over the tower Fq2 = Fq[u]/(u^2 + 1), Fq6 = Fq2[v]/(v^3 - xi),
    Fq12 = Fq6[w]/(w^2 - v) (pairing.cuh): xi, the twist's 3 b', the Frobenius coefficients, the Miller loop scalar and the
    joint base-p digits of the hard part of the final exponentiation."""
    p, r = c["p"], c["r"]
    xi0 = 1 if cname == "bls12_381" else 9
    xi = (xi0, 1)
    if cname == "bls12_381":      # M-type twist y^2 = x^3 + b xi
        b2 = (4 * xi[0] % p, 4 * xi[1] % p)
        loop, neg, frob = BLS_X, 1, 0
    else:                         # D-type twist y^2 = x^3 + b / xi
        n = pow(xi0 * xi0 + 1, -1, p)
        b2 = (3 * xi0 * n % p, (-3 * n) % p)
        loop, neg, frob = 6 * BN_U + 2, 0, 1
    assert (p - 1) % 6 == 0
    # a^(p^k) of c0 + c1 v + c2 v^2 scales c1 by xi^((p^k - 1) / 3) and c2 by xi^(2 (p^k - 1) / 3); of c0 + c1 w scales c1 by
    # xi^((p^k - 1) / 6)
    frob_tab = []
    for k in (1, 2, 3):
        e = p ** k - 1
        frob_tab += [fq2_pow(xi, e // 3, p), fq2_pow(xi, 2 * e // 3, p), fq2_pow(xi, e // 6, p)]
    # pi on the D-type twist: (x, y) -> (conj(x) xi^((p - 1) / 3), conj(y) xi^((p - 1) / 2))
    tw_x, tw_y = fq2_pow(xi, (p - 1) // 3, p), fq2_pow(xi, (p - 1) // 2, p)
    # hard part: e = (p^4 - p^2 + 1) / r exactly, as sum lambda_i p^i with 0 <= lambda_i < p; digit j packs bit j of lambda_i
    # at bit i
    hard = (p ** 4 - p ** 2 + 1)
    assert hard % r == 0
    hard //= r
    lam = [(hard // p ** i) % p for i in range(4)]
    assert sum(l * p ** i for i, l in enumerate(lam)) == hard
    bits = max(l.bit_length() for l in lam)
    digits = [sum(((lam[i] >> j) & 1) << i for i in range(4)) for j in range(bits)]
    words = [sum(digits[j] << (4 * (j - 8 * w)) for j in range(8 * w, min(8 * w + 8, bits))) for w in range((bits + 7) // 8)]
    return dict(xi0=xi0, twist_m=1 if cname == "bls12_381" else 0, b3=(3 * b2[0] % p, 3 * b2[1] % p), frob=frob_tab,
                tw_x=tw_x, tw_y=tw_y, loop=loop, loop_neg=neg, loop_frob=frob, hard_bits=bits, hard_words=words)


def check_curve(c):
    p, r = c["p"], c["r"]
    gx, gy = c["gx"] % p, c["gy"] % p
    assert (gy * gy - gx * gx * gx - c["b"]) % p == 0, "generator not on curve"
    assert pow(c["fr_gen"], (r - 1) // 2, r) == r - 1, "fr_gen is a square"
    assert (r - 1) % (1 << c["two_adicity"]) == 0 and ((r - 1) >> c["two_adicity"]) & 1


def cuh_field(name, fc, extra=""):
    n = fc["n32"]
    def arr(fn, v):
        return (f"  PCGPU_HD static constexpr uint32_t {fn}(int i) {{\n"
                f"    constexpr uint32_t v[{n}] = {{{fmt(limbs(v, n, 32), 32)}}};\n"
                f"    return v[i];\n  }}\n")
    s = f"struct {name} {{\n  static constexpr int N = {n};\n  static constexpr int BITS = {fc['bits']};\n"
    s += f"  static constexpr uint32_t M0 = 0x{fc['m0_32']:08x}u;\n"
    s += arr("mod", fc["mod"]) + arr("one", fc["R"]) + arr("r2", fc["R2"])
    s += extra + "};\n\n"
    return s


def c_field(name, fc, extra=""):
    n = fc["n64"]
    s = f"static const uint64_t {name}_MOD[{n}] = {{{fmt(limbs(fc['mod'], n, 64), 64)}}};\n"
    s += f"static const uint64_t {name}_ONE[{n}] = {{{fmt(limbs(fc['R'], n, 64), 64)}}};\n"
    s += f"static const uint64_t {name}_R2[{n}] = {{{fmt(limbs(fc['R2'], n, 64), 64)}}};\n"
    s += f"#define {name}_M0 0x{fc['m0_64']:016x}ull\n#define {name}_N {n}\n#define {name}_BITS {fc['bits']}\n"
    return s + extra + "\n"


def main():
    cuh = ["// GENERATED by tools/gen_params.py -- do not edit.\n#pragma once\n#include <stdint.h>\n"
           "#ifndef PCGPU_HD\n#ifdef __CUDACC__\n#define PCGPU_HD __host__ __device__ __forceinline__\n"
           "#else\n#define PCGPU_HD inline\n#endif\n#endif\n\nnamespace pcgpu {\n\n"]
    ch = ["/* GENERATED by tools/gen_params.py -- do not edit. */\n#pragma once\n#include <stdint.h>\n\n"]
    for cname, c in CURVES.items():
        check_curve(c)
        fq, fr = field_consts(c["p"]), field_consts(c["r"])
        p, r = c["p"], c["r"]
        Rq, Rr = fq["R"], fr["R"]
        gx, gy = c["gx"] % p, c["gy"] % p
        root = pow(c["fr_gen"], (r - 1) >> c["two_adicity"], r)
        CN = "".join(w.capitalize() for w in cname.split("_"))
        n = fq["n32"]
        def arrq(fn, v, n=n):
            return (f"  PCGPU_HD static constexpr uint32_t {fn}(int i) {{\n"
                    f"    constexpr uint32_t v[{n}] = {{{fmt(limbs(v, n, 32), 32)}}};\n    return v[i];\n  }}\n")
        extra_q = arrq("curve_b", c["b"] * Rq % p) + arrq("gen_x", gx * Rq % p) + arrq("gen_y", gy * Rq % p)
        extra_q += f"  static constexpr uint32_t CURVE_B_SMALL = {c['b']};\n"
        sq = sqrt_consts(p)
        extra_q += (f"  // wire formats (wire.cuh): square root, sign comparison and subgroup-check constants\n"
                    f"  static constexpr int SQRT_TONELLI = {sq['ts']};\n  static constexpr int FQ_TWO_ADICITY = {sq['s']};\n"
                    f"  static constexpr int SQRT_EXP_BITS = {sq['exp'].bit_length()};\n")
        extra_q += arrq("sqrt_exp", sq["exp"]) + arrq("ts_root", sq["root"] * Rq % p) + arrq("half", (p - 1) // 2)
        if cname == "bls12_381":
            # sigma(x, y) = (beta x, y) acts on G1 as multiplication by an eigenvalue; pick the cube root of unity for which
            # sigma(P) = -[z^2] P on the prime-order subgroup (the test of ark-bls12-381's subgroup check)
            G = (gx, gy)
            t = ec_mul(BLS_X * BLS_X, G, p)
            target = (t[0], (-t[1]) % p)
            cands = [b for b in (pow(2, (p - 1) // 3, p), pow(2, 2 * (p - 1) // 3, p)) if b != 1]
            beta = [b for b in cands if ((b * gx) % p, gy) == target]
            assert len(beta) == 1 and ec_mul(r, G, p) is None
            extra_q += arrq("beta", beta[0] * Rq % p)
            extra_q += f"  static constexpr unsigned long long SUBGROUP_X = 0x{BLS_X:x}ull;\n  static constexpr int COFACTOR_ONE = 0;\n"
        else:
            assert ec_mul(r, (gx, gy), p) is None
            extra_q += arrq("beta", 0) + "  static constexpr unsigned long long SUBGROUP_X = 0ull;\n  static constexpr int COFACTOR_ONE = 1;\n"
        nr = fr["n32"]
        extra_r = arrq("root_of_unity", root * Rr % r, nr) + f"  static constexpr int TWO_ADICITY = {c['two_adicity']};\n"
        if cname in ("bls12_381", "bn254"):
            pc = pairing_consts(cname, c)

            def arrq2(fn, vals):
                """Fq2 constants, Montgomery: entry j holds c0 in words 0..N-1 and c1 in words N..2N-1"""
                rows = ["{" + fmt(limbs(v[0] * Rq % p, n, 32) + limbs(v[1] * Rq % p, n, 32), 32) + "}" for v in vals]
                return (f"  PCGPU_HD static constexpr uint32_t {fn}(int j, int i) {{\n"
                        f"    constexpr uint32_t v[{len(vals)}][{2 * n}] = {{{', '.join(rows)}}};\n    return v[j][i];\n  }}\n")
            lw = [(pc["loop"] >> (32 * i)) & 0xFFFFFFFF for i in range((pc["loop"].bit_length() + 31) // 32)]
            extra_q += ("  // optimal-ate pairing (pairing.cuh): xi = XI0 + u; TWIST_M: M-type twist (else D-type)\n"
                        f"  static constexpr int XI0 = {pc['xi0']};\n  static constexpr int TWIST_M = {pc['twist_m']};\n")
            extra_q += "  // 3 b' of the twist\n" + arrq2("twist_b3", [pc["b3"]])
            extra_q += ("  // Frobenius a^(p^k), k = 1, 2, 3: entry 3 (k - 1) + 0 / 1 scales Fq6's v / v^2 coefficient, + 2 scales Fq12's w"
                        " coefficient\n") + arrq2("frob", pc["frob"])
            extra_q += "  // pi on the twist: x scales by entry 0, y by entry 1 (after conjugation)\n" + arrq2("twist_frob", [pc["tw_x"], pc["tw_y"]])
            extra_q += (f"  // Miller loop scalar (|x| for BLS12-381, 6u + 2 for BN254), its bit length, 32-bit words low first\n"
                        f"  static constexpr int MILLER_BITS = {pc['loop'].bit_length()};\n"
                        f"  static constexpr int MILLER_NEG = {pc['loop_neg']};\n  static constexpr int MILLER_FROB = {pc['loop_frob']};\n"
                        f"  PCGPU_HD static constexpr uint32_t miller_loop(int i) {{\n"
                        f"    constexpr uint32_t v[{len(lw)}] = {{{fmt(lw, 32)}}};\n    return v[i];\n  }}\n")
            hw = pc["hard_words"]
            extra_q += (f"  // hard part (p^4 - p^2 + 1) / r = sum_i lambda_i p^i: 4-bit digit j (8 per word) has bit i = bit j of lambda_i\n"
                        f"  static constexpr int HARD_BITS = {pc['hard_bits']};\n"
                        f"  PCGPU_HD static constexpr uint32_t hard_digits(int i) {{\n"
                        f"    constexpr uint32_t v[{len(hw)}] = {{{fmt(hw, 32)}}};\n    return v[i];\n  }}\n")
        gl = glv_consts(c)
        extra_q += "  // GLV endomorphism phi(x, y) = (glv_zeta x, y) = [glv_lambda] (x, y)  (ipa.cuh key folding)\n" + arrq("glv_zeta", gl["zeta"] * Rq % p)
        extra_r += "  // GLV: lambda (Montgomery) and the lattice basis |a1|, |b1|, |a2|, |b2| (128-bit magnitudes) with their signs\n"
        extra_r += arrq("glv_lambda", gl["lam"] * Rr % r, nr)
        for nm, v in (("glv_a1", gl["v1"][0]), ("glv_b1", gl["v1"][1]), ("glv_a2", gl["v2"][0]), ("glv_b2", gl["v2"][1])):
            extra_r += arrq(nm, abs(v), 4) + f"  static constexpr int {nm.upper()}_NEG = {1 if v < 0 else 0};\n"
        cuh.append(cuh_field(f"{CN}Fq", fq, extra_q))
        cuh.append(cuh_field(f"{CN}Fr", fr, extra_r))
        U = cname.upper()
        nq64, nr64 = fq["n64"], fr["n64"]
        eq = (f"static const uint64_t {U}_FQ_B[{nq64}] = {{{fmt(limbs(c['b'] * Rq % p, nq64, 64), 64)}}};\n"
              f"static const uint64_t {U}_FQ_GX[{nq64}] = {{{fmt(limbs(gx * Rq % p, nq64, 64), 64)}}};\n"
              f"static const uint64_t {U}_FQ_GY[{nq64}] = {{{fmt(limbs(gy * Rq % p, nq64, 64), 64)}}};\n")
        er = (f"static const uint64_t {U}_FR_ROOT[{nr64}] = {{{fmt(limbs(root * Rr % r, nr64, 64), 64)}}};\n"
              f"#define {U}_FR_TWO_ADICITY {c['two_adicity']}\n")
        ch.append(c_field(f"{U}_FQ", fq, eq))
        ch.append(c_field(f"{U}_FR", fr, er))
    cuh.append("}  // namespace pcgpu\n")
    open(os.path.join(ROOT, "poly-commit_b200", "csrc", "params_gen.cuh"), "w").write("".join(cuh))
    open(os.path.join(ROOT, "oracle", "params_gen.h"), "w").write("".join(ch))
    print("ok")


if __name__ == "__main__":
    main()
