// Device-resident state and kernels for the InnerProductArgPC::open halving loop
// (ipa_pc/mod.rs:665-711): per round two MSMs over the current (folded) key halves, two inner products,
// the folds  coeffs_l += chal^-1 coeffs_r,  z_l += chal z_r,  key_l[i] += chal * key_r[i]  followed by
// normalize_batch (:699-707).  The Fiat-Shamir hash between rounds stays on the host (it consumes two affine
// points and produces one scalar); everything O(n) stays in HBM across the 18 rounds of cfg3.
#pragma once
#include "frops.cuh"
#include "msm.cuh"

namespace pcgpu {

// out[i] = z^i (ipa_pc/mod.rs:643-648)
template <class R>
struct FrPowersBody {
  const uint32_t *z; uint32_t *out;
  PCGPU_KERNEL_DEV void operator()(size_t i) const {
    Fp<R> acc = Fp<R>::one(), base = load_fr<R>(z, 0);
    size_t e = i;
    while (e) { if (e & 1) acc = fp_mul<R>(acc, base); base = fp_sqr<R>(base); e >>= 1; }
    store_fr<R>(out, i, acc);
  }
};

// key[i] = affine(key[i] + chal * key[i + m])   -- k_l += k_r.mul(chal); normalize_batch  (:699-707)
// projective -> affine with the binary-GCD inverse (fp_inv_gcd runs on the ALU pipe, which idles while the ladders of the
// other warps saturate the integer-multiply pipe; the Fermat inverse of xyzz_to_affine costs ~380 more multiplications per point)
template <class C>
PCGPU_DEV Affine<C> xyzz_to_affine_gcd(const XYZZ<C> &p, const uint32_t *pow2) {
  using Q = typename C::Fq;
  if (p.is_inf()) return Affine<C>::inf();
  Fp<Q> inv = fp_inv_gcd<Q>(fp_mul<Q>(p.zz, p.zzz), pow2);
  Affine<C> a;
  a.x = fp_mul<Q>(p.x, fp_mul<Q>(inv, p.zzz));
  a.y = fp_mul<Q>(p.y, fp_mul<Q>(inv, p.zz));
  return a;
}

template <class C>
struct G1FoldBody {
  Affine<C> *key; uint32_t m; uint32_t chal[8];  // canonical scalar, same for every point
  const uint32_t *pow2;
  PCGPU_KERNEL_DEV void operator()(size_t i) const {
    Affine<C> r = load_affine<C>(key + m + i);
    XYZZ<C> acc = XYZZ<C>::inf();
    for (int b = 255; b >= 0; b--) {
      acc = xyzz_dbl<C>(acc);
      if ((chal[b >> 5] >> (b & 31)) & 1) xyzz_madd<C>(acc, r, false);
    }
    Affine<C> l = load_affine<C>(key + i);
    xyzz_madd<C>(acc, l, false);
    key[i] = xyzz_to_affine_gcd<C>(acc, pow2);
  }
};

// The same fold through the GLV endomorphism (curves with cofactor 1: Pallas, BN254): chal = k1 + k2 lambda with ~128-bit
// k1, k2 (host_glv.hpp), chal * R = k1 * R + k2 * phi(R), phi(x, y) = (zeta x, y) -- one joint ladder of <= 133 columns in
// JOINT SPARSE FORM over {P1 = +-R, P2 = +-phi(R), P1 + P2, P1 - P2} instead of 256 steps over {R}: half of the columns are
// (0, 0) on average (the plain binary joint ladder adds in three columns of four), and all four table points are AFFINE --
// P1 + P2 and P1 - P2 share the denominator x2 - x1, so one binary-GCD inverse yields both -- so every addition is a mixed one.
// Every thread runs the same scalar, so the ladder's control flow is uniform across the grid.
template <class C>
struct G1FoldGlvBody {
  Affine<C> *key; uint32_t m; uint32_t u1_nz[5], u1_sg[5], u2_nz[5], u2_sg[5]; uint32_t neg1, neg2, ncols;
  const uint32_t *pow2;
  PCGPU_KERNEL_DEV void operator()(size_t i) const {
    using Q = typename C::Fq;
    Affine<C> r = load_affine<C>(key + m + i);
    Affine<C> l = load_affine<C>(key + i);
    if (r.is_inf()) { key[i] = l; return; }
    Fp<Q> zeta;
    for (int j = 0; j < Q::N; j++) zeta.l[j] = Q::glv_zeta(j);
    Affine<C> p1 = r, p2, ps, pd;
    p1.y = fp_cneg<Q>(r.y, neg1 != 0);
    p2.x = fp_mul<Q>(r.x, zeta); p2.y = fp_cneg<Q>(r.y, neg2 != 0);
    {   // P1 + P2 and P1 - P2 (x2 != x1 for R != O: phi has no fixed point in a group of prime order)
      const Fp<Q> inv = fp_inv_gcd<Q>(fp_sub<Q>(p2.x, p1.x), pow2);
      const Fp<Q> xsum = fp_add<Q>(p1.x, p2.x);
      Fp<Q> lam = fp_mul<Q>(fp_sub<Q>(p2.y, p1.y), inv);
      ps.x = fp_sub<Q>(fp_sqr<Q>(lam), xsum);
      ps.y = fp_sub<Q>(fp_mul<Q>(lam, fp_sub<Q>(p1.x, ps.x)), p1.y);
      lam = fp_mul<Q>(fp_sub<Q>(fp_neg<Q>(p2.y), p1.y), inv);
      pd.x = fp_sub<Q>(fp_sqr<Q>(lam), xsum);
      pd.y = fp_sub<Q>(fp_mul<Q>(lam, fp_sub<Q>(p1.x, pd.x)), p1.y);
    }
    XYZZ<C> acc = XYZZ<C>::inf();
    for (int b = (int)ncols - 1; b >= 0; b--) {
      acc = xyzz_dbl<C>(acc);
      const uint32_t w = (uint32_t)b >> 5, sh = (uint32_t)b & 31;
      const bool n1 = (u1_nz[w] >> sh) & 1, n2 = (u2_nz[w] >> sh) & 1, s1 = (u1_sg[w] >> sh) & 1, s2 = (u2_sg[w] >> sh) & 1;
      if (!(n1 || n2)) continue;
      // the table point is SELECTED (register moves) and added at ONE call site: with an addition inlined per case the loop
      // body outgrows the instruction cache
      Affine<C> a = p1;
      bool neg = s1;
      if (n1 && n2) { if (s1 == s2) a = ps; else a = pd; }      // +-(P1 + P2) / +-(P1 - P2): the sign is u1's
      else if (n2) { a = p2; neg = s2; }
      xyzz_madd<C>(acc, a, neg);
    }
    xyzz_madd<C>(acc, l, false);
    key[i] = xyzz_to_affine_gcd<C>(acc, pow2);
  }
};

// ---- late rounds on a FROZEN key ------------------------------------------------------------------------------------------
// Once the key has been folded down to M <= SMALL_MAX_N points it is not folded any further.  The key of a later round of
// logical size n_t is  key_t[i] = sum_{j = i (mod n_t)} w[j] * B[j]  over the frozen points B, where w[j] is the product of the
// round challenges selected by the bits of j above log2(n_t) (the first challenge after the freeze on the top bit -- the
// coefficient structure of SuccinctCheckPolynomial, ipa_pc/data_structures.rs:204-220).  Hence
//   l_t = cm_commit(key_l, coeffs_r) = sum_j [ (j mod n_t) <  n_t/2 ] w[j] coeffs[(j mod n_t) + n_t/2] * B[j]
//   r_t = cm_commit(key_r, coeffs_l) = sum_j [ (j mod n_t) >= n_t/2 ] w[j] coeffs[(j mod n_t) - n_t/2] * B[j]
// are two M-term MSMs that run in ONE launch of the small-MSM kernel, the fold of the key (ipa_pc/mod.rs:699-707) becomes
// M field multiplications on w, and final_comm_key = sum_j w[j] B[j].  Same group elements as the reference's explicit
// folds; what disappears are the 128-step scalar-multiplication ladders of the twelve latency-bound late rounds.
template <class R>
struct IpaFrozenScalarsBody {   // s_l[j], s_r[j] (Montgomery) from w, coeffs and the logical size n_t
  const uint32_t *w, *coeffs; uint32_t n_t; uint32_t *s_l, *s_r;
  PCGPU_KERNEL_DEV void operator()(size_t j) const {
    const uint32_t i = (uint32_t)j & (n_t - 1), half = n_t >> 1;
    const Fp<R> wj = load_fr<R>(w, j);
    const bool left = i < half;
    const Fp<R> v = fp_mul<R>(wj, load_fr<R>(coeffs, left ? i + half : i - half));
    store_fr<R>(s_l, j, left ? v : Fp<R>::zero());
    store_fr<R>(s_r, j, left ? Fp<R>::zero() : v);
  }
};
template <class R>
struct IpaFrozenWeightBody {    // the fold of a frozen key: w[j] *= chal for the j in the right half of their period n_t
  uint32_t *w; const uint32_t *chal; uint32_t n_t;
  PCGPU_KERNEL_DEV void operator()(size_t j) const {
    if (((uint32_t)j & (n_t - 1)) >= (n_t >> 1)) store_fr<R>(w, j, fp_mul<R>(load_fr<R>(w, j), load_fr<R>(chal, 0)));
  }
};
template <class R>
struct FrFillOneBody {
  uint32_t *out;
  PCGPU_KERNEL_DEV void operator()(size_t j) const { store_fr<R>(out, j, Fp<R>::one()); }
};

// SuccinctCheckPolynomial::compute_coeffs (ipa_pc/data_structures.rs:204-220): coeffs[idx] = product of challenge_i over
// the set bits of idx, challenge_1 on the top bit.  One thread per coefficient (<= log_d multiplications).
template <class R>
struct FrCheckCoeffsBody {
  const uint32_t *challenges; uint32_t log_d; uint32_t *out;
  PCGPU_KERNEL_DEV void operator()(size_t idx) const {
    Fp<R> acc = Fp<R>::one();
    for (uint32_t i = 1; i <= log_d; i++)
      if ((idx >> (log_d - i)) & 1) acc = fp_mul<R>(acc, load_fr<R>(challenges, i - 1));
    store_fr<R>(out, idx, acc);
  }
};

}  // namespace pcgpu
