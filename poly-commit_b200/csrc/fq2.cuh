// Quadratic extension Fq2 = Fq[u] / (u^2 + 1) over the device prime field (fp.cuh): the coordinate field of G2 on the
// BLS12-381 and BN254 twists.  An element is (c0, c1) = c0 + c1 u, both Montgomery Fp<P>, c0 first -- the byte image of
// ark-ff's QuadExtField { c0, c1 } and of the ABI's G2 coordinates (g2_host.py).
//
// The operations are overloads of the fp_* names, so the point formulas of ec.cuh run unchanged on either coordinate field
// (a call fp_mul<Q>(a, b) picks the Fq2 overload when a and b are Fq2<Q>).
//   product  c0 = a0 b0 + a1 (-b1), c1 = a0 b1 + a1 b0: one sum-of-products reduction each (mont_mul2 needs 3p < 2^(32N),
//            true for both base fields here): 4 products, 2 reductions
//   square   c0 = (a0 + a1)(a0 - a1), c1 = 2 a0 a1: 2 products
//   inverse  through the norm a0^2 + a1^2 and one Fq inversion; the inverse of 0 is 0
#pragma once
#include "fp.cuh"

namespace pcgpu {

template <class P>
struct Fq2 {
  Fp<P> c0, c1;
  static constexpr int WORDS = 2 * P::N;
  PCGPU_HD static Fq2 zero() { Fq2 r; r.c0 = Fp<P>::zero(); r.c1 = Fp<P>::zero(); return r; }
  PCGPU_HD static Fq2 one() { Fq2 r; r.c0 = Fp<P>::one(); r.c1 = Fp<P>::zero(); return r; }
  PCGPU_HD bool is_zero() const { return c0.is_zero() && c1.is_zero(); }
  PCGPU_HD bool operator==(const Fq2 &b) const { return c0 == b.c0 && c1 == b.c1; }
  PCGPU_HD bool operator!=(const Fq2 &b) const { return !(*this == b); }
};

// 32-bit word j of a coordinate in its packed layout (c0 words, then c1 words); j is a compile-time constant after unrolling
template <class P> PCGPU_DEV uint32_t &coord_word(Fp<P> &a, int j) { return a.l[j]; }
template <class P> PCGPU_DEV uint32_t coord_word(const Fp<P> &a, int j) { return a.l[j]; }
template <class P> PCGPU_DEV uint32_t &coord_word(Fq2<P> &a, int j) { return j < P::N ? a.c0.l[j] : a.c1.l[j - P::N]; }
template <class P> PCGPU_DEV uint32_t coord_word(const Fq2<P> &a, int j) { return j < P::N ? a.c0.l[j] : a.c1.l[j - P::N]; }
template <class F> PCGPU_HD constexpr int coord_words() { return (int)(sizeof(F) / 4); }

template <class P> PCGPU_DEV Fq2<P> fp_add(const Fq2<P> &a, const Fq2<P> &b) { Fq2<P> r; r.c0 = fp_add<P>(a.c0, b.c0); r.c1 = fp_add<P>(a.c1, b.c1); return r; }
template <class P> PCGPU_DEV Fq2<P> fp_sub(const Fq2<P> &a, const Fq2<P> &b) { Fq2<P> r; r.c0 = fp_sub<P>(a.c0, b.c0); r.c1 = fp_sub<P>(a.c1, b.c1); return r; }
template <class P> PCGPU_DEV Fq2<P> fp_neg(const Fq2<P> &a) { Fq2<P> r; r.c0 = fp_neg<P>(a.c0); r.c1 = fp_neg<P>(a.c1); return r; }
template <class P> PCGPU_DEV Fq2<P> fp_cneg(const Fq2<P> &a, bool neg) { Fq2<P> r; r.c0 = fp_cneg<P>(a.c0, neg); r.c1 = fp_cneg<P>(a.c1, neg); return r; }
template <class P> PCGPU_DEV Fq2<P> fp_dbl(const Fq2<P> &a) { return fp_add<P>(a, a); }
template <class P> PCGPU_DEV Fq2<P> fp_mul3(const Fq2<P> &a) { return fp_add<P>(fp_dbl<P>(a), a); }

template <class P>
PCGPU_DEV Fq2<P> fp_mul(const Fq2<P> &a, const Fq2<P> &b) {
  Fq2<P> r;
  r.c0 = fp_mul2<P>(a.c0, b.c0, a.c1, fp_neg<P>(b.c1));
  r.c1 = fp_mul2<P>(a.c0, b.c1, a.c1, b.c0);
  return r;
}

template <class P>
PCGPU_DEV Fq2<P> fp_sqr(const Fq2<P> &a) {
  Fq2<P> r;
  const Fp<P> t = fp_mul<P>(a.c0, a.c1);
  r.c0 = fp_mul<P>(fp_add<P>(a.c0, a.c1), fp_sub<P>(a.c0, a.c1));
  r.c1 = fp_dbl<P>(t);
  return r;
}

// a*b + c*d
template <class P>
PCGPU_DEV Fq2<P> fp_mul2(const Fq2<P> &a, const Fq2<P> &b, const Fq2<P> &c, const Fq2<P> &d) {
  return fp_add<P>(fp_mul<P>(a, b), fp_mul<P>(c, d));
}

template <class P>
PCGPU_DEV Fq2<P> fp_inv(const Fq2<P> &a) {
  const Fp<P> t = fp_inv<P>(fp_mul2<P>(a.c0, a.c0, a.c1, a.c1));   // 1 / (a0^2 + a1^2); 0 for a = 0
  Fq2<P> r;
  r.c0 = fp_mul<P>(a.c0, t);
  r.c1 = fp_neg<P>(fp_mul<P>(a.c1, t));
  return r;
}

}  // namespace pcgpu
