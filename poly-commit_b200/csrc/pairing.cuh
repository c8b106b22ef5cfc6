// The optimal-ate pairing of BLS12-381 and BN254 on the device: E::multi_pairing of the reference's verifiers
// (kzg10/mod.rs:326-330, :382-387; multilinear_pc/mod.rs:179-199).
//
// Tower (ark-ff's):  Fq2 = Fq[u]/(u^2 + 1) (fq2.cuh),  Fq6 = Fq2[v]/(v^3 - xi),  Fq12 = Fq6[w]/(w^2 - v),  xi = XI0 + u
// (1 + u on BLS12-381, 9 + u on BN254).  An Fq12 element's words are c0.c0.c0, c0.c0.c1, c0.c1.c0 ... c1.c2.c1, each N words
// Montgomery: the byte image of ark's QuadExtField<Fp6> and of the ABI's GT elements.  Frobenius coefficients come from
// tools/gen_params.py (params_gen.cuh).
//
// Miller loop, one thread per pair: T runs in homogeneous projective coordinates on the twist y^2 = x^3 + b'.  Every line
// through untwisted points, evaluated at P, is scaled by factors the final exponentiation maps to 1 (elements of Fq2 and, on
// the M-type twist, w^3), so it has three non-zero Fq2 coefficients:
//   D-type (BN254, psi(x, y) = (x w^2, y w^3)):      ell0 yP + ell1 xP w + ell2 w^3        slots 0, 3, 4 (c0.c0, c1.c0, c1.c1)
//   M-type (BLS12-381, psi(x, y) = (x/w^2, y/w^3)):  ell2 + ell1 xP w^2 + ell0 yP w^3      slots 0, 1, 4 (c0.c0, c0.c1, c1.c1)
// with (ell0, ell1, ell2) = (-2YZ, 3X^2, 3b'Z^2 - Y^2) for the tangent at T and (X - xq Z, -(Y - yq Z), theta xq - lambda yq)
// for the chord through T and Q.  Vertical lines are dropped (the final exponentiation maps them to 1).
//   BLS12-381: the loop runs over |x| = 0xd201000000010000, then f is conjugated (x < 0).
//   BN254: the loop runs over 6u + 2, then the lines through pi(Q) and -pi^2(Q).
// A fixed Q can be prepared once (ark's G2Prepared): G2PrepareBody walks the same loop with the same step functions and stores
// every line; MillerPreparedBody then only squares f and folds the stored lines in at P.
// Final exponentiation, one thread per equation: f^((p^6 - 1)(p^2 + 1)) by conjugation, inversion and Frobenius, then the hard
// part (p^4 - p^2 + 1) / r exactly -- not a multiple of it, so GT values are those of the definition -- as
// prod_i (f^(p^i))^lambda_i over the base-p digits lambda_i of the exponent, one joint square-and-multiply over a table of the
// 15 products of the four Frobenius images.
//
// Compile size: the Fq6 / Fq12 products and the Miller steps are out-of-line functions (__noinline__); inlined, the 12-limb
// BLS12-381 products would multiply into a kernel that takes minutes to compile and does not fit the instruction cache.
#pragma once
#include "ec.cuh"
#include "rt.cuh"

#ifdef __CUDACC__
#define PCGPU_DEV_OUTLINE __device__ __noinline__
#else
#define PCGPU_DEV_OUTLINE inline
#endif

namespace pcgpu {

template <class P> struct Fq6 { Fq2<P> c0, c1, c2; };
template <class P>
struct Fq12 {
  Fq6<P> c0, c1;
  static constexpr int WORDS = 12 * P::N;
  PCGPU_DEV static Fq12 one() {
    Fq12 r;
    r.c0.c0 = Fq2<P>::one(); r.c0.c1 = r.c0.c2 = r.c1.c0 = r.c1.c1 = r.c1.c2 = Fq2<P>::zero();
    return r;
  }
  // Fq2 coefficient s in ark order (0..5: c0.c0, c0.c1, c0.c2, c1.c0, c1.c1, c1.c2)
  PCGPU_DEV Fq2<P> &slot(int s) {
    Fq6<P> &h = s < 3 ? c0 : c1;
    const int t = s % 3;
    return t == 0 ? h.c0 : (t == 1 ? h.c1 : h.c2);
  }
  PCGPU_DEV bool is_one() const {
    return c0.c0 == Fq2<P>::one() && c0.c1.is_zero() && c0.c2.is_zero() && c1.c0.is_zero() && c1.c1.is_zero() && c1.c2.is_zero();
  }
};

template <class P> PCGPU_DEV void fq12_load(Fq12<P> &a, const uint32_t *src) {
#pragma unroll
  for (int s = 0; s < 6; s++)
#pragma unroll
    for (int j = 0; j < 2 * P::N; j++) coord_word(a.slot(s), j) = src[s * 2 * P::N + j];
}
template <class P> PCGPU_DEV void fq12_store(uint32_t *dst, Fq12<P> a) {
#pragma unroll
  for (int s = 0; s < 6; s++)
#pragma unroll
    for (int j = 0; j < 2 * P::N; j++) dst[s * 2 * P::N + j] = coord_word(a.slot(s), j);
}

// ---- Fq2 helpers -------------------------------------------------------------------------------------------------------
// generated Fq2 constants (params_gen.cuh)
#define PCGPU_FQ2_CONST(NAME)                                                         \
  template <class P> PCGPU_DEV Fq2<P> NAME##_const(int j) {                           \
    Fq2<P> r;                                                                         \
    _Pragma("unroll") for (int i = 0; i < 2 * P::N; i++) coord_word(r, i) = P::NAME(j, i); \
    return r;                                                                         \
  }
PCGPU_FQ2_CONST(frob)
PCGPU_FQ2_CONST(twist_b3)
PCGPU_FQ2_CONST(twist_frob)
#undef PCGPU_FQ2_CONST
template <class P> PCGPU_DEV Fq2<P> fq2_conj(const Fq2<P> &a) { Fq2<P> r; r.c0 = a.c0; r.c1 = fp_neg<P>(a.c1); return r; }
template <class P> PCGPU_DEV Fq2<P> fq2_mul_fp(const Fq2<P> &a, const Fp<P> &s) { Fq2<P> r; r.c0 = fp_mul<P>(a.c0, s); r.c1 = fp_mul<P>(a.c1, s); return r; }
template <class P> PCGPU_DEV Fp<P> fp_mul_xi0(const Fp<P> &a) {
  static_assert(P::XI0 == 1 || P::XI0 == 9, "xi = 1 + u or 9 + u");
  if constexpr (P::XI0 == 1) return a;
  else return fp_add<P>(fp_dbl<P>(fp_dbl<P>(fp_dbl<P>(a))), a);
}
// a * xi = (XI0 a0 - a1) + (XI0 a1 + a0) u
template <class P> PCGPU_DEV Fq2<P> fq2_mul_xi(const Fq2<P> &a) {
  Fq2<P> r;
  r.c0 = fp_sub<P>(fp_mul_xi0<P>(a.c0), a.c1);
  r.c1 = fp_add<P>(fp_mul_xi0<P>(a.c1), a.c0);
  return r;
}

// ---- Fq6 -----------------------------------------------------------------------------------------------------------------
template <class P> PCGPU_DEV Fq6<P> fq6_add(const Fq6<P> &a, const Fq6<P> &b) {
  return Fq6<P>{fp_add<P>(a.c0, b.c0), fp_add<P>(a.c1, b.c1), fp_add<P>(a.c2, b.c2)};
}
template <class P> PCGPU_DEV Fq6<P> fq6_sub(const Fq6<P> &a, const Fq6<P> &b) {
  return Fq6<P>{fp_sub<P>(a.c0, b.c0), fp_sub<P>(a.c1, b.c1), fp_sub<P>(a.c2, b.c2)};
}
template <class P> PCGPU_DEV Fq6<P> fq6_neg(const Fq6<P> &a) { return Fq6<P>{fp_neg<P>(a.c0), fp_neg<P>(a.c1), fp_neg<P>(a.c2)}; }
template <class P> PCGPU_DEV Fq6<P> fq6_mul_by_v(const Fq6<P> &a) { return Fq6<P>{fq2_mul_xi<P>(a.c2), a.c0, a.c1}; }

// Karatsuba: 6 Fq2 products
template <class P>
PCGPU_DEV_OUTLINE Fq6<P> fq6_mul(const Fq6<P> a, const Fq6<P> b) {
  const Fq2<P> t0 = fp_mul<P>(a.c0, b.c0), t1 = fp_mul<P>(a.c1, b.c1), t2 = fp_mul<P>(a.c2, b.c2);
  Fq6<P> r;
  r.c0 = fp_add<P>(t0, fq2_mul_xi<P>(fp_sub<P>(fp_sub<P>(fp_mul<P>(fp_add<P>(a.c1, a.c2), fp_add<P>(b.c1, b.c2)), t1), t2)));
  r.c1 = fp_add<P>(fp_sub<P>(fp_sub<P>(fp_mul<P>(fp_add<P>(a.c0, a.c1), fp_add<P>(b.c0, b.c1)), t0), t1), fq2_mul_xi<P>(t2));
  r.c2 = fp_add<P>(fp_sub<P>(fp_sub<P>(fp_mul<P>(fp_add<P>(a.c0, a.c2), fp_add<P>(b.c0, b.c2)), t0), t2), t1);
  return r;
}

// a * (b0 + b1 v)
template <class P>
PCGPU_DEV_OUTLINE Fq6<P> fq6_mul_by_01(const Fq6<P> a, const Fq2<P> b0, const Fq2<P> b1) {
  Fq6<P> r;
  r.c0 = fp_add<P>(fp_mul<P>(a.c0, b0), fq2_mul_xi<P>(fp_mul<P>(a.c2, b1)));
  r.c1 = fp_add<P>(fp_mul<P>(a.c0, b1), fp_mul<P>(a.c1, b0));
  r.c2 = fp_add<P>(fp_mul<P>(a.c1, b1), fp_mul<P>(a.c2, b0));
  return r;
}

// a * b1 v
template <class P>
PCGPU_DEV_OUTLINE Fq6<P> fq6_mul_by_1(const Fq6<P> a, const Fq2<P> b1) {
  return Fq6<P>{fq2_mul_xi<P>(fp_mul<P>(a.c2, b1)), fp_mul<P>(a.c0, b1), fp_mul<P>(a.c1, b1)};
}

template <class P>
PCGPU_DEV_OUTLINE Fq6<P> fq6_mul_fq2(const Fq6<P> a, const Fq2<P> s) {
  return Fq6<P>{fp_mul<P>(a.c0, s), fp_mul<P>(a.c1, s), fp_mul<P>(a.c2, s)};
}

// (t0 + t1 v + t2 v^2) / N with t0 = a0^2 - xi a1 a2, t1 = xi a2^2 - a0 a1, t2 = a1^2 - a0 a2, N = a0 t0 + xi (a2 t1 + a1 t2);
// the inverse of 0 is 0
template <class P>
PCGPU_DEV_OUTLINE Fq6<P> fq6_inv(const Fq6<P> a) {
  const Fq2<P> t0 = fp_sub<P>(fp_sqr<P>(a.c0), fq2_mul_xi<P>(fp_mul<P>(a.c1, a.c2)));
  const Fq2<P> t1 = fp_sub<P>(fq2_mul_xi<P>(fp_sqr<P>(a.c2)), fp_mul<P>(a.c0, a.c1));
  const Fq2<P> t2 = fp_sub<P>(fp_sqr<P>(a.c1), fp_mul<P>(a.c0, a.c2));
  const Fq2<P> n = fp_add<P>(fp_mul<P>(a.c0, t0), fq2_mul_xi<P>(fp_add<P>(fp_mul<P>(a.c2, t1), fp_mul<P>(a.c1, t2))));
  const Fq2<P> ni = fp_inv<P>(n);
  return Fq6<P>{fp_mul<P>(t0, ni), fp_mul<P>(t1, ni), fp_mul<P>(t2, ni)};
}

// a^(p^K): conjugate the coefficients K times, scale c1 and c2 by the generated xi powers
template <class P, int K>
PCGPU_DEV Fq6<P> fq6_frob(const Fq6<P> &a) {
  Fq6<P> r = a;
  if (K % 2) { r.c0 = fq2_conj<P>(a.c0); r.c1 = fq2_conj<P>(a.c1); r.c2 = fq2_conj<P>(a.c2); }
  r.c1 = fp_mul<P>(r.c1, frob_const<P>(3 * (K - 1)));
  r.c2 = fp_mul<P>(r.c2, frob_const<P>(3 * (K - 1) + 1));
  return r;
}

// ---- Fq12 ----------------------------------------------------------------------------------------------------------------
template <class P> PCGPU_DEV Fq12<P> fq12_add(const Fq12<P> &a, const Fq12<P> &b) { return Fq12<P>{fq6_add<P>(a.c0, b.c0), fq6_add<P>(a.c1, b.c1)}; }
template <class P> PCGPU_DEV Fq12<P> fq12_sub(const Fq12<P> &a, const Fq12<P> &b) { return Fq12<P>{fq6_sub<P>(a.c0, b.c0), fq6_sub<P>(a.c1, b.c1)}; }
template <class P> PCGPU_DEV Fq12<P> fq12_neg(const Fq12<P> &a) { return Fq12<P>{fq6_neg<P>(a.c0), fq6_neg<P>(a.c1)}; }
// a^(p^6)
template <class P> PCGPU_DEV Fq12<P> fq12_conj(const Fq12<P> &a) { return Fq12<P>{a.c0, fq6_neg<P>(a.c1)}; }

// Karatsuba over Fq6: 3 Fq6 products
template <class P>
PCGPU_DEV_OUTLINE Fq12<P> fq12_mul(const Fq12<P> a, const Fq12<P> b) {
  const Fq6<P> t0 = fq6_mul<P>(a.c0, b.c0), t1 = fq6_mul<P>(a.c1, b.c1);
  Fq12<P> r;
  r.c1 = fq6_sub<P>(fq6_sub<P>(fq6_mul<P>(fq6_add<P>(a.c0, a.c1), fq6_add<P>(b.c0, b.c1)), t0), t1);
  r.c0 = fq6_add<P>(t0, fq6_mul_by_v<P>(t1));
  return r;
}

// complex squaring: c0 = (a0 + a1)(a0 + v a1) - t - v t, c1 = 2 t with t = a0 a1
template <class P>
PCGPU_DEV_OUTLINE Fq12<P> fq12_sqr(const Fq12<P> a) {
  const Fq6<P> t = fq6_mul<P>(a.c0, a.c1);
  const Fq6<P> m = fq6_mul<P>(fq6_add<P>(a.c0, a.c1), fq6_add<P>(a.c0, fq6_mul_by_v<P>(a.c1)));
  Fq12<P> r;
  r.c0 = fq6_sub<P>(fq6_sub<P>(m, t), fq6_mul_by_v<P>(t));
  r.c1 = fq6_add<P>(t, t);
  return r;
}

// Squaring in the cyclotomic subgroup (a^(p^6 + 1) = 1, so a0^2 = 1 + v a1^2): with B = a1^2 and S = (a0 + a1)^2,
// a^2 = (1 + 2 v B) + (S - 1 - v B - B) w -- two Fq6 squarings instead of two Fq6 products and a third for the cross term
template <class P>
PCGPU_DEV_OUTLINE Fq12<P> fq12_cyclotomic_sqr(const Fq12<P> a) {
  const Fq6<P> B = fq6_mul<P>(a.c1, a.c1);
  const Fq6<P> s = fq6_add<P>(a.c0, a.c1);
  const Fq6<P> S = fq6_mul<P>(s, s);
  const Fq6<P> vB = fq6_mul_by_v<P>(B);
  Fq12<P> r;
  r.c0 = fq6_add<P>(vB, vB);
  r.c0.c0 = fp_add<P>(r.c0.c0, Fq2<P>::one());
  r.c1 = fq6_sub<P>(fq6_sub<P>(S, vB), B);
  r.c1.c0 = fp_sub<P>(r.c1.c0, Fq2<P>::one());
  return r;
}

// (a0 - a1 w) / (a0^2 - v a1^2); the inverse of 0 is 0
template <class P>
PCGPU_DEV_OUTLINE Fq12<P> fq12_inv(const Fq12<P> a) {
  const Fq6<P> n = fq6_sub<P>(fq6_mul<P>(a.c0, a.c0), fq6_mul_by_v<P>(fq6_mul<P>(a.c1, a.c1)));
  const Fq6<P> ni = fq6_inv<P>(n);
  return Fq12<P>{fq6_mul<P>(a.c0, ni), fq6_neg<P>(fq6_mul<P>(a.c1, ni))};
}

// a^(p^K), K = 1, 2, 3
template <class P, int K>
PCGPU_DEV_OUTLINE Fq12<P> fq12_frob(const Fq12<P> a) {
  return Fq12<P>{fq6_frob<P, K>(a.c0), fq6_mul_fq2<P>(fq6_frob<P, K>(a.c1), frob_const<P>(3 * (K - 1) + 2))};
}

// f times a line with Fq2 coefficients a, b, c in its three non-zero slots (0, 3, 4 on a D-type twist; 0, 1, 4 on an M-type
// twist); Karatsuba over Fq6 with the sparse factors: 13 Fq2 products
template <class P>
PCGPU_DEV_OUTLINE Fq12<P> fq12_mul_line(const Fq12<P> f, const Fq2<P> a, const Fq2<P> b, const Fq2<P> c) {
  Fq6<P> t0, t1, m;
  if constexpr (P::TWIST_M) {         // L0 = a + b v, L1 = c v
    t0 = fq6_mul_by_01<P>(f.c0, a, b);
    t1 = fq6_mul_by_1<P>(f.c1, c);
    m = fq6_mul_by_01<P>(fq6_add<P>(f.c0, f.c1), a, fp_add<P>(b, c));
  } else {                            // L0 = a, L1 = b + c v
    t0 = fq6_mul_fq2<P>(f.c0, a);
    t1 = fq6_mul_by_01<P>(f.c1, b, c);
    m = fq6_mul_by_01<P>(fq6_add<P>(f.c0, f.c1), fp_add<P>(a, b), c);
  }
  Fq12<P> r;
  r.c1 = fq6_sub<P>(fq6_sub<P>(m, t0), t1);
  r.c0 = fq6_add<P>(t0, fq6_mul_by_v<P>(t1));
  return r;
}

// ---- Miller loop ---------------------------------------------------------------------------------------------------------
template <class P> struct G2Proj { Fq2<P> x, y, z; };
template <class P> struct G2Aff { Fq2<P> x, y; };

// the line at P: its three coefficients scaled by yP / xP and folded into f with the sparse product of the twist
template <class P>
PCGPU_DEV Fq12<P> mul_line_at(const Fq12<P> &f, const Fq2<P> &ell0, const Fq2<P> &ell1, const Fq2<P> &ell2, const Fp<P> &xp,
                              const Fp<P> &yp) {
  if constexpr (P::TWIST_M) return fq12_mul_line<P>(f, ell2, fq2_mul_fp<P>(ell1, xp), fq2_mul_fp<P>(ell0, yp));
  else return fq12_mul_line<P>(f, fq2_mul_fp<P>(ell0, yp), fq2_mul_fp<P>(ell1, xp), ell2);
}

// one Miller line (ell0, ell1, ell2), independent of P
template <class P> struct MillerLine { Fq2<P> ell0, ell1, ell2; };

// T <- 2T and the tangent at T.  (X3 : Y3 : Z3) = (2 X Y (B - F), (B + F)^2 - 12 E^2, 4 B H) with B = Y^2, C = Z^2, E = 3 b' C,
// F = 3 E, H = 2 Y Z: four times the usual doubling, which needs no halving
template <class P>
PCGPU_DEV MillerLine<P> dbl_step(G2Proj<P> &T) {
  const Fq2<P> B = fp_sqr<P>(T.y), C = fp_sqr<P>(T.z);
  const Fq2<P> E = fp_mul<P>(C, twist_b3_const<P>(0));
  const Fq2<P> F = fp_mul3<P>(E);
  const Fq2<P> H = fp_sub<P>(fp_sub<P>(fp_sqr<P>(fp_add<P>(T.y, T.z)), B), C);
  const Fq2<P> ell1 = fp_mul3<P>(fp_sqr<P>(T.x));
  const Fq2<P> ell2 = fp_sub<P>(E, B);
  const Fq2<P> e2 = fp_sqr<P>(E);
  T.x = fp_dbl<P>(fp_mul<P>(fp_mul<P>(T.x, T.y), fp_sub<P>(B, F)));
  T.y = fp_sub<P>(fp_sqr<P>(fp_add<P>(B, F)), fp_dbl<P>(fp_dbl<P>(fp_mul3<P>(e2))));
  T.z = fp_dbl<P>(fp_dbl<P>(fp_mul<P>(B, H)));
  return MillerLine<P>{fp_neg<P>(H), ell1, ell2};
}

// T <- T + Q (Q affine) and the chord through T and Q
template <class P>
PCGPU_DEV MillerLine<P> add_step(G2Proj<P> &T, const G2Aff<P> &Q) {
  const Fq2<P> theta = fp_sub<P>(T.y, fp_mul<P>(Q.y, T.z));
  const Fq2<P> lambda = fp_sub<P>(T.x, fp_mul<P>(Q.x, T.z));
  const Fq2<P> C = fp_sqr<P>(theta), D = fp_sqr<P>(lambda);
  const Fq2<P> E = fp_mul<P>(lambda, D), F = fp_mul<P>(T.z, C), G = fp_mul<P>(T.x, D);
  const Fq2<P> H = fp_sub<P>(fp_add<P>(E, F), fp_dbl<P>(G));
  const Fq2<P> ell2 = fp_sub<P>(fp_mul<P>(theta, Q.x), fp_mul<P>(lambda, Q.y));
  T.x = fp_mul<P>(lambda, H);
  T.y = fp_sub<P>(fp_mul<P>(theta, fp_sub<P>(G, H)), fp_mul<P>(E, T.y));
  T.z = fp_mul<P>(T.z, E);
  return MillerLine<P>{lambda, fp_neg<P>(theta), ell2};
}

// f * line(T, T) at P, T <- 2T
template <class P>
PCGPU_DEV_OUTLINE Fq12<P> miller_dbl(G2Proj<P> &T, const Fq12<P> f, const Fp<P> xp, const Fp<P> yp) {
  const MillerLine<P> l = dbl_step<P>(T);
  return mul_line_at<P>(f, l.ell0, l.ell1, l.ell2, xp, yp);
}

// f * line(T, Q) at P, T <- T + Q (Q affine)
template <class P>
PCGPU_DEV_OUTLINE Fq12<P> miller_add(G2Proj<P> &T, const G2Aff<P> Q, const Fq12<P> f, const Fp<P> xp, const Fp<P> yp) {
  const MillerLine<P> l = add_step<P>(T, Q);
  return mul_line_at<P>(f, l.ell0, l.ell1, l.ell2, xp, yp);
}

// pi on the D-type twist: (conj(x) xi^((p - 1) / 3), conj(y) xi^((p - 1) / 2))
template <class P>
PCGPU_DEV G2Aff<P> twist_frob(const G2Aff<P> &q) {
  return G2Aff<P>{fp_mul<P>(fq2_conj<P>(q.x), twist_frob_const<P>(0)), fp_mul<P>(fq2_conj<P>(q.y), twist_frob_const<P>(1))};
}

// the Miller value of (P, Q); 1 when either is the identity
template <class P>
PCGPU_DEV Fq12<P> miller_loop(const Fp<P> &xp, const Fp<P> &yp, const G2Aff<P> &q) {
  Fq12<P> f = Fq12<P>::one();
  G2Proj<P> T{q.x, q.y, Fq2<P>::one()};
  for (int i = P::MILLER_BITS - 2; i >= 0; i--) {
    f = fq12_sqr<P>(f);
    f = miller_dbl<P>(T, f, xp, yp);
    if ((P::miller_loop(i / 32) >> (i % 32)) & 1) f = miller_add<P>(T, q, f, xp, yp);
  }
  if constexpr (P::MILLER_NEG) f = fq12_conj<P>(f);
  if constexpr (P::MILLER_FROB) {
    const G2Aff<P> q1 = twist_frob<P>(q);
    G2Aff<P> q2 = twist_frob<P>(q1);
    q2.y = fp_neg<P>(q2.y);
    f = miller_add<P>(T, q1, f, xp, yp);
    f = miller_add<P>(T, q2, f, xp, yp);
  }
  return f;
}

// The lines miller_loop folds in for one Q, in its order: one tangent per step, one chord per set bit of the loop scalar
// below the top bit, and the pi(Q) and -pi^2(Q) chords on BN254 -- ark's G2Prepared::ell_coeffs
template <class P>
PCGPU_HD constexpr int miller_line_count() {
  int n = P::MILLER_FROB ? 2 : 0;
  for (int i = P::MILLER_BITS - 2; i >= 0; i--) n += 1 + (int)((P::miller_loop(i / 32) >> (i % 32)) & 1);
  return n;
}
// words of one prepared point: its lines, each ell0 ell1 ell2 as Fq2 Montgomery words
template <class P> PCGPU_HD constexpr size_t prepared_point_words() { return (size_t)miller_line_count<P>() * 6 * P::N; }

template <class P> PCGPU_DEV void line_store(uint32_t *dst, const MillerLine<P> &l) {
#pragma unroll
  for (int j = 0; j < 2 * P::N; j++) {
    dst[j] = coord_word(l.ell0, j); dst[2 * P::N + j] = coord_word(l.ell1, j); dst[4 * P::N + j] = coord_word(l.ell2, j);
  }
}
template <class P> PCGPU_DEV MillerLine<P> line_load(const uint32_t *src) {
  MillerLine<P> l;
#pragma unroll
  for (int j = 0; j < 2 * P::N; j++) {
    coord_word(l.ell0, j) = src[j]; coord_word(l.ell1, j) = src[2 * P::N + j]; coord_word(l.ell2, j) = src[4 * P::N + j];
  }
  return l;
}

// ---- final exponentiation: f^((p^12 - 1) / r) ----------------------------------------------------------------------------
template <class P>
PCGPU_DEV Fq12<P> final_exponentiation(const Fq12<P> &f) {
  Fq12<P> g = fq12_mul<P>(fq12_conj<P>(f), fq12_inv<P>(f));     // f^(p^6 - 1)
  g = fq12_mul<P>(fq12_frob<P, 2>(g), g);                         // ^(p^2 + 1): now in the cyclotomic subgroup
  Fq12<P> tab[16];                                                // tab[m] = prod over the set bits i of m of g^(p^i)
  tab[1] = g;
  tab[2] = fq12_frob<P, 1>(g);
  tab[4] = fq12_frob<P, 2>(g);
  tab[8] = fq12_frob<P, 3>(g);
  for (int m = 3; m < 16; m++)
    if (m & (m - 1)) tab[m] = fq12_mul<P>(tab[m & (m - 1)], tab[m & -m]);
  Fq12<P> acc = Fq12<P>::one();
  for (int j = P::HARD_BITS - 1; j >= 0; j--) {
    acc = fq12_cyclotomic_sqr<P>(acc);
    const uint32_t d = (P::hard_digits(j / 8) >> (4 * (j % 8))) & 15u;
    if (d) acc = fq12_mul<P>(acc, tab[d]);
  }
  return acc;
}

// ---- kernels -------------------------------------------------------------------------------------------------------------
// Miller value of pair i: g1 (x || y) and g2 (x.c0 x.c1 y.c0 y.c1) affine Montgomery words; an identity flag or the all-zero
// encoding makes the pair contribute 1.
template <class P>
struct MillerBody {
  const uint32_t *g1; const uint8_t *g1_inf; const uint32_t *g2; const uint8_t *g2_inf; uint32_t *out;
  PCGPU_KERNEL_DEV void operator()(size_t i) const {
    constexpr int N = P::N;
    Fp<P> xp, yp;
    G2Aff<P> q;
    for (int j = 0; j < N; j++) { xp.l[j] = g1[i * 2 * N + j]; yp.l[j] = g1[i * 2 * N + N + j]; }
    for (int j = 0; j < 2 * N; j++) { coord_word(q.x, j) = g2[i * 4 * N + j]; coord_word(q.y, j) = g2[i * 4 * N + 2 * N + j]; }
    const bool inf = (g1_inf && g1_inf[i]) || (g2_inf && g2_inf[i]) || (xp.is_zero() && yp.is_zero()) || (q.x.is_zero() && q.y.is_zero());
    fq12_store<P>(out + i * Fq12<P>::WORDS, inf ? Fq12<P>::one() : miller_loop<P>(xp, yp, q));
  }
};

// G2Prepared::from for point i: the lines of miller_loop over Q, in loop order, into lines[i * prepared_point_words]; inf[i]
// is set for an identity flag or the all-zero encoding (its lines are not written: pairs with it contribute 1)
template <class P>
struct G2PrepareBody {
  const uint32_t *g2; const uint8_t *g2_inf; uint32_t *lines; uint8_t *inf;
  PCGPU_KERNEL_DEV void operator()(size_t i) const {
    constexpr int N = P::N;
    G2Aff<P> q;
    for (int j = 0; j < 2 * N; j++) { coord_word(q.x, j) = g2[i * 4 * N + j]; coord_word(q.y, j) = g2[i * 4 * N + 2 * N + j]; }
    inf[i] = (g2_inf && g2_inf[i]) || (q.x.is_zero() && q.y.is_zero());
    if (inf[i]) return;
    uint32_t *dst = lines + i * prepared_point_words<P>();
    G2Proj<P> T{q.x, q.y, Fq2<P>::one()};
    for (int b = P::MILLER_BITS - 2; b >= 0; b--) {
      line_store<P>(dst, dbl_step<P>(T)); dst += 6 * N;
      if ((P::miller_loop(b / 32) >> (b % 32)) & 1) { line_store<P>(dst, add_step<P>(T, q)); dst += 6 * N; }
    }
    if constexpr (P::MILLER_FROB) {
      const G2Aff<P> q1 = twist_frob<P>(q);
      G2Aff<P> q2 = twist_frob<P>(q1);
      q2.y = fp_neg<P>(q2.y);
      line_store<P>(dst, add_step<P>(T, q1)); dst += 6 * N;
      line_store<P>(dst, add_step<P>(T, q2));
    }
  }
};

// MillerBody with Q prepared: pair i is g1 point i against prepared point q_index[i]; each step squares f and folds in the
// stored lines, so T never lives in registers.  Writes MillerBody's output layout.
template <class P>
struct MillerPreparedBody {
  const uint32_t *g1; const uint8_t *g1_inf; const uint32_t *lines; const uint8_t *q_inf; const uint32_t *q_index; uint32_t *out;
  PCGPU_KERNEL_DEV void operator()(size_t i) const {
    constexpr int N = P::N;
    Fp<P> xp, yp;
    for (int j = 0; j < N; j++) { xp.l[j] = g1[i * 2 * N + j]; yp.l[j] = g1[i * 2 * N + N + j]; }
    const uint32_t q = q_index[i];
    if ((g1_inf && g1_inf[i]) || q_inf[q] || (xp.is_zero() && yp.is_zero())) { fq12_store<P>(out + i * Fq12<P>::WORDS, Fq12<P>::one()); return; }
    const uint32_t *src = lines + q * prepared_point_words<P>();
    Fq12<P> f = Fq12<P>::one();
    MillerLine<P> l;
    for (int b = P::MILLER_BITS - 2; b >= 0; b--) {
      f = fq12_sqr<P>(f);
      l = line_load<P>(src); src += 6 * N;
      f = mul_line_at<P>(f, l.ell0, l.ell1, l.ell2, xp, yp);
      if ((P::miller_loop(b / 32) >> (b % 32)) & 1) {
        l = line_load<P>(src); src += 6 * N;
        f = mul_line_at<P>(f, l.ell0, l.ell1, l.ell2, xp, yp);
      }
    }
    if constexpr (P::MILLER_NEG) f = fq12_conj<P>(f);
    if constexpr (P::MILLER_FROB) {
      for (int t = 0; t < 2; t++) {
        l = line_load<P>(src); src += 6 * N;
        f = mul_line_at<P>(f, l.ell0, l.ell1, l.ell2, xp, yp);
      }
    }
    fq12_store<P>(out + i * Fq12<P>::WORDS, f);
  }
};

// equation e: the product of its k Miller values, then the final exponentiation
template <class P>
struct FinalExpBody {
  const uint32_t *miller; size_t k; uint32_t *gt; uint8_t *is_one;
  PCGPU_KERNEL_DEV void operator()(size_t e) const {
    Fq12<P> f = Fq12<P>::one();
    for (size_t i = 0; i < k; i++) {
      Fq12<P> m;
      fq12_load<P>(m, miller + (e * k + i) * Fq12<P>::WORDS);
      f = i ? fq12_mul<P>(f, m) : m;
    }
    const Fq12<P> r = final_exponentiation<P>(f);
    fq12_store<P>(gt + e * Fq12<P>::WORDS, r);
    is_one[e] = r.is_one() ? 1 : 0;
  }
};

// pcgpu_diag_field_op which = 3: ops 0 a b, 2 a + b, 3 a - b, 4 -a, 5 a^-1 (0 -> 0), 9 a^2, 10 a^p, 11 the final exponentiation
template <class P>
struct Fq12OpBody {
  const uint32_t *a, *b; uint32_t *out; int op;
  PCGPU_KERNEL_DEV void operator()(size_t i) const {
    Fq12<P> x, y, r;
    fq12_load<P>(x, a + i * Fq12<P>::WORDS);
    fq12_load<P>(y, b + i * Fq12<P>::WORDS);
    switch (op) {
      case 0: r = fq12_mul<P>(x, y); break;
      case 2: r = fq12_add<P>(x, y); break;
      case 3: r = fq12_sub<P>(x, y); break;
      case 4: r = fq12_neg<P>(x); break;
      case 5: r = fq12_inv<P>(x); break;
      case 9: r = fq12_sqr<P>(x); break;
      case 10: r = fq12_frob<P, 1>(x); break;
      case 11: r = final_exponentiation<P>(x); break;
      default: r = fq12_sub<P>(x, x); break;
    }
    fq12_store<P>(out + i * Fq12<P>::WORDS, r);
  }
};

}  // namespace pcgpu
