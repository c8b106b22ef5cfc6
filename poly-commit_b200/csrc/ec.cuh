// Short-Weierstrass (a = 0) group arithmetic in XYZZ coordinates (x = X/ZZ, y = Y/ZZZ, ZZ^3 = ZZZ^2)
// for G1 of the three curves BASELINE.json names (BLS12-381, BN254, Pallas) and G2 of the two pairing curves: the same
// formulas over the group's coordinate field C::F (Fq, or Fq2 of fq2.cuh).
//
// Serves the group operations ark-ec 0.5.0 performs inside VariableBaseMSM::msm_bigint (call sites
// kzg10/mod.rs:175-178, :255-258; ipa_pc/mod.rs:64; hyrax/mod.rs:92) -- ark-ec uses Jacobian
// coordinates; the formulas here are the EFD "xyzz" set (madd-2008-s, add-2008-s, dbl-2008-s-1,
// mdbl-2008-s-1), chosen because the mixed add is 8M+2S with no inversion and no Z tracking.  Any
// correct group law yields the same affine result, which is where parity is checked.
//
// Conventions: affine (0, 0) encodes the point at infinity on the device (not on any of the curves
// since b != 0); the ABI's separate infinity byte is folded into that at SRS registration.
// XYZZ identity: ZZ == 0.
#pragma once
#include "fp.cuh"
#include "fq2.cuh"

namespace pcgpu {

// A group: its base field Fq, scalar field Fr, coordinate field F (Fq for G1, Fq2 for G2), extension degree EXT of F over Fq,
// and ID, the curve index of per-curve tables (d_pow2, NTT plans).
struct Bls12381 { using Fq = Bls12381Fq; using Fr = Bls12381Fr; using F = Fp<Fq>; static constexpr int ID = 0, EXT = 1; };
struct Bn254 { using Fq = Bn254Fq; using Fr = Bn254Fr; using F = Fp<Fq>; static constexpr int ID = 1, EXT = 1; };
struct Pallas { using Fq = PallasFq; using Fr = PallasFr; using F = Fp<Fq>; static constexpr int ID = 2, EXT = 1; };
// G2 on the sextic twists y^2 = x^3 + b' over Fq2 (b' = 4(1 + u) on BLS12-381, 3 / (9 + u) on BN254; b' != 0, so (0, 0) is
// not on either twist and stays the identity encoding).  Only the MSM, fixed-base and MultilinearPC paths instantiate them.
struct Bls12381G2 { using Fq = Bls12381Fq; using Fr = Bls12381Fr; using F = Fq2<Fq>; static constexpr int ID = 0, EXT = 2; };
struct Bn254G2 { using Fq = Bn254Fq; using Fr = Bn254Fr; using F = Fq2<Fq>; static constexpr int ID = 1, EXT = 2; };

template <class C>
struct Affine {
  typename C::F x, y;
  PCGPU_HD bool is_inf() const { return x.is_zero() && y.is_zero(); }
  PCGPU_HD static Affine inf() { Affine a; a.x = C::F::zero(); a.y = a.x; return a; }
};

template <class C>
struct XYZZ {
  typename C::F x, y, zz, zzz;
  PCGPU_HD bool is_inf() const { return zz.is_zero(); }
  PCGPU_HD static XYZZ inf() { XYZZ p; p.x = C::F::zero(); p.y = p.x; p.zz = p.x; p.zzz = p.x; return p; }
};

template <class C>
PCGPU_DEV XYZZ<C> xyzz_from_affine(const Affine<C> &a) {
  using F = typename C::F;
  XYZZ<C> p;
  if (a.is_inf()) return XYZZ<C>::inf();
  p.x = a.x; p.y = a.y; p.zz = F::one(); p.zzz = F::one();
  return p;
}

// mdbl-2008-s-1: 2 * (affine point)
template <class C>
PCGPU_DEV XYZZ<C> xyzz_dbl_affine(const Affine<C> &a) {
  using Q = typename C::Fq;
  using F = typename C::F;
  if (a.is_inf()) return XYZZ<C>::inf();
  XYZZ<C> r;
  F U = fp_dbl<Q>(a.y);
  F V = fp_sqr<Q>(U);
  F W = fp_mul<Q>(U, V);
  F S = fp_mul<Q>(a.x, V);
  F M = fp_mul3<Q>(fp_sqr<Q>(a.x));
  r.x = fp_sub<Q>(fp_sqr<Q>(M), fp_dbl<Q>(S));
  r.y = fp_mul2<Q>(M, fp_sub<Q>(S, r.x), W, fp_neg<Q>(a.y));
  r.zz = V; r.zzz = W;
  return r;
}

// dbl-2008-s-1
template <class C>
PCGPU_DEV XYZZ<C> xyzz_dbl(const XYZZ<C> &p) {
  using Q = typename C::Fq;
  using F = typename C::F;
  if (p.is_inf()) return p;
  XYZZ<C> r;
  F U = fp_dbl<Q>(p.y);
  F V = fp_sqr<Q>(U);
  F W = fp_mul<Q>(U, V);
  F S = fp_mul<Q>(p.x, V);
  F M = fp_mul3<Q>(fp_sqr<Q>(p.x));
  r.x = fp_sub<Q>(fp_sqr<Q>(M), fp_dbl<Q>(S));
  r.y = fp_mul2<Q>(M, fp_sub<Q>(S, r.x), W, fp_neg<Q>(p.y));
  r.zz = fp_mul<Q>(V, p.zz);
  r.zzz = fp_mul<Q>(W, p.zzz);
  return r;
}

// madd-2008-s with the exceptional cases (identity operands, P + P, P + (-P)) handled.
// `neg` adds -a instead of a (signed Pippenger digits).
template <class C>
PCGPU_DEV void xyzz_madd(XYZZ<C> &p, const Affine<C> &a_in, bool neg) {
  using Q = typename C::Fq;
  using F = typename C::F;
  if (a_in.is_inf()) return;
  Affine<C> a = a_in;
  a.y = fp_cneg<Q>(a.y, neg);
  if (p.is_inf()) { p.x = a.x; p.y = a.y; p.zz = F::one(); p.zzz = F::one(); return; }
  F U2 = fp_mul<Q>(a.x, p.zz);
  F S2 = fp_mul<Q>(a.y, p.zzz);
  F Pd = fp_sub<Q>(U2, p.x);
  F R = fp_sub<Q>(S2, p.y);
  if (Pd.is_zero()) {
    if (R.is_zero()) p = xyzz_dbl_affine<C>(a); else p = XYZZ<C>::inf();
    return;
  }
  F PP = fp_sqr<Q>(Pd);
  F PPP = fp_mul<Q>(Pd, PP);
  F Qv = fp_mul<Q>(p.x, PP);
  F x3 = fp_sub<Q>(fp_sub<Q>(fp_sqr<Q>(R), PPP), fp_dbl<Q>(Qv));
  F y3 = fp_mul2<Q>(R, fp_sub<Q>(Qv, x3), fp_neg<Q>(p.y), PPP);
  p.x = x3; p.y = y3;
  p.zz = fp_mul<Q>(p.zz, PP);
  p.zzz = fp_mul<Q>(p.zzz, PPP);
}

// add-2008-s with exceptional cases
template <class C>
PCGPU_DEV void xyzz_add(XYZZ<C> &p, const XYZZ<C> &q) {
  using Q = typename C::Fq;
  using F = typename C::F;
  if (q.is_inf()) return;
  if (p.is_inf()) { p = q; return; }
  F U1 = fp_mul<Q>(p.x, q.zz);
  F U2 = fp_mul<Q>(q.x, p.zz);
  F S1 = fp_mul<Q>(p.y, q.zzz);
  F S2 = fp_mul<Q>(q.y, p.zzz);
  F Pd = fp_sub<Q>(U2, U1);
  F R = fp_sub<Q>(S2, S1);
  if (Pd.is_zero()) {
    if (R.is_zero()) p = xyzz_dbl<C>(p); else p = XYZZ<C>::inf();
    return;
  }
  F PP = fp_sqr<Q>(Pd);
  F PPP = fp_mul<Q>(Pd, PP);
  F Qv = fp_mul<Q>(U1, PP);
  F x3 = fp_sub<Q>(fp_sub<Q>(fp_sqr<Q>(R), PPP), fp_dbl<Q>(Qv));
  F y3 = fp_mul2<Q>(R, fp_sub<Q>(Qv, x3), fp_neg<Q>(S1), PPP);
  p.x = x3; p.y = y3;
  p.zz = fp_mul<Q>(fp_mul<Q>(p.zz, q.zz), PP);
  p.zzz = fp_mul<Q>(fp_mul<Q>(p.zzz, q.zzz), PPP);
}

// x = X/ZZ, y = Y/ZZZ with one inversion of ZZ*ZZZ
template <class C>
PCGPU_DEV Affine<C> xyzz_to_affine(const XYZZ<C> &p) {
  using Q = typename C::Fq;
  using F = typename C::F;
  if (p.is_inf()) return Affine<C>::inf();
  F inv = fp_inv<Q>(fp_mul<Q>(p.zz, p.zzz));
  Affine<C> a;
  a.x = fp_mul<Q>(p.x, fp_mul<Q>(inv, p.zzz));
  a.y = fp_mul<Q>(p.y, fp_mul<Q>(inv, p.zz));
  return a;
}

template <class C>
PCGPU_DEV bool affine_on_curve(const Affine<C> &a) {
  using Q = typename C::Fq;
  if (a.is_inf()) return true;
  Fp<Q> b;
#pragma unroll
  for (int i = 0; i < Q::N; i++) b.l[i] = Q::curve_b(i);
  Fp<Q> lhs = fp_sqr<Q>(a.y);
  Fp<Q> rhs = fp_add<Q>(fp_mul<Q>(fp_sqr<Q>(a.x), a.x), b);
  return lhs == rhs;
}

}  // namespace pcgpu
