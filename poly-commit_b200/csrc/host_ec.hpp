// Host-side finishing arithmetic: the last O(c) group operations of an MSM and the projective ->
// affine conversion, on 64-bit limbs.
//
// Why the host: a lone GPU thread retires one 381-bit Montgomery product far more slowly than a
// CPU core, so any strictly serial chain -- the Horner combination of the c bit-plane sums and the
// single field inversion -- is faster on the host.  The device does all O(n) work and hands back S*c points (3 KB for c = 16); this file adds
// them up.  It mirrors what the reference itself does on the CPU after the MSM:
// `commitment.into()` / `w.into_affine()` (kzg10/mod.rs:209, :281).  It is product code (always
// executed, never a substitute for the kernels) and shares nothing with oracle/.
//
// Same Montgomery radix and byte layout as the device (R = 2^(64 N)), so device XYZZ points are
// used as they come off the wire.
#pragma once
#include <stdint.h>
#include <string.h>
#include <type_traits>
#include "params_gen.cuh"

namespace pcgpu {
namespace host {

typedef unsigned __int128 u128;

template <class P>
struct HFp {
  static constexpr int N = P::N / 2;
  uint64_t l[N];
  struct ModTab { uint64_t v[P::N / 2]; ModTab() { for (int i = 0; i < P::N / 2; i++) v[i] = (uint64_t)P::mod(2 * i) | ((uint64_t)P::mod(2 * i + 1) << 32); } };
  static const uint64_t *modv() { static const ModTab t; return t.v; }
  static uint64_t mod(int i) { return modv()[i]; }
  static uint64_t m0() {  // -p^-1 mod 2^64 by Newton iteration
    uint64_t p0 = mod(0), inv = 1;
    for (int i = 0; i < 7; i++) inv *= 2 - p0 * inv;
    return (uint64_t)0 - inv;
  }
  static HFp zero() { HFp r; memset(r.l, 0, sizeof r.l); return r; }
  static HFp one() { HFp r; for (int i = 0; i < N; i++) r.l[i] = (uint64_t)P::one(2 * i) | ((uint64_t)P::one(2 * i + 1) << 32); return r; }
  bool is_zero() const { uint64_t o = 0; for (int i = 0; i < N; i++) o |= l[i]; return o == 0; }
  bool operator==(const HFp &b) const { uint64_t o = 0; for (int i = 0; i < N; i++) o |= l[i] ^ b.l[i]; return o == 0; }
};

template <class P> inline bool geq_mod(const uint64_t *a) {
  for (int i = HFp<P>::N - 1; i >= 0; i--) { uint64_t m = HFp<P>::mod(i); if (a[i] > m) return true; if (a[i] < m) return false; }
  return true;
}
template <class P> inline void sub_mod(uint64_t *a) {
  uint64_t br = 0;
  for (int i = 0; i < HFp<P>::N; i++) { u128 d = (u128)a[i] - HFp<P>::mod(i) - br; a[i] = (uint64_t)d; br = (uint64_t)(d >> 64) & 1; }
}
template <class P> inline HFp<P> add(const HFp<P> &a, const HFp<P> &b) {
  HFp<P> r; uint64_t c = 0;
  for (int i = 0; i < HFp<P>::N; i++) { u128 s = (u128)a.l[i] + b.l[i] + c; r.l[i] = (uint64_t)s; c = (uint64_t)(s >> 64); }
  if (c || geq_mod<P>(r.l)) sub_mod<P>(r.l);
  return r;
}
template <class P> inline HFp<P> sub(const HFp<P> &a, const HFp<P> &b) {
  HFp<P> r; uint64_t br = 0;
  for (int i = 0; i < HFp<P>::N; i++) { u128 d = (u128)a.l[i] - b.l[i] - br; r.l[i] = (uint64_t)d; br = (uint64_t)(d >> 64) & 1; }
  if (br) { uint64_t c = 0; for (int i = 0; i < HFp<P>::N; i++) { u128 s = (u128)r.l[i] + HFp<P>::mod(i) + c; r.l[i] = (uint64_t)s; c = (uint64_t)(s >> 64); } }
  return r;
}
template <class P> inline HFp<P> mul(const HFp<P> &a, const HFp<P> &b) {
  // CIOS with the two carry chains interleaved ("no-carry" variant: valid because the top bit of every modulus word N-1 is
  // clear, so t never needs an (N+1)-th word)
  constexpr int N = HFp<P>::N;
  static const uint64_t M0 = HFp<P>::m0();
  const uint64_t *q = HFp<P>::modv();
  uint64_t t[N];
  for (int j = 0; j < N; j++) t[j] = 0;
  for (int i = 0; i < N; i++) {
    const uint64_t bi = b.l[i];
    u128 s = (u128)a.l[0] * bi + t[0];
    uint64_t A = (uint64_t)(s >> 64), lo = (uint64_t)s;
    const uint64_t m = lo * M0;
    u128 r = (u128)m * q[0] + lo;
    uint64_t Cc = (uint64_t)(r >> 64);
    for (int j = 1; j < N; j++) {
      s = (u128)a.l[j] * bi + t[j] + A; A = (uint64_t)(s >> 64);
      r = (u128)m * q[j] + (uint64_t)s + Cc; Cc = (uint64_t)(r >> 64);
      t[j - 1] = (uint64_t)r;
    }
    t[N - 1] = Cc + A;
  }
  if (geq_mod<P>(t)) sub_mod<P>(t);
  HFp<P> rr; memcpy(rr.l, t, sizeof rr.l);
  return rr;
}
template <class P> inline HFp<P> sqr(const HFp<P> &a) { return mul<P>(a, a); }
template <class P> inline HFp<P> dbl(const HFp<P> &a) { return add<P>(a, a); }
template <class P> inline HFp<P> inv(const HFp<P> &a) {  // a^(p-2)
  constexpr int N = HFp<P>::N;
  uint64_t e[N]; uint64_t borrow = 2;
  for (int i = 0; i < N; i++) { uint64_t m = HFp<P>::mod(i); e[i] = m - borrow; borrow = m < borrow ? 1 : 0; }
  HFp<P> acc = HFp<P>::one();
  for (int i = N * 64 - 1; i >= 0; i--) { acc = sqr<P>(acc); if ((e[i / 64] >> (i % 64)) & 1) acc = mul<P>(acc, a); }
  return acc;
}

// Fq2 = Fq[u] / (u^2 + 1), c0 then c1 (the device's Fq2<P>, fq2.cuh): the coordinate field of G2.  Same function names as
// HFp, so the point code below runs on either field.
template <class P>
struct HFq2 {
  HFp<P> c0, c1;
  static HFq2 zero() { HFq2 r; r.c0 = HFp<P>::zero(); r.c1 = r.c0; return r; }
  static HFq2 one() { HFq2 r; r.c0 = HFp<P>::one(); r.c1 = HFp<P>::zero(); return r; }
  bool is_zero() const { return c0.is_zero() && c1.is_zero(); }
  bool operator==(const HFq2 &b) const { return c0 == b.c0 && c1 == b.c1; }
};
template <class P> inline HFq2<P> add(const HFq2<P> &a, const HFq2<P> &b) { HFq2<P> r; r.c0 = add<P>(a.c0, b.c0); r.c1 = add<P>(a.c1, b.c1); return r; }
template <class P> inline HFq2<P> sub(const HFq2<P> &a, const HFq2<P> &b) { HFq2<P> r; r.c0 = sub<P>(a.c0, b.c0); r.c1 = sub<P>(a.c1, b.c1); return r; }
template <class P> inline HFq2<P> mul(const HFq2<P> &a, const HFq2<P> &b) {
  HFq2<P> r;
  r.c0 = sub<P>(mul<P>(a.c0, b.c0), mul<P>(a.c1, b.c1));
  r.c1 = add<P>(mul<P>(a.c0, b.c1), mul<P>(a.c1, b.c0));
  return r;
}
template <class P> inline HFq2<P> sqr(const HFq2<P> &a) { return mul<P>(a, a); }
template <class P> inline HFq2<P> dbl(const HFq2<P> &a) { return add<P>(a, a); }
template <class P> inline HFq2<P> inv(const HFq2<P> &a) {   // conjugate over the norm; 0 -> 0
  const HFp<P> t = inv<P>(add<P>(mul<P>(a.c0, a.c0), mul<P>(a.c1, a.c1)));
  HFq2<P> r;
  r.c0 = mul<P>(a.c0, t);
  r.c1 = sub<P>(HFp<P>::zero(), mul<P>(a.c1, t));
  return r;
}

// XYZZ point; the byte image equals the device's XYZZ<C>.  F: HFp<Fq> for G1, HFq2<Fq> for G2 (C::EXT)
template <class C>
struct HXYZZ {
  using Q = typename C::Fq;
  using F = typename std::conditional<C::EXT == 2, HFq2<Q>, HFp<Q>>::type;
  F x, y, zz, zzz;
  bool is_inf() const { return zz.is_zero(); }
  static HXYZZ inf() { HXYZZ p; memset(&p, 0, sizeof p); return p; }
};

template <class C> inline HXYZZ<C> pdbl(const HXYZZ<C> &p) {  // dbl-2008-s-1
  using Q = typename C::Fq;
  using F = typename HXYZZ<C>::F;
  if (p.is_inf()) return p;
  HXYZZ<C> r;
  F U = dbl<Q>(p.y), V = sqr<Q>(U), W = mul<Q>(U, V), S = mul<Q>(p.x, V);
  F X2 = sqr<Q>(p.x), M = add<Q>(dbl<Q>(X2), X2);
  r.x = sub<Q>(sqr<Q>(M), dbl<Q>(S));
  r.y = sub<Q>(mul<Q>(M, sub<Q>(S, r.x)), mul<Q>(W, p.y));
  r.zz = mul<Q>(V, p.zz); r.zzz = mul<Q>(W, p.zzz);
  return r;
}
template <class C> inline HXYZZ<C> padd(const HXYZZ<C> &p, const HXYZZ<C> &q) {  // add-2008-s
  using Q = typename C::Fq;
  using F = typename HXYZZ<C>::F;
  if (q.is_inf()) return p;
  if (p.is_inf()) return q;
  F U1 = mul<Q>(p.x, q.zz), U2 = mul<Q>(q.x, p.zz), S1 = mul<Q>(p.y, q.zzz), S2 = mul<Q>(q.y, p.zzz);
  F Pd = sub<Q>(U2, U1), R = sub<Q>(S2, S1);
  if (Pd.is_zero()) return R.is_zero() ? pdbl<C>(p) : HXYZZ<C>::inf();
  F PP = sqr<Q>(Pd), PPP = mul<Q>(Pd, PP), Qv = mul<Q>(U1, PP);
  HXYZZ<C> r;
  r.x = sub<Q>(sub<Q>(sqr<Q>(R), PPP), dbl<Q>(Qv));
  r.y = sub<Q>(mul<Q>(R, sub<Q>(Qv, r.x)), mul<Q>(S1, PPP));
  r.zz = mul<Q>(mul<Q>(p.zz, q.zz), PP);
  r.zzz = mul<Q>(mul<Q>(p.zzz, q.zzz), PPP);
  return r;
}
// affine x||y (zeros + flag for the identity)
template <class C> inline void to_affine(const HXYZZ<C> &p, void *out_xy, uint8_t *out_inf) {
  using Q = typename C::Fq;
  using F = typename HXYZZ<C>::F;
  constexpr size_t FB = sizeof(F);
  if (p.is_inf()) { if (out_xy) memset(out_xy, 0, 2 * FB); if (out_inf) *out_inf = 1; return; }
  F iv = inv<Q>(mul<Q>(p.zz, p.zzz));
  F x = mul<Q>(p.x, mul<Q>(iv, p.zzz)), y = mul<Q>(p.y, mul<Q>(iv, p.zz));
  if (out_xy) { memcpy(out_xy, &x, FB); memcpy((char *)out_xy + FB, &y, FB); }
  if (out_inf) *out_inf = 0;
}

// k * P for an affine P (x||y Montgomery limbs, identity = all zero) and a CANONICAL 256-bit scalar
template <class C> inline HXYZZ<C> pmul_affine(const void *p_xy, const uint64_t *k) {
  using F = typename HXYZZ<C>::F;
  HXYZZ<C> base;
  memcpy(&base.x, p_xy, sizeof base.x); memcpy(&base.y, (const char *)p_xy + sizeof base.x, sizeof base.y);
  if (base.x.is_zero() && base.y.is_zero()) return HXYZZ<C>::inf();
  base.zz = F::one(); base.zzz = F::one();
  HXYZZ<C> acc = HXYZZ<C>::inf();
  for (int b = 255; b >= 0; b--) { acc = pdbl<C>(acc); if ((k[b >> 6] >> (b & 63)) & 1) acc = padd<C>(acc, base); }
  return acc;
}
// Montgomery -> canonical for one Fr element on the host
template <class R> inline void fr_from_mont_host(const void *in, uint64_t *out) {
  HFp<R> a, one = HFp<R>::zero(); memcpy(a.l, in, sizeof a.l); one.l[0] = 1;
  HFp<R> r = mul<R>(a, one); memcpy(out, r.l, sizeof r.l);
}

// Small-MSM path (msm_small.cuh): the device hands back one point per window, U_w = sum_k k B_{w,k};
//   result = sum_w 2^(c w) U_w   -- c * (W - 1) doublings and W additions
template <class C> inline HXYZZ<C> combine_windows(const HXYZZ<C> *U, uint32_t W, uint32_t c) {
  HXYZZ<C> acc = HXYZZ<C>::inf();
  for (uint32_t w = W; w-- > 0;) {
    if (w + 1 < W) for (uint32_t k = 0; k < c; k++) acc = pdbl<C>(acc);
    acc = padd<C>(acc, U[w]);
  }
  return acc;
}

// Combination of the device's bit-plane sums (msm.cuh, two-level reduction): per set the device hands back the planes of the
// column sums C (weights lo+1, bits_c of them) followed by the planes of the row sums R (weights hi, bits_r):
//   set value = sum_j 2^j TC_j + 2^h * sum_j 2^j TR_j,   result = sum_s 2^(c s) * set value
// (S = c = 1, h = 0: the one plane itself -- the peer path's one-point record)
template <class C> inline HXYZZ<C> combine_bit_planes_2level(const HXYZZ<C> *T, uint32_t S, uint32_t c, uint32_t h) {
  const uint32_t bits_c = h + 1, bits_r = c - 1 - h, per = bits_c + bits_r;
  HXYZZ<C> acc = HXYZZ<C>::inf();
  for (uint32_t s = S; s-- > 0;) {
    const HXYZZ<C> *Ts = T + (size_t)s * per;
    HXYZZ<C> vr = HXYZZ<C>::inf(), vc = HXYZZ<C>::inf();
    for (uint32_t j = bits_r; j-- > 0;) { vr = pdbl<C>(vr); vr = padd<C>(vr, Ts[bits_c + j]); }
    for (uint32_t k = 0; k < h; k++) vr = pdbl<C>(vr);
    for (uint32_t j = bits_c; j-- > 0;) { vc = pdbl<C>(vc); vc = padd<C>(vc, Ts[j]); }
    HXYZZ<C> v = padd<C>(vr, vc);
    if (s + 1 < S) for (uint32_t k = 0; k < c; k++) acc = pdbl<C>(acc);
    acc = padd<C>(acc, v);
  }
  return acc;
}

}  // namespace host
}  // namespace pcgpu
