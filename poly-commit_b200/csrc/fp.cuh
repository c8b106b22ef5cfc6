// Prime-field arithmetic for sm_90a: N x 32-bit limbs held in registers, Montgomery form
// with R = 2^(32 N) (identical to ark-ff's 2^(64 N/2), so the byte image of an element equals
// ark-ff's Fp<MontBackend, N/2>; SURVEY.md section 8b "Data conventions").
//
// Replaces (on the device) the ark-ff 0.5.0 arithmetic that sits under every hot call site of the
// reference: kzg10/mod.rs:175-178 (MSM), :463-470 (into_bigint), marlin_pc/mod.rs:286 (axpy),
// kzg10/mod.rs:222-226 (division).  ark-ff is an un-vendored dependency; nothing here is derived
// from its source.
//
// The multiplier is an operand-scanning Montgomery product whose partial products are split into an
// even-column and an odd-column accumulator so that every (mad.lo.cc, madc.hi.cc) pair works on one
// 64-bit product and carries ripple along a single chain per accumulator; ptxas fuses each pair into
// one IMAD.WIDE.U32 with carry-in/out.  A plain 64-bit-accumulate version (mont_mul_ref) is kept for
// differential tests.  When compiled for the host (tests/host_emul) the PTX carry instructions are
// emulated with an explicit carry flag so the very same limb schedule can be checked on a CPU.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include "params_gen.cuh"

#ifdef __CUDACC__
#define PCGPU_DEV __device__ __forceinline__
#else
#define PCGPU_DEV inline
#endif

namespace pcgpu {

// ---------------------------------------------------------------------------------------------
// carry-flag primitives
// ---------------------------------------------------------------------------------------------
#ifdef __CUDA_ARCH__
PCGPU_DEV uint32_t add_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("add.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
PCGPU_DEV uint32_t addc_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("addc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
PCGPU_DEV uint32_t addc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("addc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
PCGPU_DEV uint32_t sub_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("sub.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
PCGPU_DEV uint32_t subc_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("subc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
PCGPU_DEV uint32_t subc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("subc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
PCGPU_DEV uint32_t mad_lo_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("mad.lo.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
PCGPU_DEV uint32_t madc_lo_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("madc.lo.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
PCGPU_DEV uint32_t madc_hi_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("madc.hi.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
PCGPU_DEV uint32_t madc_hi(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("madc.hi.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
PCGPU_DEV uint32_t mul_lo(uint32_t a, uint32_t b) { return a * b; }
PCGPU_DEV uint32_t mul_hi(uint32_t a, uint32_t b) { return __umulhi(a, b); }
#else
// Host emulation (tests only): one carry flag per thread, same semantics as PTX CC.CF.
namespace emul { inline uint32_t &cf() { static thread_local uint32_t f = 0; return f; } }
inline uint32_t add_cc(uint32_t a, uint32_t b) { uint64_t s = (uint64_t)a + b; emul::cf() = (uint32_t)(s >> 32); return (uint32_t)s; }
inline uint32_t addc_cc(uint32_t a, uint32_t b) { uint64_t s = (uint64_t)a + b + emul::cf(); emul::cf() = (uint32_t)(s >> 32); return (uint32_t)s; }
inline uint32_t addc(uint32_t a, uint32_t b) { return a + b + emul::cf(); }
inline uint32_t sub_cc(uint32_t a, uint32_t b) { uint64_t d = (uint64_t)a - b; emul::cf() = (uint32_t)(d >> 63); return (uint32_t)d; }
inline uint32_t subc_cc(uint32_t a, uint32_t b) { uint64_t d = (uint64_t)a - b - emul::cf(); emul::cf() = (uint32_t)(d >> 63); return (uint32_t)d; }
inline uint32_t subc(uint32_t a, uint32_t b) { return a - b - emul::cf(); }
inline uint32_t mul_lo(uint32_t a, uint32_t b) { return a * b; }
inline uint32_t mul_hi(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) >> 32); }
inline uint32_t mad_lo_cc(uint32_t a, uint32_t b, uint32_t c) { return add_cc(mul_lo(a, b), c); }
inline uint32_t madc_lo_cc(uint32_t a, uint32_t b, uint32_t c) { return addc_cc(mul_lo(a, b), c); }
inline uint32_t madc_hi_cc(uint32_t a, uint32_t b, uint32_t c) { return addc_cc(mul_hi(a, b), c); }
inline uint32_t madc_hi(uint32_t a, uint32_t b, uint32_t c) { return addc(mul_hi(a, b), c); }
#endif
// NOTE on PTX borrow semantics: sub.cc sets CC.CF to the borrow-out and subc consumes it as a
// borrow-in, so the host emulation keeps "1 = borrow" in the same flag.

// ---------------------------------------------------------------------------------------------
// Fp<P>: P supplies N, M0 = -p^-1 mod 2^32, mod(i), one(i) = R mod p, r2(i) = R^2 mod p
// ---------------------------------------------------------------------------------------------
template <class P>
struct Fp {
  static constexpr int N = P::N;
  uint32_t l[N];

  PCGPU_HD static Fp zero() { Fp r;
#pragma unroll
    for (int i = 0; i < N; i++) r.l[i] = 0;
    return r; }
  PCGPU_HD static Fp one() { Fp r;
#pragma unroll
    for (int i = 0; i < N; i++) r.l[i] = P::one(i);
    return r; }
  PCGPU_HD static Fp r2() { Fp r;
#pragma unroll
    for (int i = 0; i < N; i++) r.l[i] = P::r2(i);
    return r; }
  PCGPU_HD static Fp modulus() { Fp r;
#pragma unroll
    for (int i = 0; i < N; i++) r.l[i] = P::mod(i);
    return r; }
  PCGPU_HD bool is_zero() const { uint32_t o = 0;
#pragma unroll
    for (int i = 0; i < N; i++) o |= l[i];
    return o == 0; }
  PCGPU_HD bool operator==(const Fp &b) const { uint32_t o = 0;
#pragma unroll
    for (int i = 0; i < N; i++) o |= l[i] ^ b.l[i];
    return o == 0; }
  PCGPU_HD bool operator!=(const Fp &b) const { return !(*this == b); }
};

// r = (a >= p) ? a - p : a, for a < 2p
template <class P>
PCGPU_DEV void fp_reduce_once(uint32_t *a) {
  constexpr int N = P::N;
  uint32_t t[N];
  t[0] = sub_cc(a[0], P::mod(0));
#pragma unroll
  for (int i = 1; i < N; i++) t[i] = subc_cc(a[i], P::mod(i));
  uint32_t borrow = subc(0u, 0u);  // 0xffffffff if a < p
#pragma unroll
  for (int i = 0; i < N; i++) a[i] = borrow ? a[i] : t[i];
}

template <class P>
PCGPU_DEV Fp<P> fp_add(const Fp<P> &a, const Fp<P> &b) {
  constexpr int N = P::N;
  Fp<P> r;
  r.l[0] = add_cc(a.l[0], b.l[0]);
#pragma unroll
  for (int i = 1; i < N - 1; i++) r.l[i] = addc_cc(a.l[i], b.l[i]);
  r.l[N - 1] = addc(a.l[N - 1], b.l[N - 1]);  // 2p < 2^(32N): no carry out
  fp_reduce_once<P>(r.l);
  return r;
}

template <class P>
PCGPU_DEV Fp<P> fp_sub(const Fp<P> &a, const Fp<P> &b) {
  constexpr int N = P::N;
  Fp<P> r;
  r.l[0] = sub_cc(a.l[0], b.l[0]);
#pragma unroll
  for (int i = 1; i < N; i++) r.l[i] = subc_cc(a.l[i], b.l[i]);
  uint32_t mask = subc(0u, 0u);  // all ones if a < b
  r.l[0] = add_cc(r.l[0], P::mod(0) & mask);
#pragma unroll
  for (int i = 1; i < N - 1; i++) r.l[i] = addc_cc(r.l[i], P::mod(i) & mask);
  r.l[N - 1] = addc(r.l[N - 1], P::mod(N - 1) & mask);
  return r;
}

template <class P>
PCGPU_DEV Fp<P> fp_neg(const Fp<P> &a) {
  constexpr int N = P::N;
  Fp<P> r;
  uint32_t nz = 0;
#pragma unroll
  for (int i = 0; i < N; i++) nz |= a.l[i];
  r.l[0] = sub_cc(P::mod(0), a.l[0]);
#pragma unroll
  for (int i = 1; i < N - 1; i++) r.l[i] = subc_cc(P::mod(i), a.l[i]);
  r.l[N - 1] = subc(P::mod(N - 1), a.l[N - 1]);
  uint32_t mask = nz ? 0xffffffffu : 0u;  // -0 = 0
#pragma unroll
  for (int i = 0; i < N; i++) r.l[i] &= mask;
  return r;
}

// conditional negate (used for signed Pippenger digits)
template <class P>
PCGPU_DEV Fp<P> fp_cneg(const Fp<P> &a, bool neg) {
  Fp<P> n = fp_neg<P>(a);
  Fp<P> r;
#pragma unroll
  for (int i = 0; i < P::N; i++) r.l[i] = neg ? n.l[i] : a.l[i];
  return r;
}

template <class P>
PCGPU_DEV Fp<P> fp_dbl(const Fp<P> &a) { return fp_add<P>(a, a); }

// ---- reference multiplier: textbook CIOS with 64-bit accumulation (host + device) ----
template <class P>
PCGPU_HD Fp<P> mont_mul_ref(const Fp<P> &a, const Fp<P> &b) {
  constexpr int N = P::N;
  uint32_t t[N + 2];
#pragma unroll
  for (int i = 0; i < N + 2; i++) t[i] = 0;
#pragma unroll
  for (int i = 0; i < N; i++) {
    uint64_t c = 0;
#pragma unroll
    for (int j = 0; j < N; j++) { uint64_t s = (uint64_t)a.l[j] * b.l[i] + t[j] + c; t[j] = (uint32_t)s; c = s >> 32; }
    uint64_t s = (uint64_t)t[N] + c; t[N] = (uint32_t)s; t[N + 1] = (uint32_t)(s >> 32);
    uint32_t m = t[0] * P::M0;
    s = (uint64_t)m * P::mod(0) + t[0]; c = s >> 32;
#pragma unroll
    for (int j = 1; j < N; j++) { s = (uint64_t)m * P::mod(j) + t[j] + c; t[j - 1] = (uint32_t)s; c = s >> 32; }
    s = (uint64_t)t[N] + c; t[N - 1] = (uint32_t)s; t[N] = t[N + 1] + (uint32_t)(s >> 32);
  }
  // t < 2p < 2^(32N) so t[N] == 0; conditional subtraction without carry flags
  uint32_t d[N]; uint64_t br = 0;
#pragma unroll
  for (int i = 0; i < N; i++) { uint64_t x = (uint64_t)t[i] - P::mod(i) - br; d[i] = (uint32_t)x; br = (x >> 63) & 1; }
  Fp<P> r;
#pragma unroll
  for (int i = 0; i < N; i++) r.l[i] = br ? t[i] : d[i];
  return r;
}

// ---- production multiplier: even/odd column accumulators, carry-chained mad.lo/mad.hi pairs ----
//
// State: T = X + Y * 2^32 with X, Y N-limb arrays.  One row (operand limb bi):
//   X[0] += Yold[1]                      (the limb that falls out of the 64-bit shift of the old even part)
//   Y    = (Yold >> 64) + a_odd  * bi    (in place, carry chained from the line above)
//   X   +=                a_even * bi    (carry out -> Y[N-1])
//   m    = X[0] * M0
//   Y   += p_odd  * m                    (cannot carry out: T < 2^(32N+32))
//   X   += p_even * m                    (carry out -> Y[N-1]); now X[0] == 0
//   T >>= 32 is realised by exchanging the roles of X and Y for the next row.
template <class P, bool FIRST>
PCGPU_DEV void mont_row(uint32_t *X, uint32_t *Y, const uint32_t *a, uint32_t bi) {
  constexpr int N = P::N;
  if (FIRST) {
#pragma unroll
    for (int j = 0; j < N; j += 2) {
      X[j] = mul_lo(a[j], bi); X[j + 1] = mul_hi(a[j], bi);
      Y[j] = mul_lo(a[j + 1], bi); Y[j + 1] = mul_hi(a[j + 1], bi);
    }
  } else {
    X[0] = add_cc(X[0], Y[1]);
#pragma unroll
    for (int j = 0; j < N - 2; j += 2) {
      Y[j] = madc_lo_cc(a[j + 1], bi, Y[j + 2]);
      Y[j + 1] = madc_hi_cc(a[j + 1], bi, Y[j + 3]);
    }
    Y[N - 2] = madc_lo_cc(a[N - 1], bi, 0u);
    Y[N - 1] = madc_hi(a[N - 1], bi, 0u);
    X[0] = mad_lo_cc(a[0], bi, X[0]);
    X[1] = madc_hi_cc(a[0], bi, X[1]);
#pragma unroll
    for (int j = 2; j < N; j += 2) {
      X[j] = madc_lo_cc(a[j], bi, X[j]);
      X[j + 1] = madc_hi_cc(a[j], bi, X[j + 1]);
    }
    Y[N - 1] = addc(Y[N - 1], 0u);
  }
  uint32_t m = X[0] * P::M0;
  Y[0] = mad_lo_cc(P::mod(1), m, Y[0]);
  Y[1] = madc_hi_cc(P::mod(1), m, Y[1]);
#pragma unroll
  for (int j = 2; j < N; j += 2) {
    Y[j] = madc_lo_cc(P::mod(j + 1), m, Y[j]);
    Y[j + 1] = madc_hi_cc(P::mod(j + 1), m, Y[j + 1]);
  }
  X[0] = mad_lo_cc(P::mod(0), m, X[0]);
  X[1] = madc_hi_cc(P::mod(0), m, X[1]);
#pragma unroll
  for (int j = 2; j < N; j += 2) {
    X[j] = madc_lo_cc(P::mod(j), m, X[j]);
    X[j + 1] = madc_hi_cc(P::mod(j), m, X[j + 1]);
  }
  Y[N - 1] = addc(Y[N - 1], 0u);
}

template <class P>
PCGPU_DEV Fp<P> mont_mul(const Fp<P> &a, const Fp<P> &b) {
  constexpr int N = P::N;
  static_assert(N % 2 == 0, "even limb count required");
  uint32_t X[N], Y[N];
  mont_row<P, true>(X, Y, a.l, b.l[0]);
  mont_row<P, false>(Y, X, a.l, b.l[1]);
#pragma unroll
  for (int i = 2; i < N; i += 2) {
    mont_row<P, false>(X, Y, a.l, b.l[i]);
    mont_row<P, false>(Y, X, a.l, b.l[i + 1]);
  }
  // after an even number of rows the low (zero) limb sits in Y[0]... see below: roles are back to
  // (X = even part with X[0] == 0 consumed, Y = odd part); result = Y' + (X' >> 32) with
  // X' = last row's X (zero low limb) and Y' = last row's Y.  The last call used (X=Y_arr, Y=X_arr).
  Fp<P> r;
  r.l[0] = add_cc(X[0], Y[1]);
#pragma unroll
  for (int i = 1; i < N - 1; i++) r.l[i] = addc_cc(X[i], Y[i + 1]);
  r.l[N - 1] = addc(X[N - 1], 0u);
  fp_reduce_once<P>(r.l);
  return r;
}

// ---- sum of two products with ONE Montgomery reduction:  a*b + c*d  (mod p, Montgomery form) ----
// Same row structure as mont_row with a second pair of product chains per row; T stays below 3p
// (3p < 2^(32N) for every field here), so the result needs two conditional subtractions.  Saves one
// reduction phase (N^2/2 wide multiplies) wherever a formula has the shape x*y - z*w.
template <class P, bool FIRST>
PCGPU_DEV void mont_row2(uint32_t *X, uint32_t *Y, const uint32_t *a, uint32_t bi, const uint32_t *c, uint32_t di) {
  constexpr int N = P::N;
  if (FIRST) {
#pragma unroll
    for (int j = 0; j < N; j += 2) {
      X[j] = mul_lo(a[j], bi); X[j + 1] = mul_hi(a[j], bi);
      Y[j] = mul_lo(a[j + 1], bi); Y[j + 1] = mul_hi(a[j + 1], bi);
    }
  } else {
    X[0] = add_cc(X[0], Y[1]);
#pragma unroll
    for (int j = 0; j < N - 2; j += 2) {
      Y[j] = madc_lo_cc(a[j + 1], bi, Y[j + 2]);
      Y[j + 1] = madc_hi_cc(a[j + 1], bi, Y[j + 3]);
    }
    Y[N - 2] = madc_lo_cc(a[N - 1], bi, 0u);
    Y[N - 1] = madc_hi(a[N - 1], bi, 0u);
    X[0] = mad_lo_cc(a[0], bi, X[0]);
    X[1] = madc_hi_cc(a[0], bi, X[1]);
#pragma unroll
    for (int j = 2; j < N; j += 2) {
      X[j] = madc_lo_cc(a[j], bi, X[j]);
      X[j + 1] = madc_hi_cc(a[j], bi, X[j + 1]);
    }
    Y[N - 1] = addc(Y[N - 1], 0u);
  }
  // second product c * di
  Y[0] = mad_lo_cc(c[1], di, Y[0]);
  Y[1] = madc_hi_cc(c[1], di, Y[1]);
#pragma unroll
  for (int j = 2; j < N; j += 2) {
    Y[j] = madc_lo_cc(c[j + 1], di, Y[j]);
    Y[j + 1] = madc_hi_cc(c[j + 1], di, Y[j + 1]);
  }
  X[0] = mad_lo_cc(c[0], di, X[0]);
  X[1] = madc_hi_cc(c[0], di, X[1]);
#pragma unroll
  for (int j = 2; j < N; j += 2) {
    X[j] = madc_lo_cc(c[j], di, X[j]);
    X[j + 1] = madc_hi_cc(c[j], di, X[j + 1]);
  }
  Y[N - 1] = addc(Y[N - 1], 0u);
  // reduction row
  uint32_t m = X[0] * P::M0;
  Y[0] = mad_lo_cc(P::mod(1), m, Y[0]);
  Y[1] = madc_hi_cc(P::mod(1), m, Y[1]);
#pragma unroll
  for (int j = 2; j < N; j += 2) {
    Y[j] = madc_lo_cc(P::mod(j + 1), m, Y[j]);
    Y[j + 1] = madc_hi_cc(P::mod(j + 1), m, Y[j + 1]);
  }
  X[0] = mad_lo_cc(P::mod(0), m, X[0]);
  X[1] = madc_hi_cc(P::mod(0), m, X[1]);
#pragma unroll
  for (int j = 2; j < N; j += 2) {
    X[j] = madc_lo_cc(P::mod(j), m, X[j]);
    X[j + 1] = madc_hi_cc(P::mod(j), m, X[j + 1]);
  }
  Y[N - 1] = addc(Y[N - 1], 0u);
}

template <class P>
PCGPU_HD constexpr bool mont_mul2_supported() { return 3ull * ((unsigned long long)P::mod(P::N - 1) + 1) <= (1ull << 32); }

template <class P>
PCGPU_DEV Fp<P> mont_mul2(const Fp<P> &a, const Fp<P> &b, const Fp<P> &c, const Fp<P> &d) {
  constexpr int N = P::N;
  static_assert(mont_mul2_supported<P>(), "sum-of-products reduction needs 3p < 2^(32N) (not true for BLS12-381 Fr)");
  uint32_t X[N], Y[N];
  mont_row2<P, true>(X, Y, a.l, b.l[0], c.l, d.l[0]);
  mont_row2<P, false>(Y, X, a.l, b.l[1], c.l, d.l[1]);
#pragma unroll
  for (int i = 2; i < N; i += 2) {
    mont_row2<P, false>(X, Y, a.l, b.l[i], c.l, d.l[i]);
    mont_row2<P, false>(Y, X, a.l, b.l[i + 1], c.l, d.l[i + 1]);
  }
  Fp<P> r;
  r.l[0] = add_cc(X[0], Y[1]);
#pragma unroll
  for (int i = 1; i < N - 1; i++) r.l[i] = addc_cc(X[i], Y[i + 1]);
  r.l[N - 1] = addc(X[N - 1], 0u);
  fp_reduce_once<P>(r.l);
  fp_reduce_once<P>(r.l);
  return r;
}

// ---- dedicated squaring: product scanning with a three-limb column accumulator ----
// a^2 needs N(N+1)/2 limb products instead of N^2 (the off-diagonal ones are computed once and doubled); the
// Montgomery reduction is done column-wise on the double-width square.  222 wide multiplies for N = 12 instead of 288
// (-23 %), at the price of one extra carry add per product (ALU pipe, which has slack in every kernel here).
// acc3: (c0, c1, c2) += x * y
#define PCGPU_ACC3_MAD(c0, c1, c2, x, y) do { c0 = mad_lo_cc(x, y, c0); c1 = madc_hi_cc(x, y, c1); c2 = addc(c2, 0u); } while (0)
template <class P>
PCGPU_DEV Fp<P> mont_sqr(const Fp<P> &a) {
  constexpr int N = P::N;
  uint32_t t[2 * N];
  // phase A: u = sum_{i<j} a_i a_j 2^(32(i+j))   (column k collects the pairs with i + j = k)
  {
    uint32_t c0 = 0, c1 = 0, c2 = 0;
    t[0] = 0;
#pragma unroll
    for (int k = 1; k <= 2 * N - 3; k++) {
#pragma unroll
      for (int i = 0; i < N; i++) {
        const int j = k - i;
        if (i < j && j < N) PCGPU_ACC3_MAD(c0, c1, c2, a.l[i], a.l[j]);
      }
      t[k] = c0; c0 = c1; c1 = c2; c2 = 0;
    }
    t[2 * N - 2] = c0; t[2 * N - 1] = c1;
  }
  // phase B: t = 2u + sum_i a_i^2 2^(64 i)
  {
    uint32_t top = 0;   // bit shifted out of the previous limb
#pragma unroll
    for (int k = 0; k < 2 * N; k++) { uint32_t v = t[k]; t[k] = (v << 1) | top; top = v >> 31; }
    // add the diagonal squares with one carry chain
    t[0] = add_cc(t[0], mul_lo(a.l[0], a.l[0]));
    t[1] = addc_cc(t[1], mul_hi(a.l[0], a.l[0]));
#pragma unroll
    for (int i = 1; i < N; i++) {
      t[2 * i] = addc_cc(t[2 * i], mul_lo(a.l[i], a.l[i]));
      t[2 * i + 1] = addc_cc(t[2 * i + 1], mul_hi(a.l[i], a.l[i]));
    }
  }
  // phase C: Montgomery reduction of the 2N-limb square, column by column (m_k chosen so that column k vanishes)
  uint32_t m[N];
  Fp<P> r;
  {
    uint32_t c0 = 0, c1 = 0, c2 = 0;
#pragma unroll
    for (int k = 0; k < N; k++) {
#pragma unroll
      for (int i = 0; i < k; i++) PCGPU_ACC3_MAD(c0, c1, c2, m[i], P::mod(k - i));
      c0 = add_cc(c0, t[k]); c1 = addc_cc(c1, 0u); c2 = addc(c2, 0u);
      m[k] = c0 * P::M0;
      PCGPU_ACC3_MAD(c0, c1, c2, m[k], P::mod(0));   // c0 becomes 0
      c0 = c1; c1 = c2; c2 = 0;
    }
#pragma unroll
    for (int k = N; k < 2 * N; k++) {
#pragma unroll
      for (int i = k - N + 1; i < N; i++) PCGPU_ACC3_MAD(c0, c1, c2, m[i], P::mod(k - i));
      c0 = add_cc(c0, t[k]); c1 = addc_cc(c1, 0u); c2 = addc(c2, 0u);
      r.l[k - N] = c0;
      c0 = c1; c1 = c2; c2 = 0;
    }
    // a^2 / R + correction < 2p < 2^(32N): nothing is left in the accumulator
  }
  fp_reduce_once<P>(r.l);
  return r;
}

#ifdef PCGPU_USE_REF_MUL
template <class P> PCGPU_DEV Fp<P> fp_mul(const Fp<P> &a, const Fp<P> &b) { return mont_mul_ref<P>(a, b); }
template <class P> PCGPU_DEV Fp<P> fp_mul2(const Fp<P> &a, const Fp<P> &b, const Fp<P> &c, const Fp<P> &d) { return fp_add<P>(mont_mul_ref<P>(a, b), mont_mul_ref<P>(c, d)); }
#else
template <class P> PCGPU_DEV Fp<P> fp_mul(const Fp<P> &a, const Fp<P> &b) { return mont_mul<P>(a, b); }
template <class P> PCGPU_DEV Fp<P> fp_mul2(const Fp<P> &a, const Fp<P> &b, const Fp<P> &c, const Fp<P> &d) { return mont_mul2<P>(a, b, c, d); }
#endif
#if defined(PCGPU_USE_REF_MUL) || defined(PCGPU_NO_SQR)
template <class P> PCGPU_DEV Fp<P> fp_sqr(const Fp<P> &a) { return fp_mul<P>(a, a); }
#else
template <class P> PCGPU_DEV Fp<P> fp_sqr(const Fp<P> &a) { return mont_sqr<P>(a); }
#endif

// Montgomery -> canonical (F::into_bigint, kzg10/mod.rs:463-470): multiply by 1
template <class P>
PCGPU_DEV Fp<P> fp_from_mont(const Fp<P> &a) {
  Fp<P> o = Fp<P>::zero(); o.l[0] = 1;
  return fp_mul<P>(a, o);
}
template <class P>
PCGPU_DEV Fp<P> fp_to_mont(const Fp<P> &a) { return fp_mul<P>(a, Fp<P>::r2()); }

// a^(p-2) by square-and-multiply over the bits of p-2 (inverse of 0 is 0)
template <class P>
PCGPU_DEV Fp<P> fp_inv(const Fp<P> &a) {
  constexpr int N = P::N;
  uint32_t e[N];  // p - 2 (the low limb of p may be 1, so propagate the borrow)
  uint32_t borrow = 2;
  for (int i = 0; i < N; i++) { uint32_t m = P::mod(i); e[i] = m - borrow; borrow = m < borrow ? 1u : 0u; }
  Fp<P> acc = Fp<P>::one();
  for (int i = N * 32 - 1; i >= 0; i--) {
    acc = fp_sqr<P>(acc);
    if ((e[i / 32] >> (i % 32)) & 1) acc = fp_mul<P>(acc, a);
  }
  return acc;
}

// ---- inversion by Kaliski's "almost Montgomery inverse" (binary extended GCD) ----
// Phase 1 runs on shifts / adds / subtracts only (the ALU pipe, idle while the integer-multiply pipe is the
// bottleneck) and yields x = a^-1 * 2^k (mod p), bits(p) <= k <= 2 bits(p); one Montgomery product by
// pow2[64N/2.. ] = 2^e * R (e = 32*2N - k) turns it into the Montgomery-form inverse.  ~540 iterations of ~15N
// instructions instead of ~460 modular multiplications for the Fermat exponentiation.
// pow2: table of 2^e * R mod p for e = 0 .. 64N (device memory, built once per context; see Pow2TableBody).
PCGPU_DEV uint32_t funnel_r1(uint32_t lo, uint32_t hi) {
#ifdef __CUDA_ARCH__
  return __funnelshift_r(lo, hi, 1);
#else
  return (lo >> 1) | (hi << 31);
#endif
}
PCGPU_DEV uint32_t funnel_l1(uint32_t lo, uint32_t hi) {
#ifdef __CUDA_ARCH__
  return __funnelshift_l(lo, hi, 1);
#else
  return (hi << 1) | (lo >> 31);
#endif
}

PCGPU_DEV uint32_t ctz32(uint32_t x) {
#ifdef __CUDA_ARCH__
  return (uint32_t)(__ffs((int)x) - 1);
#else
  return (uint32_t)__builtin_ctz(x);
#endif
}
PCGPU_DEV uint32_t funnel_r(uint32_t lo, uint32_t hi, uint32_t sh) {   // (hi:lo >> sh) low word, 0 < sh < 32
#ifdef __CUDA_ARCH__
  return __funnelshift_r(lo, hi, sh);
#else
  return (lo >> sh) | (hi << (32 - sh));
#endif
}
PCGPU_DEV uint32_t funnel_l(uint32_t lo, uint32_t hi, uint32_t sh) {   // (hi:lo << sh) high word, 0 < sh < 32
#ifdef __CUDA_ARCH__
  return __funnelshift_l(lo, hi, sh);
#else
  return (hi << sh) | (lo >> (32 - sh));
#endif
}

// Both u and v are kept odd: every iteration is one subtraction followed by the removal of ALL trailing zero bits
// (several Kaliski halving steps at once), about 0.7 * bits(p) iterations.
template <class P>
PCGPU_DEV Fp<P> fp_inv_gcd(const Fp<P> &a, const uint32_t *pow2) {
  constexpr int N = P::N;
  if (a.is_zero()) return a;
  uint32_t u[N], v[N], r[N], s[N];
#pragma unroll
  for (int i = 0; i < N; i++) { u[i] = P::mod(i); v[i] = a.l[i]; r[i] = 0; s[i] = 0; }
  s[0] = 1;
  uint32_t k = 0;
  // make v odd (r = 0, so its doublings are no-ops)
  while (!(v[0] & 1u)) {
    uint32_t sh = v[0] ? ctz32(v[0]) : 31u;
    if (sh > 31u) sh = 31u;
#pragma unroll
    for (int i = 0; i < N - 1; i++) v[i] = funnel_r(v[i], v[i + 1], sh);
    v[N - 1] >>= sh;
    k += sh;
  }
  for (;;) {
    // gt = u > v  (borrow of v - u);  eq when u == v
    uint32_t t = sub_cc(v[0], u[0]), diff = t;
#pragma unroll
    for (int i = 1; i < N; i++) { t = subc_cc(v[i], u[i]); diff |= t; }
    const bool gt = subc(0u, 0u) != 0;
    if (diff == 0) {                         // u == v == 1: last step (v = 0; s += r; r *= 2)
      r[0] = add_cc(r[0], r[0]);             // only r is used afterwards: r <- 2r
#pragma unroll
      for (int i = 1; i < N - 1; i++) r[i] = addc_cc(r[i], r[i]);
      r[N - 1] = addc(r[N - 1], r[N - 1]);
      k++;
      break;
    }
    uint32_t X[N], Y[N], Pp[N], Qq[N];       // X = the larger of (u, v); (Pp, Qq) = (r, s) in the matching order
#pragma unroll
    for (int i = 0; i < N; i++) {
      X[i] = gt ? u[i] : v[i]; Y[i] = gt ? v[i] : u[i];
      Pp[i] = gt ? r[i] : s[i]; Qq[i] = gt ? s[i] : r[i];
    }
    X[0] = sub_cc(X[0], Y[0]);
#pragma unroll
    for (int i = 1; i < N - 1; i++) X[i] = subc_cc(X[i], Y[i]);
    X[N - 1] = subc(X[N - 1], Y[N - 1]);
    Pp[0] = add_cc(Pp[0], Qq[0]);
#pragma unroll
    for (int i = 1; i < N - 1; i++) Pp[i] = addc_cc(Pp[i], Qq[i]);
    Pp[N - 1] = addc(Pp[N - 1], Qq[N - 1]);
    // X >>= tz, Qq <<= tz, k += tz   (X is even and non-zero)
    do {
      uint32_t sh = X[0] ? ctz32(X[0]) : 31u;
      if (sh > 31u) sh = 31u;
      if (sh == 0) break;
#pragma unroll
      for (int i = 0; i < N - 1; i++) X[i] = funnel_r(X[i], X[i + 1], sh);
      X[N - 1] >>= sh;
#pragma unroll
      for (int i = N - 1; i > 0; i--) Qq[i] = funnel_l(Qq[i - 1], Qq[i], sh);
      Qq[0] <<= sh;
      k += sh;
    } while (!(X[0] & 1u));
#pragma unroll
    for (int i = 0; i < N; i++) {
      u[i] = gt ? X[i] : u[i]; v[i] = gt ? v[i] : X[i];
      r[i] = gt ? Pp[i] : Qq[i]; s[i] = gt ? Qq[i] : Pp[i];
    }
  }
  // x = p - (r mod p) = a^-1 * 2^k
  fp_reduce_once<P>(r);
  Fp<P> x;
  x.l[0] = sub_cc(P::mod(0), r[0]);
#pragma unroll
  for (int i = 1; i < N - 1; i++) x.l[i] = subc_cc(P::mod(i), r[i]);
  x.l[N - 1] = subc(P::mod(N - 1), r[N - 1]);
  fp_reduce_once<P>(x.l);
  Fp<P> corr;
  const uint32_t idx = 2u * 32u * N - k;   // multiply by 2^(2*32N - k) * R  (Montgomery product removes one R)
#pragma unroll
  for (int i = 0; i < N; i++) corr.l[i] = pow2[(size_t)idx * N + i];
  return fp_mul<P>(x, corr);
}

// pow2[e] = 2^e * R mod p, e = 0 .. 64N  (one thread)
template <class P>
struct Pow2TableBody {
  uint32_t *table;
  PCGPU_DEV void operator()(size_t) const {
    Fp<P> t = Fp<P>::one();
    for (uint32_t e = 0; e <= 64u * P::N; e++) {
#pragma unroll
      for (int i = 0; i < P::N; i++) table[(size_t)e * P::N + i] = t.l[i];
      t = fp_dbl<P>(t);
    }
  }
};

// multiply by a small constant (2, 3, 4, 8) through additions
template <class P> PCGPU_DEV Fp<P> fp_mul3(const Fp<P> &a) { return fp_add<P>(fp_dbl<P>(a), a); }

}  // namespace pcgpu
