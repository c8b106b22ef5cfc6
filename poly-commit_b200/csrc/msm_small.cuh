// Small multi-scalar multiplications (n <= SMALL_MAX_N) in ONE launch.
//
// The bucket pipeline of msm.cuh is built for 2^16 .. 2^26 terms: a dozen launches, a counting sort and a host tail over
// S * c bit planes have a fixed cost however few points there are (at 2^10 on BLS12-381 the host alone combines 26 windows
// x 10 planes).  The callers with few terms -- the late rounds of the IPA
// halving loop (ipa_pc/mod.rs:665-711), the verifier-side combinations (hyrax/mod.rs:498-504, kzg10/mod.rs:322-373), cfg1's
// degree-2^10 commitments (kzg10/mod.rs:175-178) -- run here instead:
//   grid  = (#problems) x W x split blocks (the problems are a device array: the IPA's l and r, or Hyrax's 2 per checked proof), W = ceil((bits + 2) / c) windows of c = 6 bits; a window's terms are divided
//           among `split` blocks (1 below 512 terms, else 3: 129 blocks, one wave on the 132 SMs of an H100), each producing a partial U_w
//   block = 256 threads = 32 buckets (digit magnitudes 1..32) x 8 slices of the scalars
//   1. digits: signed digits d in [-32, 31] by the offset trick: the base-2^c digits e_w of s + K, K = sum_w 2^(c-1) 2^(cw),
//      give d_w = e_w - 2^(c-1) with sum_w d_w 2^(cw) = s -- every window is computed independently, no carry chain
//   2. every thread walks its slice for the digits of its magnitude and adds the (conditionally negated) points, XYZZ
//   3. slices are summed (tree), the window value  U_w = sum_k k B_k  is formed as the sum of the suffix sums of the
//      buckets (log-step scan + tree: 13 dependent additions), and ONE point per window goes back to the host,
//      which finishes with the c * W doublings of  sum_w 2^(cw) U_w  (host_ec.hpp, combine_windows).
// An optional extra (base, scalar) pair held in device memory rides along as term n: the IPA's  + h' * <a, z>  without a
// round trip of the inner product through the host.
#pragma once
#include "msm.cuh"

namespace pcgpu {

enum { SMALL_C = 6, SMALL_NB = 32, SMALL_SLICES = 8, SMALL_BLOCK = 256, SMALL_MAX_N = 4096, SMALL_MAX_PROB = 1024, SMALL_SPLIT = 3, SMALL_SPLIT_MIN_N = 512 };

template <class C>
struct MsmSmallProblem {
  const Affine<C> *bases; const uint32_t *scalars;            // n terms
  const Affine<C> *extra_base; const uint32_t *extra_scalar;  // optional term n (device pointers), same scalar form
  uint32_t n;
};

template <class R> PCGPU_HD constexpr uint32_t small_windows() { return (R::BITS + 2 + SMALL_C - 1) / SMALL_C; }

// signed digit of window w of the canonical scalar s (8 words): digit of (s + K) minus 2^(c-1)
PCGPU_DEV int small_digit(const uint32_t *s, const uint32_t *K, uint32_t w) {
  // t = s + K over 9 words; only the words holding bits [c w, c w + c) are needed, but the carry comes from below
  uint32_t t[9];
  uint64_t carry = 0;
  for (int j = 0; j < 9; j++) {
    uint64_t v = (uint64_t)(j < 8 ? s[j] : 0u) + K[j] + carry;
    t[j] = (uint32_t)v; carry = v >> 32;
  }
  const uint32_t pos = w * SMALL_C, j = pos >> 5, sh = pos & 31;
  uint64_t two = (uint64_t)t[j] | ((uint64_t)(j + 1 < 9 ? t[j + 1] : 0u) << 32);
  return (int)((two >> sh) & ((1u << SMALL_C) - 1)) - (1 << (SMALL_C - 1));
}

template <class C>
struct MsmSmallBody {
  const MsmSmallProblem<C> *prob;   // device array, one entry per problem
  uint32_t mont;         // scalars are Montgomery Fr (converted in the digit pass) / canonical
  uint32_t split;        // blocks per window; block q of a window takes the terms i = q (mod split)
  XYZZ<C> *out;          // out[(p * W + w) * split + q] = partial U_w of problem p
  uint32_t *err;         // bit 0: a canonical scalar >= r
  PCGPU_KERNEL_DEV void operator()(size_t blk, uint32_t *smem) const {
    using R = typename C::Fr;
    constexpr uint32_t W = small_windows<R>();
    const uint32_t q = (uint32_t)(blk % split), w = (uint32_t)((blk / split) % W), p = (uint32_t)(blk / ((size_t)split * W));
    const MsmSmallProblem<C> &P = prob[p];
    const uint32_t all = P.n + (P.extra_base ? 1u : 0u);
    const uint32_t total = all > q ? (all - q + split - 1) / split : 0u;      // this block's terms: g = q + split * i
    int8_t *dig = reinterpret_cast<int8_t *>(smem);
    XYZZ<C> *sh = reinterpret_cast<XYZZ<C> *>(smem + (SMALL_MAX_N + 16) / 4);
    uint32_t K[9];
    for (int j = 0; j < 9; j++) K[j] = 0;
    for (uint32_t v = 0; v < W; v++) { uint32_t pos = v * SMALL_C + SMALL_C - 1; K[pos >> 5] |= 1u << (pos & 31); }
    PCGPU_BLOCK_FOR(i, total) {
      const uint32_t g = q + split * i;
      Fp<R> s = load_fr<R>(g < P.n ? P.scalars : P.extra_scalar, g < P.n ? g : 0);
      if (mont) s = fp_from_mont<R>(s);
      {   // not a reduced field element (>= r): rejected like the bucket pipeline does (load_scalar)
        bool lt_r = false, decided = false;
        for (int j = 7; j >= 0; j--) if (!decided && s.l[j] != R::mod(j)) { lt_r = s.l[j] < R::mod(j); decided = true; }
        if (!lt_r) rt::atomic_or(err, 1u);
      }
      dig[i] = (int8_t)small_digit(s.l, K, w);
    }
    PCGPU_BLOCK_SYNC();
    PCGPU_BLOCK_FOR(t, SMALL_BLOCK) {
      const int mag = (int)(t % SMALL_NB) + 1;
      XYZZ<C> acc = XYZZ<C>::inf();
      uint32_t i = t / SMALL_NB;
      for (;;) {
        int d = 0;
        while (i < total) { d = dig[i]; if (d == mag || d == -mag) break; i += SMALL_SLICES; }
        const bool has = i < total;
        if (!PCGPU_WARP_ANY(has)) break;          // uniform exit; the vote also reconverges the lanes before the addition
        if (has) {
          const uint32_t g = q + split * i;
          Affine<C> a = load_affine<C>(g < P.n ? P.bases + g : P.extra_base);
          xyzz_madd<C>(acc, a, d < 0);
          i += SMALL_SLICES;
        }
      }
      sh[t] = acc;
    }
    PCGPU_BLOCK_SYNC();
    for (uint32_t half = SMALL_SLICES / 2; half >= 1; half >>= 1) {
      PCGPU_BLOCK_FOR(t, SMALL_NB * half) { XYZZ<C> x = sh[t], y = sh[t + SMALL_NB * half]; xyzz_add_ool<C>(x, y); sh[t] = x; }
      PCGPU_BLOCK_SYNC();
    }
    // suffix sums S_b = sum_{m >= b} B_m (ping-pong between the two halves of sh[0 .. 2 NB)), then their total
    XYZZ<C> *src = sh, *dst = sh + SMALL_NB;
    for (uint32_t d = 1; d < SMALL_NB; d <<= 1) {
      PCGPU_BLOCK_FOR(b, SMALL_NB) { XYZZ<C> x = src[b]; if (b + d < SMALL_NB) { XYZZ<C> y = src[b + d]; xyzz_add_ool<C>(x, y); } dst[b] = x; }
      PCGPU_BLOCK_SYNC();
      XYZZ<C> *tmp = src; src = dst; dst = tmp;
    }
    for (uint32_t half = SMALL_NB / 2; half >= 1; half >>= 1) {
      PCGPU_BLOCK_FOR(b, half) { XYZZ<C> x = src[b], y = src[b + half]; xyzz_add_ool<C>(x, y); src[b] = x; }
      PCGPU_BLOCK_SYNC();
    }
    PCGPU_BLOCK_FOR(b, 1) { store_xyzz<C>(out + blk, src[0]); }
  }
};

template <class C> inline size_t msm_small_smem() { return (SMALL_MAX_N + 16) / 4 * 4 + (size_t)SMALL_BLOCK * sizeof(XYZZ<C>); }

}  // namespace pcgpu
