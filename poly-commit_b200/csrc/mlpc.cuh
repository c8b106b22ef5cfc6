// MultilinearPC (XZZPD19, multilinear_pc/mod.rs) on the device: the key's pair folding at registration and the open's fold
// chain.  The open's G2 MSMs run through the bucket pipeline / small-MSM kernel of msm.cuh and msm_small.cuh.
//
// open (:131-168), level i = 0 .. nv-1, k = nv - i, x_i = point[i]:
//   q_i[b]  = r[2b+1] - r[2b]                 r'[b] = r[2b] (1 - x_i) + r[2b+1] x_i = r[2b] + x_i q_i[b]
//   pi_i    = sum_x q_i[x >> 1] H_i[x]  =  sum_b q_i[b] (H_i[2b] + H_i[2b+1])
// so the key stores the pair-folded bases H'_i[b] = H_i[2b] + H_i[2b+1] and each open runs 2^nv - 1 G2 terms instead of
// 2^(nv+1) - 2.  The identity holds for any key (an honest key has H'_i = H_{i+1}, which is not relied on).
#pragma once
#include "frops.cuh"
#include "msm.cuh"

namespace pcgpu {

// level i of the fold chain: r_in has 2 m elements, q and r_out m (Montgomery Fr); x = point[i]
template <class R>
struct MlpcFoldBody {
  const uint32_t *r_in; const uint32_t *point; uint32_t i; uint32_t *q; uint32_t *r_out;
  PCGPU_KERNEL_DEV void operator()(size_t b) const {
    const Fp<R> a0 = load_fr<R>(r_in, 2 * b), a1 = load_fr<R>(r_in, 2 * b + 1);
    const Fp<R> d = fp_sub<R>(a1, a0);
    store_fr<R>(q, b, d);
    store_fr<R>(r_out, b, fp_add<R>(a0, fp_mul<R>(load_fr<R>(point, i), d)));
  }
};

// out[b] = H[2b] + H[2b+1], affine (identity = (0, 0)); every exceptional case of the addition (identity operands, P + P,
// P + (-P)) is handled by xyzz_madd
template <class C>
struct PairFoldBasesBody {
  const Affine<C> *in; Affine<C> *out;
  PCGPU_KERNEL_DEV void operator()(size_t b) const {
    XYZZ<C> p = xyzz_from_affine<C>(load_affine<C>(in + 2 * b));
    xyzz_madd<C>(p, load_affine<C>(in + 2 * b + 1), false);
    out[b] = xyzz_to_affine<C>(p);
  }
};

// first folded base of level i in the key (levels hold 2^(nv-1), 2^(nv-2), ..., 1 points): 2^nv - 2^(nv-i); the open's q
// buffer uses the same offsets
inline size_t mlpc_level_offset(uint32_t nv, uint32_t i) { return ((size_t)1 << nv) - ((size_t)1 << (nv - i)); }

}  // namespace pcgpu
