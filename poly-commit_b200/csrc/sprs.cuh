// Sparse (CSC) matrix-vector products over Fr and the Brakedown row encoding built from them -- the one step of the
// Brakedown commit that is not shared with Ligero (MultilinearBrakedown::encode, multilinear_brakedown/mod.rs:56-84):
//   SprsMat::row_mul        out[j] = sum_{k in col j} v[col_ind[k]] * val[k]          linear_codes/utils.rs:41-52
//   naive_reed_solomon      cw[s..oe] = evaluations at x = 1, 2, ..., oe - s of the polynomial with coefficients
//                           cw[s..ie] (lowest first), by Horner's rule                multilinear_brakedown/mod.rs:111-122
//
// Every kernel is batched over the rows of the polynomial matrix: all rows share one matrix, so one (col_ind, val) pair is
// applied to every row.  Operands are addressed with an element stride and a row stride, which lets the same body read and
// write the encoder's work buffer (element-major / row-minor: element k of row r at k * n_rows + r, so the gather of input
// index k for all rows is one contiguous segment), a row-major matrix (Matrix<F>) and a batch of plain vectors.
//
// Threads are (output column j, row r) with r fastest: with >= 32 rows a warp covers 32 rows of one column (the column's
// col_ind / val are broadcast, the gather of the work buffer is 1 KB contiguous); with fewer rows a warp spans
// 32 / n_rows columns, so 1- and 2-row encodes (the verifier's re-encode, the 2^12 shape) still fill the warp.
#pragma once
#include "frops.cuh"
#include "rt.cuh"

namespace pcgpu {

enum { SPRS_MAX_LEVELS = 16 };

// one CSC product inside a launch: outputs [out_base, out_base + cols) of every row from inputs [in_base, in_base + lim)
struct SprsLevel {
  const uint32_t *ind_ptr;   // cols + 1 offsets into col_ind / val
  const uint32_t *col_ind;   // row index of each nonzero (< lim: entries that would read a zero were dropped on upload)
  const uint32_t *val;       // Montgomery Fr, 8 words each
  uint64_t in_base, out_base, cols, first;   // first: index of this level's first output column in the launch
};

// all `nlev` levels of one launch read `src` and write `dst`; their outputs are disjoint
template <class R>
struct SprsRowMulBody {
  SprsLevel lev[SPRS_MAX_LEVELS];
  uint32_t nlev;
  const uint32_t *src; uint64_t src_es, src_rs;   // element k of row r at k * src_es + r * src_rs
  uint32_t *dst; uint64_t dst_es, dst_rs;
  uint64_t n_rows;
  PCGPU_KERNEL_DEV void operator()(size_t tid) const {
    const uint64_t r = tid % n_rows, g = tid / n_rows;
    uint32_t li = 0;
    while (li + 1 < nlev && g >= lev[li + 1].first) li++;
    const SprsLevel &L = lev[li];
    const uint64_t j = g - L.first;
    const uint64_t lo = L.ind_ptr[j], hi = L.ind_ptr[j + 1];
    const uint32_t *s = src + 8 * (L.in_base * src_es + r * src_rs);   // 8 words per element
    Fp<R> acc = Fp<R>::zero();
    uint64_t k = lo;
    for (; k + 2 <= hi; k += 2)      // pairs of nonzeros: one reduction per two products (fr_dot2)
      acc = fp_add<R>(acc, fr_dot2<R>(load_fr<R>(s, (uint64_t)L.col_ind[k] * src_es), load_fr<R>(L.val, k),
                                      load_fr<R>(s, (uint64_t)L.col_ind[k + 1] * src_es), load_fr<R>(L.val, k + 1)));
    if (k < hi) acc = fp_add<R>(acc, fp_mul<R>(load_fr<R>(s, (uint64_t)L.col_ind[k] * src_es), load_fr<R>(L.val, k)));
    store_fr<R>(dst, (L.out_base + j) * dst_es + r * dst_rs, acc);
  }
};

// naive_reed_solomon on the work buffer: output t (x = t + 1) of row r from the `n_in` coefficients in `coef`
// (element-major copy of cw[s..ie]), written to element s + t
template <class R>
struct NaiveRsBody {
  const uint32_t *coef; uint64_t n_in; uint32_t *work; uint64_t s, n_rows;
  PCGPU_KERNEL_DEV void operator()(size_t tid) const {
    const uint64_t r = tid % n_rows, t = tid / n_rows;
    Fp<R> x = Fp<R>::zero();
    x.l[0] = (uint32_t)(t + 1); x.l[1] = (uint32_t)((t + 1) >> 32);
    x = fp_mul<R>(x, Fp<R>::r2());    // to Montgomery form
    Fp<R> acc = Fp<R>::zero();
    for (uint64_t j = n_in; j-- > 0;) acc = fp_add<R>(fp_mul<R>(acc, x), load_fr<R>(coef, j * n_rows + r));
    store_fr<R>(work, (s + t) * n_rows + r, acc);
  }
};

// strided copy of every row: element k of row r from src[k * src_es + r * src_rs] to
// dst[k * dst_es + r * dst_rs]; thread (k, r) with r fastest
struct FrStridedCopyBody {
  const uint32_t *src; uint64_t src_es, src_rs; uint32_t *dst; uint64_t dst_es, dst_rs; uint64_t n_rows;
  PCGPU_KERNEL_DEV void operator()(size_t tid) const {
    const uint64_t r = tid % n_rows, k = tid / n_rows;
    const u32x4 *p = reinterpret_cast<const u32x4 *>(src) + 2 * (k * src_es + r * src_rs);
    u32x4 *q = reinterpret_cast<u32x4 *>(dst) + 2 * (k * dst_es + r * dst_rs);
    q[0] = p[0]; q[1] = p[1];
  }
};

}  // namespace pcgpu
