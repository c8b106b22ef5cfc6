// HyraxPC (poly-commit/src/hyrax) on the device: the scalar work around the comb rows and the small MSMs.
//
//   HyraxTransposeBody   [T | r]: T[row][col] = evals[col * dim + row] (flat_to_matrix_column_major, hyrax/utils.rs:13-21),
//                        the commitment randomness r_row as column dim -- the resident HyraxCommitmentState (mod.rs:248-251)
//   HyraxTensorBody      l = tensor_prime(point_lower), r = tensor_prime(point_upper) of the reversed point (mod.rs:299-307,
//                        utils.rs:27-39)
//   HyraxOpenRowsBody    eval = <lt, r>, b = <r, d> and the comb rows of com_eval, com_d, com_b (mod.rs:356-378)
//   HyraxCheckRowsBody   <r, z>, the comb rows of both left-hand sides and c * l (mod.rs:490-505)
// The row product lt = l^T [T | r] is fr_row_mul_run (frops.cuh).  Every element is Montgomery Fr.
#pragma once
#include "frops.cuh"

namespace pcgpu {

enum { HYRAX_TILE = 32, HYRAX_TILE_PITCH = 33 * 8, HYRAX_BLOCK = 256 };

inline size_t hyrax_transpose_smem() { return (size_t)HYRAX_TILE * HYRAX_TILE_PITCH * 4; }

// block (by, bx) moves the 32 x 32 tile of rows [32 by, ..) and columns [32 bx, ..) of T through shared memory: the reads run
// along evals' contiguous rows-within-a-column, the writes along T's contiguous columns-within-a-row.  Blocks of column 0 also
// write their rows' randomness into column dim.
struct HyraxTransposeBody {
  const uint32_t *evals; const uint32_t *rand; uint32_t *block; uint32_t dim, tiles;
  PCGPU_KERNEL_DEV void operator()(size_t b, uint32_t *smem) const {
    const uint32_t r0 = (uint32_t)(b / tiles) * HYRAX_TILE, c0 = (uint32_t)(b % tiles) * HYRAX_TILE;
    const size_t stride = (size_t)dim + 1;
    PCGPU_BLOCK_FOR(i, HYRAX_TILE * HYRAX_TILE * 8) {   // i = (cc, rr, limb): consecutive threads read consecutive words
      const uint32_t cc = i / (HYRAX_TILE * 8), w = i % (HYRAX_TILE * 8), rr = w / 8, l = w % 8;
      if (c0 + cc < dim && r0 + rr < dim) smem[cc * HYRAX_TILE_PITCH + w] = evals[((size_t)(c0 + cc) * dim + r0 + rr) * 8 + l];
    }
    PCGPU_BLOCK_SYNC();
    PCGPU_BLOCK_FOR(i, HYRAX_TILE * HYRAX_TILE * 8) {   // i = (rr, cc, limb)
      const uint32_t rr = i / (HYRAX_TILE * 8), w = i % (HYRAX_TILE * 8), cc = w / 8, l = w % 8;
      if (c0 + cc < dim && r0 + rr < dim) block[((size_t)(r0 + rr) * stride + c0 + cc) * 8 + l] = smem[cc * HYRAX_TILE_PITCH + rr * 8 + l];
    }
    if (c0 == 0) {
      PCGPU_BLOCK_FOR(i, HYRAX_TILE * 8) {
        const uint32_t rr = i / 8, l = i % 8;
        if (r0 + rr < dim) block[((size_t)(r0 + rr) * stride + dim) * 8 + l] = rand[(size_t)(r0 + rr) * 8 + l];
      }
    }
  }
};

// out[0 .. dim) = l, out[dim .. 2 dim) = r, dim = 2^half.  With point_rev = reverse(point), point_lower = point_rev[half ..] and
// tensor_prime putting its first value on the top index bit, bit b of an index of l selects point[b] (1 - point[b] when clear)
// and bit b of an index of r selects point[half + b].
template <class R>
struct HyraxTensorBody {
  const uint32_t *point; uint32_t half; uint32_t *out;
  PCGPU_KERNEL_DEV void operator()(size_t t) const {
    const size_t dim = (size_t)1 << half, idx = t % dim;
    const uint32_t base = t < dim ? 0u : half;
    const Fp<R> one = Fp<R>::one();
    Fp<R> acc = one;
    for (uint32_t b = 0; b < half; b++) {
      const Fp<R> p = load_fr<R>(point, base + b);
      acc = fp_mul<R>(acc, (idx >> b) & 1 ? p : fp_sub<R>(one, p));
    }
    store_fr<R>(out, t, acc);
  }
};

// sum_{i < n} term(i) over one block of HYRAX_BLOCK threads; every thread returns the sum.  smem: 8 * HYRAX_BLOCK words.
template <class R, class Term>
PCGPU_DEV Fp<R> hyrax_block_sum(uint32_t *smem, size_t n, Term term) {
  PCGPU_BLOCK_FOR(t, HYRAX_BLOCK) {
    Fp<R> v = Fp<R>::zero();
    for (size_t i = t; i < n; i += HYRAX_BLOCK) v = fp_add<R>(v, term(i));
#pragma unroll
    for (int l = 0; l < 8; l++) smem[l * HYRAX_BLOCK + t] = v.l[l];
  }
  PCGPU_BLOCK_SYNC();
  for (uint32_t half = HYRAX_BLOCK / 2; half >= 1; half >>= 1) {
    PCGPU_BLOCK_FOR(t, half) {
      Fp<R> x, y;
#pragma unroll
      for (int l = 0; l < 8; l++) { x.l[l] = smem[l * HYRAX_BLOCK + t]; y.l[l] = smem[l * HYRAX_BLOCK + t + half]; }
      x = fp_add<R>(x, y);
#pragma unroll
      for (int l = 0; l < 8; l++) smem[l * HYRAX_BLOCK + t] = x.l[l];
    }
    PCGPU_BLOCK_SYNC();
  }
  Fp<R> s;
#pragma unroll
  for (int l = 0; l < 8; l++) s.l[l] = smem[l * HYRAX_BLOCK];
  PCGPU_BLOCK_SYNC();   // smem is free again
  return s;
}

// one row [a, 0, ..., 0, z] of n + 1 scalars: a * com_key[0] + z * h over the key com_key || h
template <class R>
PCGPU_DEV void hyrax_singleton_row(uint32_t *row, size_t n, const Fp<R> &a, const uint32_t *z) {
  PCGPU_BLOCK_FOR(i, n + 1) store_fr<R>(row, i, i == 0 ? a : i == n ? load_fr<R>(z, 0) : Fp<R>::zero());
}

// block p, polynomial p: lt = the first dim elements of lt_all + p (dim + 1), blinds + p (dim + 3) = r_eval || d || r_d || r_b.
// rows + 3 p (dim + 1 each) = [eval, 0.., r_eval], [d | r_d], [b, 0.., r_b]; eval_out[p] = eval.  (n = dim for the nv = 0
// case too: the singleton rows are then [eval, r_eval].)
template <class R>
struct HyraxOpenRowsBody {
  const uint32_t *lt_all; const uint32_t *tensor; const uint32_t *blinds; uint32_t *rows; uint32_t *eval_out; uint32_t dim;
  PCGPU_KERNEL_DEV void operator()(size_t p, uint32_t *smem) const {
    const size_t n = dim, w = n + 1;
    const uint32_t *lt = lt_all + 8 * w * p, *r = tensor + 8 * n, *bl = blinds + 8 * (n + 3) * p, *d = bl + 8;
    uint32_t *row = rows + 8 * 3 * w * p;
    const Fp<R> eval = hyrax_block_sum<R>(smem, n, [&](size_t i) { return fp_mul<R>(load_fr<R>(lt, i), load_fr<R>(r, i)); });
    const Fp<R> b = hyrax_block_sum<R>(smem, n, [&](size_t i) { return fp_mul<R>(load_fr<R>(r, i), load_fr<R>(d, i)); });
    hyrax_singleton_row<R>(row, n, eval, bl);                                              // com_eval, mod.rs:359-362
    PCGPU_BLOCK_FOR(i, w) store_fr<R>(row + 8 * w, i, load_fr<R>(d, i));                    // com_d = [d | r_d], :373-374
    hyrax_singleton_row<R>(row + 16 * w, n, b, bl + 8 * (n + 2));                           // com_b, :377-378
    PCGPU_BLOCK_FOR(i, 1) store_fr<R>(eval_out, p, eval);
  }
};

// block j, proof j: zs + j (dim + 2) = z || z_d || z_b, challenge c_j.  rows + 2 j (dim + 1 each) = [<r, z>, 0.., z_b] (the left
// side of (14), mod.rs:492) and [z | z_d] (of (13), :504); cl + j dim = c_j * l (t_prime * c as one MSM, :501-505).
template <class R>
struct HyraxCheckRowsBody {
  const uint32_t *tensor; const uint32_t *zs; const uint32_t *challenges; uint32_t *rows; uint32_t *cl; uint32_t dim;
  PCGPU_KERNEL_DEV void operator()(size_t j, uint32_t *smem) const {
    const size_t n = dim, w = n + 1;
    const uint32_t *l = tensor, *r = tensor + 8 * n, *z = zs + 8 * (n + 2) * j;
    uint32_t *row = rows + 8 * 2 * w * j;
    const Fp<R> rz = hyrax_block_sum<R>(smem, n, [&](size_t i) { return fp_mul<R>(load_fr<R>(r, i), load_fr<R>(z, i)); });
    hyrax_singleton_row<R>(row, n, rz, z + 8 * (n + 1));
    PCGPU_BLOCK_FOR(i, w) store_fr<R>(row + 8 * w, i, load_fr<R>(z, i));
    const Fp<R> c = load_fr<R>(challenges, j);
    PCGPU_BLOCK_FOR(i, n) store_fr<R>(cl + 8 * n * j, i, fp_mul<R>(c, load_fr<R>(l, i)));
  }
};

}  // namespace pcgpu
