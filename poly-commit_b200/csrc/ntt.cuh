// Radix-2 number-theoretic transform over Fr, four-step decomposition.
//
// Replaces Radix2EvaluationDomain::{fft, ifft} (ark-poly 0.5.0, un-vendored) at its only call site in the
// reference, linear_codes/utils.rs:112-127 (reed_solomon): the n_in input coefficients are zero-padded to
// N = 2^logn and out[j] = p(w^j) in natural order, w = root_of_unity^(2^(TWO_ADICITY - logn))
// (test_reed_solomon, linear_codes/utils.rs:303-331, pins exactly this).  ifft is the inverse map.
//
// N = N1 * N2.  Pass 1: N2 column transforms of length N1 (stride N2) with the step-2 twiddle
// w_N^(k1 n2) fused into the store; pass 2: N1 row transforms of length N2 writing X[k1 + N1 k2].
// Each length-M transform is one thread block: bit-reversed load into shared memory (limb-major so
// unit-stride butterflies are bank-conflict free), log2(M) butterfly stages with __syncthreads, store.
// Compute: (N/2) log2(N) + 2N Montgomery products; traffic: 2 reads + 2 writes of the vector
// (algorithmic: 1 read + 1 write = 64 B/element, SURVEY.md section 8d).
#pragma once
#include "frops.cuh"
#include "rt.cuh"

namespace pcgpu {

#ifndef PCGPU_NTT_MIN_BLOCKS
#define PCGPU_NTT_MIN_BLOCKS 4
#endif
#ifndef PCGPU_NTT_FULL_TABLE_MAX_LOG
#define PCGPU_NTT_FULL_TABLE_MAX_LOG 20
#endif
enum { NTT_MAX_LOG_BLOCK = 11, NTT_LO_BITS = 10, NTT_BLOCK = 128, NTT_MIN_BLOCKS = PCGPU_NTT_MIN_BLOCKS,
       NTT_FULL_TABLE_MAX_LOG = PCGPU_NTT_FULL_TABLE_MAX_LOG };

template <class R>
PCGPU_DEV Fp<R> fp_pow_u64(Fp<R> base, uint64_t e) {
  Fp<R> acc = Fp<R>::one();
  while (e) { if (e & 1) acc = fp_mul<R>(acc, base); base = fp_sqr<R>(base); e >>= 1; }
  return acc;
}

struct NttPlan {
  int curve; uint32_t logn; int inverse;
  uint32_t m1, m2;          // N1 = 2^m1 (pass 1 length), N2 = 2^m2
  uint32_t *tw1, *tw2;      // w_{N1}^j (j < N1/2), w_{N2}^j (j < N2/2)
  uint32_t *lo, *hi;        // w_N^e = hi[e >> 10] * lo[e & 1023]
  uint32_t *scale;          // N^-1 (inverse) else null
  uint32_t *base;           // allocation
};

// roots[0] = w_N (or its inverse), roots[1] = 2^-logn
template <class R>
struct NttRootsBody {
  uint32_t logn; int inverse; uint32_t *roots;
  PCGPU_KERNEL_DEV void operator()(size_t) const {
    Fp<R> w;
#pragma unroll
    for (int i = 0; i < R::N; i++) w.l[i] = R::root_of_unity(i);
    for (uint32_t i = logn; i < (uint32_t)R::TWO_ADICITY; i++) w = fp_sqr<R>(w);
    if (inverse) w = fp_inv<R>(w);
    store_fr<R>(roots, 0, w);
    Fp<R> two = fp_dbl<R>(Fp<R>::one());
    Fp<R> half = fp_inv<R>(two), s = Fp<R>::one();
    for (uint32_t i = 0; i < logn; i++) s = fp_mul<R>(s, half);
    store_fr<R>(roots, 1, s);
  }
};

// table[k] = (w^mult)^k for k < count
template <class R>
struct NttTableBody {
  const uint32_t *roots; uint64_t mult; uint32_t *table;
  PCGPU_KERNEL_DEV void operator()(size_t k) const {
    Fp<R> w = load_fr<R>(roots, 0);
    store_fr<R>(table, k, fp_pow_u64<R>(w, mult * (uint64_t)k));
  }
};

PCGPU_DEV uint32_t bitrev32(uint32_t v, uint32_t bits) {
  uint32_t r = 0;
  for (uint32_t i = 0; i < bits; i++) { r = (r << 1) | (v & 1); v >>= 1; }
  return r;
}

// ---- the butterfly stages of one length-M transform held in shared memory -----------------------------------------------
// Layout: limb-major planes of NTT_PLANE(M) words, element i at word NTT_POS(i) = i + i/8 of every plane (the padding keeps
// the register rounds below bank-conflict free: a thread's 8 elements are 2^s0 apart, consecutive threads 1 or 8 * 2^s0 apart).
// The log2(M) radix-2 stages run in ROUNDS of K <= 3 stages: a thread pulls 2^K elements into registers, runs the K stages
// on them (12 butterflies for K = 3) and writes them back -- one shared-memory round trip and one barrier per round instead of
// per stage.  In the first round the twiddles w^0 (7 of the 12) are skipped at compile time.
PCGPU_DEV uint32_t ntt_pos(uint32_t i) { return i + (i >> 3); }
PCGPU_DEV uint32_t ntt_plane(uint32_t M) { return M + (M >> 3) + 1; }
inline size_t ntt_smem_bytes(uint64_t M) { return (size_t)(M + (M >> 3) + 1) * 32; }

template <class R, int K, bool FIRST>
PCGPU_DEV void ntt_round(uint32_t *smem, uint32_t m, uint32_t s0, const uint32_t *tw, uint32_t item) {
  constexpr int E = 1 << K;
  const uint32_t P = ntt_plane(1u << m);
  const uint32_t low = FIRST ? 0u : (item & ((1u << s0) - 1u)), high = FIRST ? item : (item >> s0);
  const uint32_t base = (high << (s0 + K)) | low;
  Fp<R> v[E];
#pragma unroll
  for (int j = 0; j < E; j++) {
    const uint32_t q = ntt_pos(base + ((uint32_t)j << s0));
#pragma unroll
    for (int l = 0; l < 8; l++) v[j].l[l] = smem[l * P + q];
  }
#pragma unroll
  for (int q = 0; q < K; q++) {                       // stage s0 + q: partners differ in bit q of j
    const uint32_t s = s0 + q;
#pragma unroll
    for (int j = 0; j < E; j++) {
      if (j & (1 << q)) continue;
      const int j1 = j | (1 << q);
      const uint32_t jl = (uint32_t)(j & ((1 << q) - 1));                 // index of the pair inside its 2^s block = low + jl * 2^s0
      Fp<R> t = v[j1];
      if (!(FIRST && jl == 0)) t = fp_mul<R>(t, load_fr<R>(tw, (size_t)(low + (jl << s0)) << (m - 1 - s)));
      v[j1] = fp_sub<R>(v[j], t);
      v[j] = fp_add<R>(v[j], t);
    }
  }
#pragma unroll
  for (int j = 0; j < E; j++) {
    const uint32_t q = ntt_pos(base + ((uint32_t)j << s0));
#pragma unroll
    for (int l = 0; l < 8; l++) smem[l * P + q] = v[j].l[l];
  }
}

template <class R>
PCGPU_DEV void ntt_block_stages(uint32_t *smem, uint32_t m, const uint32_t *tw) {
  const uint32_t M = 1u << m;
  for (uint32_t s = 0; s < m;) {
    const uint32_t left = m - s;
    const uint32_t K = (left >= 5 || left == 3) ? 3u : (left == 4 ? 2u : left);   // 10 = 3+3+2+2, 11 = 3+3+3+2
    if (s == 0) {
      if (K == 3) { PCGPU_BLOCK_FOR(it, M >> 3) ntt_round<R, 3, true>(smem, m, 0, tw, it); }
      else if (K == 2) { PCGPU_BLOCK_FOR(it, M >> 2) ntt_round<R, 2, true>(smem, m, 0, tw, it); }
      else { PCGPU_BLOCK_FOR(it, M >> 1) ntt_round<R, 1, true>(smem, m, 0, tw, it); }
    } else {
      if (K == 3) { PCGPU_BLOCK_FOR(it, M >> 3) ntt_round<R, 3, false>(smem, m, s, tw, it); }
      else if (K == 2) { PCGPU_BLOCK_FOR(it, M >> 2) ntt_round<R, 2, false>(smem, m, s, tw, it); }
      else { PCGPU_BLOCK_FOR(it, M >> 1) ntt_round<R, 1, false>(smem, m, s, tw, it); }
    }
    PCGPU_BLOCK_SYNC();
    s += K;
  }
}

// launch of a block transform of length M: a register round keeps M / 8 threads busy, so the block is M / 8 threads wide
// (32 .. 128) and the resident blocks per SM are raised to match (128 registers per thread throughout) -- the short
// transforms of the Ligero row encoding (2^15 = 256 x 128) would otherwise leave three warps of four idle
template <class Body>
inline int ntt_launch(const Body &b, size_t nblocks, size_t smem_bytes, rt::stream_t st) {
  const uint32_t M = 1u << b.m;
  // (only when the grid is large enough to fill the device with narrow blocks; a small grid is latency-bound and wants the
  // wide block's parallel loads and stores)
  if (nblocks < 4096) return rt::launch_blocks_occ<NTT_BLOCK, NTT_MIN_BLOCKS>(b, nblocks, smem_bytes, st);
  if (M <= 256) return rt::launch_blocks_occ<32, 16>(b, nblocks, smem_bytes, st);
  if (M <= 512) return rt::launch_blocks_occ<64, 8>(b, nblocks, smem_bytes, st);
  return rt::launch_blocks_occ<NTT_BLOCK, NTT_MIN_BLOCKS>(b, nblocks, smem_bytes, st);
}

template <class R>
struct NttBlockBody {
  const uint32_t *in; uint32_t *out;
  uint32_t m;                               // transform length M = 2^m
  uint64_t in_stride, in_batch_stride, out_stride, out_batch_stride;
  uint64_t n_valid;                         // input elements with linear index >= n_valid read as zero
  const uint32_t *tw;                       // w_M^j, j < M/2
  const uint32_t *lo, *hi; int step2;       // step-2 twiddle w_N^(i * batch)
  const uint32_t *scale;                    // optional final factor
  uint64_t batch_off;                       // global index of local batch 0 (sharded passes); enters the step-2 twiddle only
  uint32_t i_valid;                         // elements i >= i_valid of every batch read as zero (row-batched transforms)
  // several independent transforms ("rows") in one launch: block = row * batches_per_row + batch; 0 = a single transform
  uint64_t batches_per_row = 0, in_row_stride = 0, out_row_stride = 0;
  PCGPU_KERNEL_DEV void operator()(size_t blk, uint32_t *smem) const {
    const uint32_t M = 1u << m, P = ntt_plane(M);
    const uint64_t row = batches_per_row ? blk / batches_per_row : 0, batch = batches_per_row ? blk % batches_per_row : blk;
    const uint32_t *in = this->in + 8 * row * in_row_stride;
    uint32_t *out = this->out + 8 * row * out_row_stride;
    PCGPU_BLOCK_FOR(i, M) {
      uint64_t idx = batch * in_batch_stride + (uint64_t)i * in_stride;
      Fp<R> v = (idx < n_valid && (uint32_t)i < i_valid) ? load_fr<R>(in, idx) : Fp<R>::zero();
      uint32_t r = ntt_pos(bitrev32(i, m));
#pragma unroll
      for (int l = 0; l < 8; l++) smem[l * P + r] = v.l[l];
    }
    PCGPU_BLOCK_SYNC();
    ntt_block_stages<R>(smem, m, tw);
    PCGPU_BLOCK_FOR(i, M) {
      Fp<R> v;
#pragma unroll
      for (int l = 0; l < 8; l++) v.l[l] = smem[l * P + ntt_pos(i)];
      if (step2) {
        uint64_t e = (uint64_t)i * (batch + batch_off);
        if (e) v = fp_mul<R>(v, lo ? fp_mul<R>(load_fr<R>(hi, e >> NTT_LO_BITS), load_fr<R>(lo, e & ((1u << NTT_LO_BITS) - 1))) : load_fr<R>(hi, e));
      }
      if (scale) v = fp_mul<R>(v, load_fr<R>(scale, 0));
      store_fr<R>(out, batch * out_batch_stride + (uint64_t)i * out_stride, v);
    }
  }
};

// Pass 1 of the sharded four-step transform with the all-to-all FUSED into its stores (SURVEY.md 8e): the block that
// transforms column n2 writes element k1 straight into the row buffer of the rank that owns row k1,
//   dst[k1 / rows][(k1 % rows) * N2 + n2],   rows = N1 / world,
// where dst[] are peer-mapped device pointers (NVLink P2P stores; plain pointers of one process under host emulation).
// The exchange then overlaps the butterflies column by column and pass 2 starts after one barrier -- no staging buffer, no
// separate collective.  Same arithmetic as NttBlockBody with step2 = 1 (kept separate so the validated kernel is untouched).
enum { NTT_MAX_PEERS = 16 };
template <class R>
struct NttBlockPeerBody {
  const uint32_t *in; uint32_t *dst[NTT_MAX_PEERS];
  uint32_t m;                                // N1 = 2^m
  uint64_t N2, n_valid, col_lo;              // this launch handles columns n2 = col_lo + batch
  uint32_t rows;                             // N1 / world
  const uint32_t *tw, *lo, *hi;
  PCGPU_KERNEL_DEV void operator()(size_t batch, uint32_t *smem) const {
    const uint32_t M = 1u << m, P = ntt_plane(M);
    const uint64_t n2 = col_lo + batch;
    PCGPU_BLOCK_FOR(i, M) {
      uint64_t idx = n2 + (uint64_t)i * N2;
      Fp<R> v = idx < n_valid ? load_fr<R>(in, idx) : Fp<R>::zero();
      uint32_t r = ntt_pos(bitrev32(i, m));
#pragma unroll
      for (int l = 0; l < 8; l++) smem[l * P + r] = v.l[l];
    }
    PCGPU_BLOCK_SYNC();
    ntt_block_stages<R>(smem, m, tw);
    PCGPU_BLOCK_FOR(i, M) {
      Fp<R> v;
#pragma unroll
      for (int l = 0; l < 8; l++) v.l[l] = smem[l * P + ntt_pos(i)];
      uint64_t e = (uint64_t)i * n2;
      if (e) v = fp_mul<R>(v, lo ? fp_mul<R>(load_fr<R>(hi, e >> NTT_LO_BITS), load_fr<R>(lo, e & ((1u << NTT_LO_BITS) - 1))) : load_fr<R>(hi, e));
      store_fr<R>(dst[i / rows], (uint64_t)(i % rows) * N2 + n2, v);
    }
  }
};

inline void ntt_split(uint32_t logn, uint32_t *m1, uint32_t *m2) {
  if (logn <= NTT_MAX_LOG_BLOCK) { *m1 = logn; *m2 = 0; }
  else { *m1 = (logn + 1) / 2; *m2 = logn - *m1; }
}
inline bool ntt_supported(uint32_t logn) { return logn >= 1 && logn <= 2 * NTT_MAX_LOG_BLOCK; }

template <class R>
inline int ntt_build_plan(NttPlan &p, int curve, uint32_t logn, int inverse, rt::stream_t st) {
  p.curve = curve; p.logn = logn; p.inverse = inverse;
  ntt_split(logn, &p.m1, &p.m2);
  size_t n1h = (size_t)1 << (p.m1 ? p.m1 - 1 : 0), n2h = p.m2 ? (size_t)1 << (p.m2 - 1) : 1;
  // step-2 twiddles w_N^e: up to N = 2^NTT_FULL_TABLE_MAX_LOG the whole table (32 MB at 2^20: one load and ONE product per
  // element of pass 1; with the 32 MB vector it does not fit a 50 MB L2, so the table is streamed from HBM once per pass);
  // beyond, hi[e >> 10] * lo[e & 1023] (two products, both tables cache-resident)
  const bool full = p.m2 != 0 && logn <= NTT_FULL_TABLE_MAX_LOG;
  size_t nlo = full ? 0 : (size_t)1 << NTT_LO_BITS;
  size_t nhi = full ? (size_t)1 << logn : (logn > NTT_LO_BITS ? (size_t)1 << (logn - NTT_LO_BITS) : 1);
  size_t words = 8 * (4 + n1h + n2h + nlo + nhi);
  int rc = rt::dev_malloc((void **)&p.base, words * 4);
  if (rc) return rc;
  uint32_t *roots = p.base;
  p.scale = inverse ? roots + 8 : nullptr;
  p.tw1 = roots + 32; p.tw2 = p.tw1 + 8 * n1h; p.lo = p.tw2 + 8 * n2h; p.hi = p.lo + 8 * nlo;
  if ((rc = rt::launch<32>(NttRootsBody<R>{logn, inverse, roots}, 1, st))) return rc;
  if ((rc = rt::launch<128>(NttTableBody<R>{roots, (uint64_t)1 << (logn - p.m1), p.tw1}, n1h, st))) return rc;
  if ((rc = rt::launch<128>(NttTableBody<R>{roots, (uint64_t)1 << (logn - p.m2), p.tw2}, n2h, st))) return rc;
  if (full) {
    p.lo = nullptr;                                                      // the bodies read hi[e] directly when lo is null
    return rt::launch<128>(NttTableBody<R>{roots, 1, p.hi}, nhi, st);
  }
  if ((rc = rt::launch<128>(NttTableBody<R>{roots, 1, p.lo}, nlo, st))) return rc;
  return rt::launch<128>(NttTableBody<R>{roots, (uint64_t)1 << NTT_LO_BITS, p.hi}, nhi, st);
}

// in: n_in elements (device), out: N elements (device), tmp: N elements (device; unused when m2 == 0)
template <class R>
inline int ntt_run(const NttPlan &p, const uint32_t *in, size_t n_in, uint32_t *out, uint32_t *tmp, rt::stream_t st) {
  const uint64_t N1 = (uint64_t)1 << p.m1, N2 = (uint64_t)1 << p.m2;
  if (p.m2 == 0) {
    NttBlockBody<R> b{in, out, p.m1, 1, 0, 1, 0, n_in, p.tw1, p.lo, p.hi, 0, p.scale, 0, ~0u};
    return ntt_launch(b, 1, ntt_smem_bytes(N1), st);
  }
  NttBlockBody<R> b1{in, tmp, p.m1, N2, 1, N2, 1, n_in, p.tw1, p.lo, p.hi, 1, nullptr, 0, ~0u};
  int rc = ntt_launch(b1, N2, ntt_smem_bytes(N1), st);
  if (rc) return rc;
  NttBlockBody<R> b2{tmp, out, p.m2, 1, N2, N1, 1, N1 * N2, p.tw2, p.lo, p.hi, 0, p.scale, 0, ~0u};
  return ntt_launch(b2, N1, ntt_smem_bytes(N2), st);
}

// One pass of the four-step transform on a slice of its batches -- the building block of the multi-GPU NTT (SURVEY.md 8e):
//   pass 1: columns n2 in [lo, lo+count) of the full (zero-padded) input -> local matrix out[k1 * count + (n2 - lo)]
//           (N1 x count, step-2 twiddles applied);  the ranks then exchange blocks (all-to-all) so that each owns whole rows
//   pass 2: rows k1 in [lo, lo+count), given contiguously as in[(k1 - lo) * N2 + n2] -> out[k2 * count + (k1 - lo)]
//           (natural-order element k1 + N1 k2; the caller gathers and interleaves)
template <class R>
inline int ntt_run_pass(const NttPlan &p, int which, uint64_t lo, uint64_t count, const uint32_t *in, size_t n_in, uint32_t *out,
                        rt::stream_t st) {
  const uint64_t N1 = (uint64_t)1 << p.m1, N2 = (uint64_t)1 << p.m2;
  if (which == 1) {
    NttBlockBody<R> b{in + 8 * lo, out, p.m1, N2, 1, count, 1, n_in > lo ? n_in - lo : 0, p.tw1, p.lo, p.hi, 1, nullptr, lo, ~0u};
    return ntt_launch(b, count, ntt_smem_bytes(N1), st);
  }
  NttBlockBody<R> b{in, out, p.m2, 1, N2, count, 1, count * N2, p.tw2, p.lo, p.hi, 0, p.scale, 0, ~0u};
  return ntt_launch(b, count, ntt_smem_bytes(N2), st);
}

template <class R>
inline int ntt_run_pass1_peer(const NttPlan &p, uint64_t lo, uint64_t count, const uint32_t *in, size_t n_in, uint32_t *const *dst,
                              uint32_t world, rt::stream_t st) {
  const uint64_t N1 = (uint64_t)1 << p.m1, N2 = (uint64_t)1 << p.m2;
  NttBlockPeerBody<R> b;
  b.in = in;
  for (uint32_t d = 0; d < NTT_MAX_PEERS; d++) b.dst[d] = d < world ? dst[d] : nullptr;
  b.m = p.m1; b.N2 = N2; b.n_valid = n_in; b.col_lo = lo; b.rows = (uint32_t)(N1 / world);
  b.tw = p.tw1; b.lo = p.lo; b.hi = p.hi;
  return ntt_launch(b, count, ntt_smem_bytes(N1), st);
}

// `count` independent transforms of rows laid out back to back (row r = in[r * n_in .. (r+1) * n_in), zero-padded to N) --
// the row-wise Reed-Solomon encoding of LinearEncode::compute_matrices, linear_codes/mod.rs:118-138.  Rows that fit one
// block pass go out as ONE launch of `count` blocks; longer rows run the four-step passes row by row (each pass already
// fills the device).  tmp: N elements, used only when m2 != 0.
template <class R>
inline int ntt_run_batch(const NttPlan &p, const uint32_t *in, size_t n_in, size_t count, uint32_t *out, uint32_t *tmp, rt::stream_t st,
                         uint32_t *tmp_rows = nullptr) {
  const uint64_t N = (uint64_t)1 << p.logn;
  if (p.m2 == 0) {
    NttBlockBody<R> b{in, out, p.m1, 1, n_in, 1, N, (uint64_t)count * n_in, p.tw1, p.lo, p.hi, 0, p.scale, 0, (uint32_t)n_in};
    return ntt_launch(b, count, ntt_smem_bytes(N), st);
  }
  // four-step rows: all rows' pass 1 in one launch (count * N2 column blocks), all rows' pass 2 in another, through a
  // scratch matrix of count * N elements (`tmp_rows`); without scratch the rows run one after another
  const uint64_t N1 = (uint64_t)1 << p.m1, N2 = (uint64_t)1 << p.m2;
  if (tmp_rows) {
    NttBlockBody<R> b1{in, tmp_rows, p.m1, N2, 1, N2, 1, n_in, p.tw1, p.lo, p.hi, 1, nullptr, 0, ~0u};
    b1.batches_per_row = N2; b1.in_row_stride = n_in; b1.out_row_stride = N;
    int rc = ntt_launch(b1, count * N2, ntt_smem_bytes(N1), st);
    if (rc) return rc;
    NttBlockBody<R> b2{tmp_rows, out, p.m2, 1, N2, N1, 1, N1 * N2, p.tw2, p.lo, p.hi, 0, p.scale, 0, ~0u};
    b2.batches_per_row = N1; b2.in_row_stride = N; b2.out_row_stride = N;
    return ntt_launch(b2, count * N1, ntt_smem_bytes(N2), st);
  }
  for (size_t r = 0; r < count; r++) {
    int rc = ntt_run<R>(p, in + r * n_in * 8, n_in, out + r * N * 8, tmp, st);
    if (rc) return rc;
  }
  return rt::OK;
}

}  // namespace pcgpu
