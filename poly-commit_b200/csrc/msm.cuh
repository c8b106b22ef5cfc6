// G1 multi-scalar multiplication: Pippenger bucket method, all stages on the device.
//
// Replaces <E::G1 as VariableBaseMSM>::msm_bigint (ark-ec 0.5.0, un-vendored) at the reference call
// sites kzg10/mod.rs:175-178, :199-203, :255-258, :270-273; ipa_pc/mod.rs:64; hyrax/mod.rs:92, :501,
// with F::into_bigint (kzg10/mod.rs:463-470) fused into the digit pass when scalars arrive in
// Montgomery form.
//
// Pipeline (one stream, no host round trip until the S*c bit-plane sums):
//   1 count      thread/scalar : signed-digit recoding, histogram of (bucket set, |digit|)   [atomics]
//   2 scan       exclusive prefix sum of the histogram -> bucket offsets
//   3 scatter    thread/scalar : recompute digits, place (table group, base index, sign) by bucket
//   4 pair rounds (msm_affine.cuh) R times: halve every bucket with batched-affine additions  (DOMINANT at large n)
//   5 tasks      split what is left of every bucket into tasks of <= L points (bounds the longest serial
//                chain whatever the scalar distribution), scan, fill task -> bucket map
//   6 accumulate persistent kernel, dynamic task queue: XYZZ mixed additions
//   7 reduce     bucket sums, bit-plane sums T_j = sum of buckets whose weight has bit j set, pairwise tree
//   8 tail       (host, host_ec.hpp) sum_j 2^j T_j, Horner over the bucket sets, conversion to affine
//
// Window <-> table layout: window w = g*S + s uses table group g (bases pre-multiplied by
// 2^(c*S*g) at SRS registration) and bucket set s.  S = W, G = 1 is the plain method on raw bases;
// S = 1, G = W removes every doubling from the tail.
#pragma once
#include "ec.cuh"
#include "rt.cuh"

namespace pcgpu {

struct alignas(16) u32x4 { uint32_t x, y, z, w; };

struct MsmGeom {
  uint32_t n;            // pairs
  uint32_t c;            // window bits
  uint32_t W;            // windows
  uint32_t S;            // bucket sets
  uint32_t G;            // table groups (W <= S*G)
  uint32_t NB;           // buckets per set = 2^(c-1)
  uint32_t TB;           // S * NB
  uint32_t L;            // max entries per accumulate task
  uint32_t seg_len;      // buckets per reduce segment
  uint32_t nseg;         // segments per set
  uint32_t scalar_bits;  // scalars must be < 2^scalar_bits
  uint32_t scalars_mont; // 1: scalars are Montgomery Fr (convert in the digit pass)
  uint64_t table_stride; // points per table group
  uint64_t base_off;     // first base used inside each group
  uint32_t affine_rounds; // batched-affine pairwise rounds before the XYZZ task kernel
  uint32_t h_split;       // 0: one-level bit-plane reduction; else bucket index = hi * 2^h_split + lo and the weighted sum is
                          // 2^h * sum_hi hi * R_hi + sum_lo (lo+1) * C_lo over row sums R and column sums C (large c)
  uint32_t pt_words;      // table record stride in 32-bit words (2N raw; 32 for 128-byte aligned BLS12-381 records)
  uint32_t y_words;       // offset of y inside a record, in words (N raw; 16 in the aligned BLS12-381 layout)
  uint32_t pair_tdiv;     // the pair-round kernel runs with 1 / pair_tdiv of a full wave of threads (see msm_run)
};

enum : uint32_t { ENTRY_SIGN = 0x80000000u, ENTRY_GROUP_SHIFT = 26, ENTRY_IDX_MASK = (1u << 26) - 1 };

// ---------------------------------------------------------------------------------------------
// scalar loading + signed-digit recoding
// ---------------------------------------------------------------------------------------------
// scalar i as a canonical integer (Montgomery input converted), no range handling: the fixed-base / comb kernels of srs.cuh
template <class C>
PCGPU_DEV void load_scalar_plain(const uint32_t *scalars, size_t i, bool mont, uint32_t *k) {
  using R = typename C::Fr;
  const u32x4 *p = reinterpret_cast<const u32x4 *>(scalars) + 2 * i;
  u32x4 lo = p[0], hi = p[1];
  Fp<R> v;
  v.l[0] = lo.x; v.l[1] = lo.y; v.l[2] = lo.z; v.l[3] = lo.w;
  v.l[4] = hi.x; v.l[5] = hi.y; v.l[6] = hi.z; v.l[7] = hi.w;
  if (mont) v = fp_from_mont<R>(v);
#pragma unroll
  for (int j = 0; j < 8; j++) k[j] = v.l[j];
}

// Loads scalar i as a canonical integer k and halves its range: a scalar above (r - 1) / 2 is replaced by r - k and the
// caller negates every digit (k P = (r - k)(-P)).  The halved range is what lets W = ceil(bits / c) windows suffice for the
// signed-digit recoding: the top window then holds at most 2^(c-1) - 1, so the final carry can never leave it.  Returns
// false for a scalar that is not a reduced field element (k >= r).
template <class C>
PCGPU_DEV bool load_scalar(const uint32_t *scalars, size_t i, bool mont, uint32_t *k, bool *flip) {
  using R = typename C::Fr;
  static_assert(R::N == 8, "256-bit scalar fields only");
  const u32x4 *p = reinterpret_cast<const u32x4 *>(scalars) + 2 * i;
  u32x4 lo = p[0], hi = p[1];
  Fp<R> v;
  v.l[0] = lo.x; v.l[1] = lo.y; v.l[2] = lo.z; v.l[3] = lo.w;
  v.l[4] = hi.x; v.l[5] = hi.y; v.l[6] = hi.z; v.l[7] = hi.w;
  if (mont) v = fp_from_mont<R>(v);
  // compare with r and with (r - 1) / 2, most significant limb first
  bool lt_r = false, gt_half = false, decided_r = false, decided_h = false;
#pragma unroll
  for (int j = 7; j >= 0; j--) {
    const uint32_t m = R::mod(j), h = (R::mod(j) >> 1) | (j + 1 < 8 ? R::mod(j + 1 < 8 ? j + 1 : 7) << 31 : 0u);   // limb j of (r - 1) / 2
    if (!decided_r && v.l[j] != m) { lt_r = v.l[j] < m; decided_r = true; }
    if (!decided_h && v.l[j] != h) { gt_half = v.l[j] > h; decided_h = true; }
  }
  *flip = gt_half;
  if (gt_half) {
    Fp<R> m;
#pragma unroll
    for (int j = 0; j < 8; j++) m.l[j] = R::mod(j);
    // r - v as plain integers (v < r here unless the scalar is out of range, which the caller rejects)
    uint32_t borrow = 0;
#pragma unroll
    for (int j = 0; j < 8; j++) {
      const uint64_t dd = (uint64_t)m.l[j] - v.l[j] - borrow;
      v.l[j] = (uint32_t)dd; borrow = (uint32_t)(dd >> 63);
    }
  }
#pragma unroll
  for (int j = 0; j < 8; j++) k[j] = v.l[j];
  return lt_r;
}

// raw c-bit field starting at bit position pos of a 256-bit little-endian integer
PCGPU_DEV uint32_t scalar_bits_at(const uint32_t *k, uint32_t pos, uint32_t c) {
  uint32_t q = pos >> 5, sh = pos & 31;
  uint64_t lo = q < 8 ? k[q] : 0u;
  uint64_t hi = q + 1 < 8 ? k[q + 1] : 0u;
  uint64_t v = (lo | (hi << 32)) >> sh;
  return (uint32_t)v & ((1u << c) - 1);
}

// Calls f(w, magnitude in 1..2^(c-1), negative) for every non-zero signed digit.
template <class Fn>
PCGPU_DEV void for_each_digit(const uint32_t *k, const MsmGeom &g, Fn f) {
  uint32_t carry = 0;
  const uint32_t half = 1u << (g.c - 1);
  for (uint32_t w = 0; w < g.W; w++) {
    uint32_t d = scalar_bits_at(k, w * g.c, g.c) + carry;
    bool neg = d > half;
    carry = neg ? 1u : 0u;
    uint32_t mag = neg ? (1u << g.c) - d : d;
    if (mag) f(w, mag, neg);
  }
}

PCGPU_DEV bool scalar_in_range(const uint32_t *k, uint32_t bits) {
  if (bits >= 256) return true;
  uint32_t q = bits >> 5, sh = bits & 31;
  uint32_t o = k[q] >> sh;
  for (uint32_t j = q + 1; j < 8; j++) o |= k[j];
  return o == 0;
}

template <class C>
struct MsmCountBody {
  const uint32_t *scalars; MsmGeom g; uint32_t *counts; uint32_t *err;
  PCGPU_KERNEL_DEV void operator()(size_t i) const {
    uint32_t k[8];
    bool flip;
    if (!load_scalar<C>(scalars, i, g.scalars_mont != 0, k, &flip)) { rt::atomic_or(err, 1u); return; }
    uint32_t *cnt = counts; const MsmGeom gg = g;
    for_each_digit(k, gg, [&](uint32_t w, uint32_t mag, bool) {
      uint32_t s = w % gg.S;
      rt::atomic_add(cnt + (size_t)s * gg.NB + (mag - 1), 1u);
    });
  }
};

template <class C>
struct MsmScatterBody {
  const uint32_t *scalars; MsmGeom g; uint32_t *cursor; uint32_t *entries;
  PCGPU_KERNEL_DEV void operator()(size_t i) const {
    uint32_t k[8];
    bool flip;
    if (!load_scalar<C>(scalars, i, g.scalars_mont != 0, k, &flip)) return;
    uint32_t *cur = cursor; uint32_t *ent = entries; const MsmGeom gg = g;
    for_each_digit(k, gg, [&](uint32_t w, uint32_t mag, bool neg) {
      uint32_t s = w % gg.S, grp = w / gg.S;
      uint32_t pos = rt::atomic_add(cur + (size_t)s * gg.NB + (mag - 1), 1u);
      ent[pos] = ((neg != flip) ? ENTRY_SIGN : 0u) | (grp << ENTRY_GROUP_SHIFT) | (uint32_t)i;
    });
  }
};

// ---------------------------------------------------------------------------------------------
// exclusive scan of uint32 (out has n+1 entries; out[n] = total).  Three tiny kernels.
// ---------------------------------------------------------------------------------------------
enum { SCAN_CHUNK = 256 };
struct ScanChunkSumBody {
  const uint32_t *in; size_t n; uint32_t *partial;
  PCGPU_KERNEL_DEV void operator()(size_t t) const {
    size_t lo = t * SCAN_CHUNK, hi = lo + SCAN_CHUNK < n ? lo + SCAN_CHUNK : n;
    uint32_t s = 0;
    for (size_t i = lo; i < hi; i++) s += in[i];
    partial[t] = s;
  }
};
struct ScanPartialsBody {
  uint32_t *partial; size_t m;
  PCGPU_KERNEL_DEV void operator()(size_t) const {
    uint32_t run = 0;
    for (size_t i = 0; i < m; i++) { uint32_t v = partial[i]; partial[i] = run; run += v; }
    partial[m] = run;
  }
};
struct ScanApplyBody {
  const uint32_t *in; size_t n; const uint32_t *partial; uint32_t *out; size_t m;
  PCGPU_KERNEL_DEV void operator()(size_t t) const {
    size_t lo = t * SCAN_CHUNK, hi = lo + SCAN_CHUNK < n ? lo + SCAN_CHUNK : n;
    uint32_t run = partial[t];
    for (size_t i = lo; i < hi; i++) { uint32_t v = in[i]; out[i] = run; run += v; }
    if (t + 1 == m) out[n] = partial[m];
  }
};

// One-launch variant for inputs up to SCAN_BLOCK_MAX elements (every histogram of a window-folded MSM): a single block walks
// the input in tiles of SCAN_BLOCK * SCAN_PER elements -- coalesced loads (thread t owns SCAN_PER consecutive elements of the
// tile), a shared-memory scan of the per-thread sums, a running carry from tile to tile.
enum { SCAN_BLOCK = 1024, SCAN_PER = 8, SCAN_BLOCK_MAX = 1 << 17 };
struct ScanBlockBody {
  const uint32_t *in; size_t n; uint32_t *out;
  PCGPU_KERNEL_DEV void operator()(size_t, uint32_t *smem) const {
    uint32_t *a = smem, *b = smem + SCAN_BLOCK, *carry = smem + 2 * SCAN_BLOCK;
    PCGPU_BLOCK_FOR(t, 1) { carry[0] = 0; }
    PCGPU_BLOCK_SYNC();
    const size_t tile = (size_t)SCAN_BLOCK * SCAN_PER;
    for (size_t base = 0; base < n; base += tile) {
      PCGPU_BLOCK_FOR(t, SCAN_BLOCK) {
        const size_t lo = base + (size_t)t * SCAN_PER;
        uint32_t sum = 0;
        for (uint32_t k = 0; k < SCAN_PER; k++) if (lo + k < n) sum += in[lo + k];
        a[t] = sum;
      }
      PCGPU_BLOCK_SYNC();
      uint32_t *x = a, *y = b;
      for (uint32_t d = 1; d < SCAN_BLOCK; d <<= 1) {      // Hillis-Steele inclusive scan of the per-thread sums
        PCGPU_BLOCK_FOR(t, SCAN_BLOCK) { y[t] = x[t] + (t >= d ? x[t - d] : 0u); }
        PCGPU_BLOCK_SYNC();
        uint32_t *tmp = x; x = y; y = tmp;
      }
      PCGPU_BLOCK_FOR(t, SCAN_BLOCK) {
        const size_t lo = base + (size_t)t * SCAN_PER;
        uint32_t run = carry[0] + (t ? x[t - 1] : 0u);
        for (uint32_t k = 0; k < SCAN_PER; k++) if (lo + k < n) { uint32_t v = in[lo + k]; out[lo + k] = run; run += v; }
      }
      PCGPU_BLOCK_SYNC();
      PCGPU_BLOCK_FOR(t, 1) { carry[0] += x[SCAN_BLOCK - 1]; }
      PCGPU_BLOCK_SYNC();
    }
    PCGPU_BLOCK_FOR(t, 1) { out[n] = carry[0]; }
  }
};

// scratch: (n/SCAN_CHUNK + 2) uint32
inline size_t scan_scratch_words(size_t n) { return (n + SCAN_CHUNK - 1) / SCAN_CHUNK + 2; }
inline int exclusive_scan_u32(const uint32_t *in, size_t n, uint32_t *out, uint32_t *scratch, rt::stream_t st) {
  size_t m = (n + SCAN_CHUNK - 1) / SCAN_CHUNK;
  if (m == 0) { return rt::dev_memset(out, 0, sizeof(uint32_t), st); }
  if (n <= SCAN_BLOCK_MAX) return rt::launch_blocks<SCAN_BLOCK>(ScanBlockBody{in, n, out}, 1, (2 * SCAN_BLOCK + 4) * sizeof(uint32_t), st);
  int rc;
  if ((rc = rt::launch<128>(ScanChunkSumBody{in, n, scratch}, m, st))) return rc;
  if ((rc = rt::launch<32>(ScanPartialsBody{scratch, m}, 1, st))) return rc;
  return rt::launch<128>(ScanApplyBody{in, n, scratch, out, m}, m, st);
}

// ---------------------------------------------------------------------------------------------
// tasks
// ---------------------------------------------------------------------------------------------
struct TaskCountBody {
  const uint32_t *offsets; uint32_t L; uint32_t *ntasks; uint32_t heavy_min; uint32_t *heavy_count; uint32_t *heavy_list;
  PCGPU_KERNEL_DEV void operator()(size_t b) const {
    uint32_t cnt = offsets[b + 1] - offsets[b];
    uint32_t nt = (cnt + L - 1) / L;
    ntasks[b] = nt;
    // buckets with many task partials (repeated scalars, a short top window) are reduced by whole blocks before the row pass
    if (nt > heavy_min) heavy_list[rt::atomic_add(heavy_count, 1u)] = (uint32_t)b;
  }
};
struct TaskFillBody {
  const uint32_t *task_off; uint32_t *task_bucket;
  PCGPU_KERNEL_DEV void operator()(size_t b) const {
    uint32_t lo = task_off[b], hi = task_off[b + 1];
    for (uint32_t t = lo; t < hi; t++) task_bucket[t] = (uint32_t)b;
  }
};

// ---------------------------------------------------------------------------------------------
// accumulate: one thread per task
// ---------------------------------------------------------------------------------------------
template <class C>
PCGPU_DEV Affine<C> load_affine(const Affine<C> *p) {
  constexpr int N = coord_words<typename C::F>();
  const u32x4 *q = reinterpret_cast<const u32x4 *>(p);
  Affine<C> a;
  uint32_t tmp[2 * N];
#pragma unroll
  for (int j = 0; j < 2 * N / 4; j++) { u32x4 v = q[j]; tmp[4 * j] = v.x; tmp[4 * j + 1] = v.y; tmp[4 * j + 2] = v.z; tmp[4 * j + 3] = v.w; }
#pragma unroll
  for (int j = 0; j < N; j++) {
    // G1 writes the limbs directly: routed through coord_word, ptxas schedules the IPA fold kernels differently
    if constexpr (C::EXT == 1) { a.x.l[j] = tmp[j]; a.y.l[j] = tmp[N + j]; }
    else { coord_word(a.x, j) = tmp[j]; coord_word(a.y, j) = tmp[N + j]; }
  }
  return a;
}

// Table records: x at word 0, y at word g.y_words, record stride g.pt_words.  The window-folded BLS12-381 tables use
// 128-byte records (x in the first 64-byte half, y in the second) so that an x-only read is ONE aligned 64-byte DRAM
// access and a full read one aligned 128-byte line; raw base arrays keep the ABI's packed x||y.
template <class C>
PCGPU_DEV const uint32_t *table_record(const uint32_t *tables, size_t idx, const MsmGeom &g) { return tables + idx * g.pt_words; }
template <class C>
PCGPU_DEV Affine<C> load_table_point(const uint32_t *tables, size_t idx, const MsmGeom &g) {
  constexpr int N = coord_words<typename C::F>();
  const uint32_t *rec = tables + idx * g.pt_words;
  const u32x4 *qx = reinterpret_cast<const u32x4 *>(rec), *qy = reinterpret_cast<const u32x4 *>(rec + g.y_words);
  Affine<C> a;
#pragma unroll
  for (int j = 0; j < N / 4; j++) {
    u32x4 v = qx[j]; coord_word(a.x, 4 * j) = v.x; coord_word(a.x, 4 * j + 1) = v.y; coord_word(a.x, 4 * j + 2) = v.z; coord_word(a.x, 4 * j + 3) = v.w;
    u32x4 w = qy[j]; coord_word(a.y, 4 * j) = w.x; coord_word(a.y, 4 * j + 1) = w.y; coord_word(a.y, 4 * j + 2) = w.z; coord_word(a.y, 4 * j + 3) = w.w;
  }
  return a;
}
template <class C>
PCGPU_DEV void store_table_point(uint32_t *tables, size_t idx, uint32_t pt_words, uint32_t y_words, const Affine<C> &a) {
  constexpr int N = coord_words<typename C::F>();
  uint32_t *rec = tables + idx * pt_words;
  u32x4 *qx = reinterpret_cast<u32x4 *>(rec), *qy = reinterpret_cast<u32x4 *>(rec + y_words);
#pragma unroll
  for (int j = 0; j < N / 4; j++) {
    u32x4 v; v.x = coord_word(a.x, 4 * j); v.y = coord_word(a.x, 4 * j + 1); v.z = coord_word(a.x, 4 * j + 2); v.w = coord_word(a.x, 4 * j + 3); qx[j] = v;
    u32x4 w; w.x = coord_word(a.y, 4 * j); w.y = coord_word(a.y, 4 * j + 1); w.z = coord_word(a.y, 4 * j + 2); w.w = coord_word(a.y, 4 * j + 3); qy[j] = w;
  }
}
template <class C> constexpr uint32_t aligned_pt_words() { return C::Fq::N == 12 ? 32u : 2u * C::Fq::N; }
template <class C> constexpr uint32_t aligned_y_words() { return C::Fq::N == 12 ? 16u : (uint32_t)C::Fq::N; }

template <class C>
PCGPU_DEV void store_xyzz(XYZZ<C> *dst, const XYZZ<C> &p) {
  constexpr int N = coord_words<typename C::F>();
  u32x4 *q = reinterpret_cast<u32x4 *>(dst);
  const uint32_t *src = reinterpret_cast<const uint32_t *>(&p);
#pragma unroll
  for (int j = 0; j < 4 * N / 4; j++) { u32x4 v; v.x = src[4 * j]; v.y = src[4 * j + 1]; v.z = src[4 * j + 2]; v.w = src[4 * j + 3]; q[j] = v; }
}

template <class C>
PCGPU_DEV XYZZ<C> load_xyzz(const XYZZ<C> *src) {
  constexpr int N = coord_words<typename C::F>();
  const u32x4 *q = reinterpret_cast<const u32x4 *>(src);
  XYZZ<C> p;
  uint32_t *dst = reinterpret_cast<uint32_t *>(&p);
#pragma unroll
  for (int j = 0; j < 4 * N / 4; j++) { u32x4 v = q[j]; dst[4 * j] = v.x; dst[4 * j + 1] = v.y; dst[4 * j + 2] = v.z; dst[4 * j + 3] = v.w; }
  return p;
}

template <class C>
struct MsmAccumulateBody {
  const uint32_t *tables; MsmGeom g;
  const uint32_t *offsets;      // TB+1 bucket offsets into entries
  const uint32_t *task_off;     // TB+1
  const uint32_t *task_bucket;  // per task
  const uint32_t *entries;
  XYZZ<C> *partial;             // per task
  uint32_t *queue;              // global task counter (zeroed before the launch)
  const Affine<C> *pts;         // non-null after batched-affine rounds: entry e IS the point pts[e]
  // Persistent: every warp keeps claiming 32 consecutive tasks until the queue is empty.  A bucket with cnt entries
  // and T = ceil(cnt / L) tasks is split EVENLY (task j covers [cnt*j/T, cnt*(j+1)/T)), so the lanes of a warp --
  // neighbouring tasks, mostly of the same bucket -- run chains of equal length.
  PCGPU_KERNEL_DEV void operator()(size_t) const {
    const uint32_t total = task_off[g.TB];
    for (;;) {
      uint32_t t = rt::next_task(queue);
      if (t - (t & 31u) >= total) break;   // the whole warp is past the end
      if (t >= total) continue;
      uint32_t b = task_bucket[t];
      uint32_t t0 = task_off[b], T = task_off[b + 1] - t0, j = t - t0;
      uint32_t base = offsets[b], cnt = offsets[b + 1] - base;
      uint32_t lo = base + (uint32_t)(((uint64_t)cnt * j) / T);
      uint32_t hi = base + (uint32_t)(((uint64_t)cnt * (j + 1)) / T);
      XYZZ<C> acc = XYZZ<C>::inf();
      if (pts) {
        for (uint32_t e = lo; e < hi; e++) { Affine<C> a = load_affine<C>(pts + e); xyzz_madd<C>(acc, a, false); }
      } else {
        for (uint32_t e = lo; e < hi; e++) {
          uint32_t v = entries[e];
          uint32_t grp = (v & ~ENTRY_SIGN) >> ENTRY_GROUP_SHIFT;
          size_t idx = (size_t)grp * g.table_stride + g.base_off + (v & ENTRY_IDX_MASK);
          Affine<C> a = load_table_point<C>(tables, idx, g);
          xyzz_madd<C>(acc, a, (v & ENTRY_SIGN) != 0);
        }
      }
      store_xyzz<C>(partial + t, acc);
    }
  }
};

// ---------------------------------------------------------------------------------------------
// bucket reduction: bucket sums, then bit-plane sums  T[s][j] = sum_{k : bit j of (k+1)} B[s][k]
// (every stage is a plain sum, so the serial depth stays at chunk + log2(chunks) additions; the
// c-term Horner combination  sum_j 2^j T[s][j]  and the final inversion run on the host, host_ec.hpp)
// ---------------------------------------------------------------------------------------------
enum { HEAVY_BUCKET_TASKS = 8, HEAVY_BLOCK = 128, HEAVY_GRID = 64, REDUCE_BLOCK = 128 };

// Out-of-line XYZZ addition for the latency-bound reduction kernels: keeps every kernel small (with the addition inlined at
// each site the BLS12-381 unit spent > 10 minutes in cicc) at no measurable cost -- these kernels wait on chains of dependent
// additions, not on issue slots.
template <class C>
#ifdef __CUDACC__
__device__ __noinline__
#else
inline
#endif
void xyzz_add_ool(XYZZ<C> &acc, const XYZZ<C> &p) { xyzz_add<C>(acc, p); }

// one thread block per heavy bucket (grid-strided over the list): strided partial sums, then a shared-memory tree
template <class C>
struct MsmHeavyBucketBody {
  const uint32_t *task_off; const XYZZ<C> *partial; XYZZ<C> *buckets; const uint32_t *heavy_count; const uint32_t *heavy_list;
  PCGPU_KERNEL_DEV void operator()(size_t blk, uint32_t *smem) const {
    XYZZ<C> *sh = reinterpret_cast<XYZZ<C> *>(smem);
    const uint32_t nheavy = *heavy_count;
    for (uint32_t hb = (uint32_t)blk; hb < nheavy; hb += HEAVY_GRID) {
      const uint32_t b = heavy_list[hb], t0 = task_off[b], t1 = task_off[b + 1];
      PCGPU_BLOCK_FOR(i, HEAVY_BLOCK) {
        XYZZ<C> acc = XYZZ<C>::inf();
#pragma unroll 1
        for (uint32_t q = t0 + i; q < t1; q += HEAVY_BLOCK) { XYZZ<C> p = load_xyzz<C>(partial + q); xyzz_add_ool<C>(acc, p); }
        sh[i] = acc;
      }
      PCGPU_BLOCK_SYNC();
#pragma unroll 1
      for (uint32_t half = HEAVY_BLOCK / 2; half >= 1; half >>= 1) {
        PCGPU_BLOCK_FOR(i, half) { XYZZ<C> x = sh[i], y = sh[i + half]; xyzz_add_ool<C>(x, y); sh[i] = x; }
        PCGPU_BLOCK_SYNC();
      }
      PCGPU_BLOCK_FOR(i, 1) { store_xyzz<C>(buckets + b, sh[0]); }
      PCGPU_BLOCK_SYNC();
    }
  }
};

// shared-memory tree over REDUCE_BLOCK per-thread values; the sum ends in sh[0]
template <class C>
PCGPU_KERNEL_DEV void block_tree_sum(XYZZ<C> *sh) {
#pragma unroll 1
  for (uint32_t half = REDUCE_BLOCK / 2; half >= 1; half >>= 1) {
    PCGPU_BLOCK_FOR(i, half) { XYZZ<C> x = sh[i], y = sh[i + half]; xyzz_add_ool<C>(x, y); sh[i] = x; }
    PCGPU_BLOCK_SYNC();
  }
}

// Bucket reduction in three block-cooperative launches.  Bucket k of a set is addressed as k = hi * cols + lo
// (cols = 2^h_split); with row sums R_hi = sum_lo B and column sums C_lo = sum_hi B the weighted sum is
//     sum_k (k + 1) B_k  =  2^h * sum_hi hi * R_hi  +  sum_lo (lo + 1) * C_lo ,
// and each of the two short weighted sums is handed to the host as bit-plane sums (plain additions only; the O(c) Horner
// combination and the inversion run in host_ec.hpp).  Serial depth: <= 8 (task partials) + 7 (row tree) | 7 | 7.
//   rows pass : one block per (set, row): bucket sums from the task partials (kept in buckets[] for the column pass), row tree
template <class C>
struct MsmRowReduceBody {
  const uint32_t *task_off; const XYZZ<C> *partial; XYZZ<C> *buckets; XYZZ<C> *Rv;
  uint32_t NB, rows, cols;
  PCGPU_KERNEL_DEV void operator()(size_t blk, uint32_t *smem) const {
    XYZZ<C> *sh = reinterpret_cast<XYZZ<C> *>(smem);
    const uint32_t s = (uint32_t)(blk / rows), hi = (uint32_t)(blk % rows);
    PCGPU_BLOCK_FOR(t, REDUCE_BLOCK) {
      XYZZ<C> acc = XYZZ<C>::inf();
#pragma unroll 1
      for (uint32_t lo = t; lo < cols; lo += REDUCE_BLOCK) {
        const size_t b = (size_t)s * NB + (size_t)hi * cols + lo;
        const uint32_t t0 = task_off[b], t1 = task_off[b + 1];
        XYZZ<C> bs;
        if (t1 - t0 > HEAVY_BUCKET_TASKS) bs = load_xyzz<C>(buckets + b);          // written by MsmHeavyBucketBody
        else {
          bs = XYZZ<C>::inf();
#pragma unroll 1
          for (uint32_t q = t0; q < t1; q++) { XYZZ<C> p = load_xyzz<C>(partial + q); xyzz_add_ool<C>(bs, p); }
          store_xyzz<C>(buckets + b, bs);
        }
        xyzz_add_ool<C>(acc, bs);
      }
      sh[t] = acc;
    }
    PCGPU_BLOCK_SYNC();
    block_tree_sum<C>(sh);
    PCGPU_BLOCK_FOR(i, 1) { store_xyzz<C>(Rv + blk, sh[0]); }
  }
};
//   columns pass : one block per (set, column)
template <class C>
struct MsmColReduceBody {
  const XYZZ<C> *buckets; XYZZ<C> *Cv;
  uint32_t NB, rows, cols;
  PCGPU_KERNEL_DEV void operator()(size_t blk, uint32_t *smem) const {
    XYZZ<C> *sh = reinterpret_cast<XYZZ<C> *>(smem);
    const uint32_t s = (uint32_t)(blk / cols), lo = (uint32_t)(blk % cols);
    PCGPU_BLOCK_FOR(t, REDUCE_BLOCK) {
      XYZZ<C> acc = XYZZ<C>::inf();
#pragma unroll 1
      for (uint32_t hi = t; hi < rows; hi += REDUCE_BLOCK) {
        XYZZ<C> p = load_xyzz<C>(buckets + (size_t)s * NB + (size_t)hi * cols + lo);
        xyzz_add_ool<C>(acc, p);
      }
      sh[t] = acc;
    }
    PCGPU_BLOCK_SYNC();
    block_tree_sum<C>(sh);
    PCGPU_BLOCK_FOR(i, 1) { store_xyzz<C>(Cv + blk, sh[0]); }
  }
};
//   planes pass : one block per (set, plane): planes 0 .. bits_c-1 are sums of the C_lo whose weight lo + 1 has that bit set,
//   planes bits_c .. are sums of the R_hi whose weight hi has bit (j - bits_c) set
template <class C>
struct MsmPlaneReduceBody {
  const XYZZ<C> *Rv, *Cv; XYZZ<C> *plane_out;
  uint32_t rows, cols, bits_c, bits_r;
  PCGPU_KERNEL_DEV void operator()(size_t blk, uint32_t *smem) const {
    XYZZ<C> *sh = reinterpret_cast<XYZZ<C> *>(smem);
    const uint32_t per = bits_c + bits_r;
    const uint32_t s = (uint32_t)(blk / per), j = (uint32_t)(blk % per);
    const bool col = j < bits_c;
    const XYZZ<C> *vals = col ? Cv + (size_t)s * cols : Rv + (size_t)s * rows;
    const uint32_t cnt = col ? cols : rows, wofs = col ? 1u : 0u, bit = col ? j : j - bits_c;
    PCGPU_BLOCK_FOR(t, REDUCE_BLOCK) {
      XYZZ<C> acc = XYZZ<C>::inf();
#pragma unroll 1
      for (uint32_t k = t; k < cnt; k += REDUCE_BLOCK)
        if (((k + wofs) >> bit) & 1) { XYZZ<C> p = load_xyzz<C>(vals + k); xyzz_add_ool<C>(acc, p); }
      sh[t] = acc;
    }
    PCGPU_BLOCK_SYNC();
    block_tree_sum<C>(sh);
    PCGPU_BLOCK_FOR(i, 1) { store_xyzz<C>(plane_out + blk, sh[0]); }
  }
};

}  // namespace pcgpu
#include "msm_affine.cuh"
namespace pcgpu {

// ---------------------------------------------------------------------------------------------
// host orchestration
// ---------------------------------------------------------------------------------------------
inline uint32_t ilog2_floor(uint64_t v) { uint32_t l = 0; while (v >>= 1) l++; return l; }

// Window size for the plain (no precomputation) method.
inline uint32_t msm_pick_c(size_t n) {
  uint32_t lg = ilog2_floor(n ? n : 1);
  int c = (int)lg - 4;
  if (c < 8) c = 8;
  if (c > 16) c = 16;
  return (uint32_t)c;
}

inline MsmGeom msm_geometry(size_t n, uint32_t c, uint32_t groups, uint32_t scalar_bits, bool mont,
                            uint64_t table_stride, uint64_t base_off) {
  MsmGeom g;
  g.n = (uint32_t)n; g.c = c;
  g.W = (scalar_bits + c - 1) / c;   // enough because load_scalar halves the scalar range (see there)
  g.G = groups < 1 ? 1 : groups;
  g.S = (g.W + g.G - 1) / g.G;
  g.NB = 1u << (c - 1);
  g.TB = g.S * g.NB;
  g.L = 32;
  if (const char *e = getenv("PCGPU_MSM_L")) { int v = atoi(e); if (v >= 4 && v <= 4096) g.L = (uint32_t)v; }  // tuning knob
  g.seg_len = 16;
  g.nseg = (g.NB + g.seg_len - 1) / g.seg_len;
  g.scalar_bits = scalar_bits; g.scalars_mont = mont ? 1 : 0;
  g.table_stride = table_stride; g.base_off = base_off;
  g.affine_rounds = 0;
  g.h_split = (c - 1) / 2;
  g.pt_words = 0; g.y_words = 0;  // set by the caller (table_layout)
  g.pair_tdiv = 1;
  return g;
}

// XYZZ scratch elements of the reduction stage: row sums and column sums of every set
inline size_t msm_plane_scratch_elems(const MsmGeom &g) {
  size_t cols = (size_t)1 << g.h_split, rows = g.NB >> g.h_split;
  return (size_t)g.S * (rows + cols);
}

// msm_run's error words: MSM_ERR_WORDS uint32 on the device, zeroed by every run
enum {
  MSM_ERR_RANGE = 0,    // non-zero: a scalar was out of range
  MSM_ERR_QUEUE = 8,    // the accumulate kernel's task counter
  MSM_ERR_HEAVY = 12,   // the number of heavy buckets
  MSM_ERR_WORDS = 16,
};

#ifndef PCGPU_PAIR_MIN_BLOCKS
#define PCGPU_PAIR_MIN_BLOCKS 4
#endif
enum { PAIR_MIN_BLOCKS = PCGPU_PAIR_MIN_BLOCKS };  // resident blocks per SM requested for the affine pair kernel

// ---- launch wrappers of the heavy kernels: separate function templates so that every one of them can be instantiated in its
// own translation unit (inst_unit.cu groups 6-9) and the BLS12-381 build does not serialise on one 9-minute ptxas run ----
template <class C>
int msm_pair_round_oneshot(bool round0, const uint32_t *tables, const MsmGeom &g, const uint32_t *entries, const Affine<C> *in,
                           uint32_t *src, const uint32_t *off_out, uint32_t T, uint32_t *prefix, const uint32_t *pow2, Affine<C> *out,
                           rt::stream_t st) {
  if (round0) return rt::launch_occ<128, PAIR_MIN_BLOCKS>(MsmAffinePairBody<C, true>{tables, g, entries, nullptr, src, off_out, T, prefix, pow2, out}, T, st);
  return rt::launch_occ<128, PAIR_MIN_BLOCKS>(MsmAffinePairBody<C, false>{tables, g, entries, in, src, off_out, T, prefix, pow2, out}, T, st);
}
template <class C> int msm_pair_oneshot_threads(size_t *out) { return rt::resident_threads_occ<128, PAIR_MIN_BLOCKS, MsmAffinePairBody<C, true>>(out); }

template <class C>
int msm_accumulate_launch(const uint32_t *tables, const MsmGeom &g, const uint32_t *offsets, const uint32_t *task_off,
                          const uint32_t *task_bucket, const uint32_t *entries, XYZZ<C> *partial, uint32_t *queue, const Affine<C> *pts,
                          rt::stream_t st) {
  return rt::launch_persistent<128>(MsmAccumulateBody<C>{tables, g, offsets, task_off, task_bucket, entries, partial, queue, pts}, st);
}

template <class C>
int msm_reduce_launch(const MsmGeom &g, const uint32_t *task_off, const XYZZ<C> *partial, XYZZ<C> *buckets, XYZZ<C> *planes,
                      XYZZ<C> *plane_out, const uint32_t *heavy_count, const uint32_t *heavy_list, rt::stream_t st) {
  const uint32_t h = g.h_split, cols = 1u << h, rows = g.NB >> h, bits_c = h + 1, bits_r = g.c - 1 - h;
  const size_t smem = REDUCE_BLOCK * sizeof(XYZZ<C>);
  XYZZ<C> *Rv = planes, *Cv = planes + (size_t)g.S * rows;
  int rc;
  if ((rc = rt::launch_blocks<HEAVY_BLOCK>(MsmHeavyBucketBody<C>{task_off, partial, buckets, heavy_count, heavy_list}, HEAVY_GRID,
                                           HEAVY_BLOCK * sizeof(XYZZ<C>), st))) return rc;
  if ((rc = rt::launch_blocks<REDUCE_BLOCK>(MsmRowReduceBody<C>{task_off, partial, buckets, Rv, g.NB, rows, cols}, (size_t)g.S * rows, smem, st))) return rc;
  if ((rc = rt::launch_blocks<REDUCE_BLOCK>(MsmColReduceBody<C>{buckets, Cv, g.NB, rows, cols}, (size_t)g.S * cols, smem, st))) return rc;
  return rt::launch_blocks<REDUCE_BLOCK>(MsmPlaneReduceBody<C>{Rv, Cv, plane_out, rows, cols, bits_c, bits_r}, (size_t)g.S * (bits_c + bits_r), smem, st);
}

// Runs the device pipeline on `st`.  d_scalars: n x 8 uint32 on the device.  On return (asynchronously)
// *d_planes points at the S*c bit-plane sums, element (s*c + j) at index (s*c + j) * plane_stride, and
// *d_err at the run's MSM_ERR_WORDS error words.  `prof` brackets stages with events.
// *pair_threads / *pair_tdiv (if given) receive the pair-round kernel's thread count and wave divisor (0 without rounds).
template <class C, class Prof>
inline int msm_run(const uint32_t *tables, const MsmGeom &g, const uint32_t *d_scalars, rt::Arena &arena,
                   const XYZZ<C> **d_planes, size_t *plane_stride, uint32_t **d_err_out, rt::stream_t st, Prof &prof,
                   const uint32_t *pow2 = nullptr, uint32_t *pair_threads = nullptr, uint32_t *pair_tdiv = nullptr) {
  using QF = Fp<typename C::Fq>;
  const size_t max_entries = (size_t)g.n * g.W, max_tasks = max_entries / g.L + g.TB + 1;
  const size_t bound0 = max_entries / 2 + g.TB + 1, bound1 = bound0 / 2 + g.TB + 1;   // pair-round output bounds
  const bool pair_rounds = C::EXT == 1 && g.affine_rounds && pow2;   // G2 (C::EXT == 2) runs with R = 0: no pair-round kernels
  uint32_t *counts, *offsets, *cursor, *ntasks, *task_off, *task_bucket, *entries, *scratch, *err;
  XYZZ<C> *partial, *buckets, *planes, *plane_out;
  uint32_t *offA = nullptr, *offB = nullptr, *cnt = nullptr, *src = nullptr;
  QF *prefix = nullptr; Affine<C> *ptsA = nullptr, *ptsB = nullptr;
  int rc = arena.carve([&](auto &&buf) {
    buf(counts, g.TB + 2); buf(offsets, g.TB + 2); buf(cursor, g.TB + 2); buf(ntasks, g.TB + 2); buf(task_off, g.TB + 2);
    buf(task_bucket, max_tasks); buf(entries, max_entries + 1); buf(scratch, scan_scratch_words(g.TB + 1)); buf(err, MSM_ERR_WORDS);
    buf(partial, max_tasks); buf(buckets, g.TB); buf(planes, msm_plane_scratch_elems(g));
    buf(plane_out, (size_t)g.S * 2 * g.c);   // compact plane sums handed to the host
    if (pair_rounds) {
      buf(offA, g.TB + 2); buf(offB, g.TB + 2); buf(cnt, g.TB + 2); buf(src, bound0);
      buf(prefix, bound0 + (1u << 20));   // prefix products: slots rounded up to whole waves of T <= 2^20 threads
      buf(ptsA, bound0); buf(ptsB, bound1);
    }
  });
  if (rc) return rc;
  *d_err_out = err; *d_planes = plane_out; *plane_stride = 1;

  prof.begin(0, st);
  if ((rc = rt::dev_memset(counts, 0, (g.TB + 2) * sizeof(uint32_t), st))) return rc;
  if ((rc = rt::dev_memset(err, 0, MSM_ERR_WORDS * sizeof(uint32_t), st))) return rc;
  if ((rc = rt::launch<256>(MsmCountBody<C>{d_scalars, g, counts, err + MSM_ERR_RANGE}, g.n, st))) return rc;
  prof.end(0, st);

  prof.begin(1, st);
  if ((rc = exclusive_scan_u32(counts, g.TB, offsets, scratch, st))) return rc;
  if ((rc = rt::copy_d2d(cursor, offsets, (g.TB + 1) * sizeof(uint32_t), st))) return rc;
  prof.end(1, st);

  prof.begin(2, st);
  if ((rc = rt::launch<256>(MsmScatterBody<C>{d_scalars, g, cursor, entries}, g.n, st))) return rc;
  prof.end(2, st);

  // ---- batched-affine pairwise rounds (msm_affine.cuh): halve every bucket g.affine_rounds times ----
  const Affine<C> *pts = nullptr;
  if constexpr (C::EXT == 1) if (pair_rounds) {
    size_t Tmax = 0;
    if ((rc = msm_pair_oneshot_threads<C>(&Tmax))) return rc;
    if (Tmax > (1u << 20)) Tmax = 1u << 20;
    // Throughput mode (several MSM pipelines in flight on sibling streams): half a wave per pair kernel, so that the pair kernels
    // of TWO pipelines are co-resident on every SM -- a full wave owns the whole register file -- and the DRAM-bound pass 1 and
    // the ALU-bound inversion of one overlap the multiply-bound pass 2 of the other; every thread then covers twice the slots
    // with the same single inversion per round.
    uint32_t tdiv = g.pair_tdiv ? g.pair_tdiv : 1;
    if (const char *e = getenv("PCGPU_MSM_AFFINE_TDIV")) { int v = atoi(e); if (v >= 1 && v <= 16) tdiv = (uint32_t)v; }  // tuning knob
    if (tdiv > 1) Tmax = (Tmax / tdiv + 127) / 128 * 128;
    if (pair_threads) *pair_threads = (uint32_t)Tmax;
    if (pair_tdiv) *pair_tdiv = tdiv;
    prof.begin(11, st);
    const uint32_t *off_in = offsets;
    size_t bound = max_entries;
    for (uint32_t r = 0; r < g.affine_rounds; r++) {
      uint32_t *off_out = (r & 1) ? offB : offA;
      Affine<C> *out = (r & 1) ? ptsB : ptsA;
      const Affine<C> *in = (r & 1) ? ptsA : ptsB;
      bound = bound / 2 + g.TB + 1;
      if ((rc = rt::launch<256>(PairCountBody{off_in, cnt}, g.TB, st))) return rc;
      if ((rc = exclusive_scan_u32(cnt, g.TB, off_out, scratch, st))) return rc;
      if ((rc = rt::launch<256>(PairPlanBody{off_in, off_out, g.TB, src}, bound, st))) return rc;
      uint32_t T = (uint32_t)Tmax;
      if (r == 0) prof.begin(12, st);
      rc = msm_pair_round_oneshot<C>(r == 0, tables, g, entries, in, src, off_out, T, (uint32_t *)prefix, pow2, out, st);
      if (rc) return rc;
      if (r == 0) prof.end(12, st);
      off_in = off_out;
      pts = out;
    }
    prof.end(11, st);
    offsets = const_cast<uint32_t *>(off_in);
  }

  prof.begin(3, st);
  if ((rc = rt::dev_memset(err + MSM_ERR_HEAVY, 0, 4, st))) return rc;   // cursor[] is free again: heavy list
  if ((rc = rt::launch<256>(TaskCountBody{offsets, g.L, ntasks, HEAVY_BUCKET_TASKS, err + MSM_ERR_HEAVY, cursor}, g.TB, st))) return rc;
  if ((rc = exclusive_scan_u32(ntasks, g.TB, task_off, scratch, st))) return rc;
  if ((rc = rt::launch<256>(TaskFillBody{task_off, task_bucket}, g.TB, st))) return rc;
  prof.end(3, st);

  prof.begin(4, st);
  if ((rc = msm_accumulate_launch<C>(tables, g, offsets, task_off, task_bucket, entries, partial, err + MSM_ERR_QUEUE, pts, st))) return rc;
  prof.end(4, st);

  prof.begin(5, st);
  if ((rc = msm_reduce_launch<C>(g, task_off, partial, buckets, planes, plane_out, err + MSM_ERR_HEAVY, cursor, st))) return rc;
  prof.end(5, st);
  return rt::OK;
}

}  // namespace pcgpu
