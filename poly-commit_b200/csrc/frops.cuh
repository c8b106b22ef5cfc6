// Scalar-field (Fr) vector kernels that surround the MSM on the reference's prover paths.
// All elements are Montgomery-form 8 x uint32 (32 bytes), natural order, unless stated.
//
//   fr_from_mont      F::into_bigint over a slice        kzg10/mod.rs:463-470 (convert_to_bigints)
//   fr_axpy           p += (c, q)                        marlin_pc/mod.rs:286; ipa_pc/mod.rs:691-697
//   fr_div_linear     p / (X - z), remainder p(z)        kzg10/mod.rs:222-226 (compute_witness_polynomial)
//   fr_inner_product  <a, b>                             utils.rs:150-155
//   fr_row_mul        v * M                              utils.rs:127-146 (Matrix::row_mul)
//
// These are the HBM-bound members of the path (SURVEY.md section 8d: 64 B/elem for conversion and
// division, 96 B/elem for axpy).
#pragma once
#include "ec.cuh"
#include "msm.cuh"
#include "rt.cuh"

namespace pcgpu {

template <class R>
PCGPU_DEV Fp<R> load_fr(const uint32_t *base, size_t i) {
  const u32x4 *p = reinterpret_cast<const u32x4 *>(base) + 2 * i;
  u32x4 lo = p[0], hi = p[1];
  Fp<R> v;
  v.l[0] = lo.x; v.l[1] = lo.y; v.l[2] = lo.z; v.l[3] = lo.w;
  v.l[4] = hi.x; v.l[5] = hi.y; v.l[6] = hi.z; v.l[7] = hi.w;
  return v;
}
template <class R>
PCGPU_DEV void store_fr(uint32_t *base, size_t i, const Fp<R> &v) {
  u32x4 *p = reinterpret_cast<u32x4 *>(base) + 2 * i;
  u32x4 lo, hi;
  lo.x = v.l[0]; lo.y = v.l[1]; lo.z = v.l[2]; lo.w = v.l[3];
  hi.x = v.l[4]; hi.y = v.l[5]; hi.z = v.l[6]; hi.w = v.l[7];
  p[0] = lo; p[1] = hi;
}

// a0 b0 + a1 b1: one Montgomery reduction for the two products when the modulus leaves the headroom (BN254, Pallas: 3r < 2^256;
// BLS12-381's r does not), two ordinary products otherwise
template <class R>
PCGPU_DEV Fp<R> fr_dot2(const Fp<R> &a0, const Fp<R> &b0, const Fp<R> &a1, const Fp<R> &b1) {
  if constexpr (mont_mul2_supported<R>()) return fp_mul2<R>(a0, b0, a1, b1);
  else return fp_add<R>(fp_mul<R>(a0, b0), fp_mul<R>(a1, b1));
}

template <class R>
struct FrFromMontBody {
  const uint32_t *in; uint32_t *out;
  PCGPU_KERNEL_DEV void operator()(size_t i) const { store_fr<R>(out, i, fp_from_mont<R>(load_fr<R>(in, i))); }
};
// out[i] = a[i] * b[i]
template <class R>
struct FrMulBody {
  const uint32_t *a, *b; uint32_t *out;
  PCGPU_KERNEL_DEV void operator()(size_t i) const { store_fr<R>(out, i, fp_mul<R>(load_fr<R>(a, i), load_fr<R>(b, i))); }
};
// y[i] += c * x[i]
template <class R>
struct FrAxpyBody {
  uint32_t *y; const uint32_t *c; const uint32_t *x;
  PCGPU_KERNEL_DEV void operator()(size_t i) const {
    Fp<R> cc = load_fr<R>(c, 0);
    store_fr<R>(y, i, fp_add<R>(load_fr<R>(y, i), fp_mul<R>(cc, load_fr<R>(x, i))));
  }
};

// ---------------------------------------------------------------------------------------------
// Division by (X - z) as a multi-level scan of the affine maps  t -> p_i + z * t.
//   level 0: chunks of DIV_K coefficients (thread per chunk) -> local Horner value
//   level l: nodes of DIV_F children each, folded with the factor z^(span of a child)
//   the top level (<= DIV_F nodes) is walked by one thread; carries are then pushed back down level by
//   level and every chunk replays its recurrence writing q.
// q[i-1] = p[i] + z*q[i]; carry into a chunk = q[hi-1] with q[n-1] := 0; remainder = p(z).
// ---------------------------------------------------------------------------------------------
enum { DIV_K = 32, DIV_F = 32, DIV_MAX_LEVELS = 8 };

template <class R>
struct DivPowersBody {  // zp[0] = z^DIV_K, zp[l] = zp[l-1]^DIV_F
  const uint32_t *z; uint32_t *zp; uint32_t levels;
  PCGPU_KERNEL_DEV void operator()(size_t) const {
    Fp<R> a = load_fr<R>(z, 0);
    for (int k = DIV_K; k > 1; k >>= 1) a = fp_sqr<R>(a);
    store_fr<R>(zp, 0, a);
    for (uint32_t l = 1; l < levels; l++) {
      for (int k = DIV_F; k > 1; k >>= 1) a = fp_sqr<R>(a);
      store_fr<R>(zp, l, a);
    }
  }
};

template <class R>
struct DivChunkLocalBody {
  const uint32_t *p; size_t n; const uint32_t *z; uint32_t *local;
  PCGPU_KERNEL_DEV void operator()(size_t c) const {
    size_t lo = c * DIV_K, hi = lo + DIV_K < n ? lo + DIV_K : n;
    Fp<R> zz = load_fr<R>(z, 0), acc = Fp<R>::zero();
    for (size_t i = hi; i-- > lo;) acc = fp_add<R>(fp_mul<R>(acc, zz), load_fr<R>(p, i));
    store_fr<R>(local, c, acc);
  }
};

// parent local value: fold the children's locals from the top child down (factor = z^(span of one child))
template <class R>
struct DivFoldBody {
  const uint32_t *child; size_t nchild; const uint32_t *factor; uint32_t *parent;
  PCGPU_KERNEL_DEV void operator()(size_t g) const {
    size_t lo = g * DIV_F, hi = lo + DIV_F < nchild ? lo + DIV_F : nchild;
    Fp<R> f = load_fr<R>(factor, 0), acc = Fp<R>::zero();
    for (size_t c = hi; c-- > lo;) acc = fp_add<R>(fp_mul<R>(acc, f), load_fr<R>(child, c));
    store_fr<R>(parent, g, acc);
  }
};

// carries into the children of node g (carry[c] = value entering child c from above); with parent_carry == null the
// node is the (single) root whose incoming carry is zero and whose outgoing value is the remainder
template <class R>
struct DivCarryBody {
  const uint32_t *child; size_t nchild; const uint32_t *factor; const uint32_t *parent_carry; uint32_t *carry; uint32_t *rem;
  PCGPU_KERNEL_DEV void operator()(size_t g) const {
    size_t lo = g * DIV_F, hi = lo + DIV_F < nchild ? lo + DIV_F : nchild;
    if (!parent_carry) { lo = 0; hi = nchild; }
    Fp<R> f = load_fr<R>(factor, 0), t = parent_carry ? load_fr<R>(parent_carry, g) : Fp<R>::zero();
    for (size_t c = hi; c-- > lo;) {
      store_fr<R>(carry, c, t);
      t = fp_add<R>(fp_mul<R>(t, f), load_fr<R>(child, c));
    }
    if (rem) store_fr<R>(rem, 0, t);
  }
};

template <class R>
struct DivChunkWriteBody {
  const uint32_t *p; size_t n; const uint32_t *z; const uint32_t *ccarry; uint32_t *q;
  PCGPU_KERNEL_DEV void operator()(size_t c) const {
    size_t lo = c * DIV_K, hi = lo + DIV_K < n ? lo + DIV_K : n;
    Fp<R> zz = load_fr<R>(z, 0), t = load_fr<R>(ccarry, c);
    for (size_t i = hi; i-- > lo;) {
      t = fp_add<R>(fp_mul<R>(t, zz), load_fr<R>(p, i));
      if (i > 0) store_fr<R>(q, i - 1, t);
    }
  }
};

// ---------------------------------------------------------------------------------------------
// Division by (X - z) in ONE pass over the coefficients: tiles of DIVT_TILE coefficients staged through shared memory
// (coalesced 16-byte granules in and out, padded so that a thread's private run of DIVT_L elements is bank-conflict free),
// chained from the top tile down by a decoupled look-back (every tile publishes its aggregate, then its inclusive value;
// a warp inspects 32 predecessors at a time).  t_i = p_i + z t_(i+1), t_n = 0;  q[i-1] = t_i,  remainder = t_0.
//   per element: 1 product in the local Horner walk + 1 in the fix-up  (t_i = local_i + z^(L-i) * carry_into_the_run),
//   per thread:  7 products of the block scan + 1;   traffic: 32 B read + 32 B written per coefficient.
// Tiles are handed out by an atomic ticket, highest tile first, so a tile's predecessors are always resident or finished.
// ---------------------------------------------------------------------------------------------
enum { DIVT_THREADS = 128, DIVT_L = 16, DIVT_TILE = DIVT_THREADS * DIVT_L, DIVT_WINDOW = 32,
       DIVT_POW_Z = 0,                                   // z^0 .. z^L
       DIVT_POW_W = DIVT_POW_Z + DIVT_L + 1,             // W^0 .. W^THREADS, W = z^L  (W^THREADS = z^TILE = Z)
       DIVT_POW_ZT = DIVT_POW_W + DIVT_THREADS + 1,      // Z^0 .. Z^WINDOW
       DIVT_POW_COUNT = DIVT_POW_ZT + DIVT_WINDOW + 1,
       DIVT_SPIN_LIMIT = 1 << 24 };
// shared memory: tile (TILE elements + one 16-byte pad per thread run) | scan ping | scan pong | look-back terms | misc words
inline size_t divt_smem_bytes() { return (size_t)(2 * DIVT_TILE + DIVT_THREADS) * 16 + 2 * DIVT_THREADS * 32 + DIVT_WINDOW * 32 + 32 * 4 + 64; }

template <class R>
PCGPU_DEV Fp<R> fr_pow_u32(Fp<R> base, uint32_t e) {
  Fp<R> acc = Fp<R>::one();
  while (e) { if (e & 1) acc = fp_mul<R>(acc, base); e >>= 1; if (e) base = fp_sqr<R>(base); }
  return acc;
}
template <class R>
struct DivTilePowersBody {
  const uint32_t *z; uint32_t *pw;
  PCGPU_KERNEL_DEV void operator()(size_t k) const {
    uint32_t e;
    if (k < DIVT_POW_W) e = (uint32_t)k;
    else if (k < DIVT_POW_ZT) e = (uint32_t)(k - DIVT_POW_W) * DIVT_L;
    else e = (uint32_t)(k - DIVT_POW_ZT) * DIVT_TILE;
    store_fr<R>(pw, k, fr_pow_u32<R>(load_fr<R>(z, 0), e));
  }
};

// L2-only load of an element another block published (never a stale L1 line)
template <class R>
PCGPU_DEV Fp<R> load_fr_cg(const uint32_t *base, size_t i) {
#if defined(__CUDA_ARCH__)
  const uint4 *p = reinterpret_cast<const uint4 *>(base) + 2 * i;
  uint4 lo = __ldcg(p), hi = __ldcg(p + 1);
  Fp<R> v;
  v.l[0] = lo.x; v.l[1] = lo.y; v.l[2] = lo.z; v.l[3] = lo.w; v.l[4] = hi.x; v.l[5] = hi.y; v.l[6] = hi.z; v.l[7] = hi.w;
  return v;
#else
  return load_fr<R>(base, i);
#endif
}
PCGPU_DEV uint32_t divt_flag_load(const uint32_t *p) {
#if defined(__CUDA_ARCH__)
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
#else
  return *(const volatile uint32_t *)p;
#endif
}
PCGPU_DEV void divt_flag_store(uint32_t *p, uint32_t v) {
#if defined(__CUDA_ARCH__)
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
#else
  *(volatile uint32_t *)p = v;
#endif
}

template <class R>
struct DivTileBody {
  const uint32_t *p; size_t n; const uint32_t *z; const uint32_t *pw;
  uint32_t *q; uint32_t *rem;
  uint32_t *ctl;            // [0] ticket counter, [1] error flag, [2 .. 2 + ntiles) tile status: 0 nothing, 1 aggregate, 2 inclusive
  uint32_t *agg, *inc;      // per tile
  uint32_t ntiles;
  PCGPU_DEV static uint32_t gpos(uint32_t e, uint32_t h) { return 2 * e + h + e / DIVT_L; }   // 16-byte granule of half h of element e
  PCGPU_DEV static Fp<R> lds(const u32x4 *t, uint32_t e) {
    u32x4 lo = t[gpos(e, 0)], hi = t[gpos(e, 1)];
    Fp<R> v;
    v.l[0] = lo.x; v.l[1] = lo.y; v.l[2] = lo.z; v.l[3] = lo.w; v.l[4] = hi.x; v.l[5] = hi.y; v.l[6] = hi.z; v.l[7] = hi.w;
    return v;
  }
  PCGPU_DEV static void sts(u32x4 *t, uint32_t e, const Fp<R> &v) {
    u32x4 lo, hi;
    lo.x = v.l[0]; lo.y = v.l[1]; lo.z = v.l[2]; lo.w = v.l[3]; hi.x = v.l[4]; hi.y = v.l[5]; hi.z = v.l[6]; hi.w = v.l[7];
    t[gpos(e, 0)] = lo; t[gpos(e, 1)] = hi;
  }
  PCGPU_KERNEL_DEV void operator()(size_t, uint32_t *smem) const {
    u32x4 *tile = reinterpret_cast<u32x4 *>(smem);
    uint32_t *scanA = smem + (size_t)(2 * DIVT_TILE + DIVT_THREADS) * 4, *scanB = scanA + 8 * DIVT_THREADS;
    uint32_t *terms = scanB + 8 * DIVT_THREADS;          // DIVT_WINDOW elements
    uint32_t *misc = terms + 8 * DIVT_WINDOW;            // [0] tile index, [1 .. 1 + WINDOW) status seen by the look-back lanes
    uint32_t *carry = misc + 40;                         // the value entering this tile from above (8 words)
    PCGPU_BLOCK_FOR(i, 1) { misc[0] = ntiles - 1 - rt::atomic_add(ctl, 1u); }
    PCGPU_BLOCK_SYNC();
    const uint32_t tl = misc[0];
    const size_t base = (size_t)tl * DIVT_TILE;
    const u32x4 *p16 = reinterpret_cast<const u32x4 *>(p);
    // ---- 1. tile -> shared memory (zero beyond n) ----
    // (eight independent 16-byte loads in flight per thread before the first shared-memory store: the loop is latency-bound)
    PCGPU_BLOCK_FOR(t, DIVT_THREADS) {
      for (uint32_t kb = 0; kb < 2 * DIVT_L; kb += 8) {
        u32x4 v[8];
#pragma unroll
        for (int k = 0; k < 8; k++) {
          const uint32_t g = (kb + k) * DIVT_THREADS + t, e = g >> 1;
          v[k].x = v[k].y = v[k].z = v[k].w = 0;
          if (base + e < n) v[k] = p16[2 * base + g];
        }
#pragma unroll
        for (int k = 0; k < 8; k++) {
          const uint32_t g = (kb + k) * DIVT_THREADS + t;
          tile[gpos(g >> 1, g & 1)] = v[k];
        }
      }
    }
    PCGPU_BLOCK_SYNC();
    // ---- 2. every thread: Horner walk down its run, local values in place, run aggregate to the scan buffer ----
    PCGPU_BLOCK_FOR(t, DIVT_THREADS) {
      const Fp<R> zz = load_fr<R>(pw, DIVT_POW_Z + 1);
      Fp<R> acc = Fp<R>::zero();
      for (uint32_t i = DIVT_L; i-- > 0;) {
        const uint32_t e = t * DIVT_L + i;
        acc = fp_add<R>(fp_mul<R>(acc, zz), lds(tile, e));
        sts(tile, e, acc);
      }
      store_fr<R>(scanA, t, acc);
    }
    PCGPU_BLOCK_SYNC();
    // ---- 3. reverse scan of the run aggregates: E_t = A_t + W E_(t+1)  (value leaving run t, nothing entering the tile) ----
    uint32_t *x = scanA, *y = scanB;
    for (uint32_t d = 1; d < DIVT_THREADS; d <<= 1) {
      PCGPU_BLOCK_FOR(t, DIVT_THREADS) {
        Fp<R> v = load_fr<R>(x, t);
        if (t + d < DIVT_THREADS) v = fp_add<R>(v, fp_mul<R>(load_fr<R>(pw, DIVT_POW_W + d), load_fr<R>(x, t + d)));
        store_fr<R>(y, t, v);
      }
      PCGPU_BLOCK_SYNC();
      uint32_t *tmp = x; x = y; y = tmp;
    }
    // ---- 4. publish the aggregate, look back for the value entering the tile, publish the inclusive value ----
    PCGPU_BLOCK_FOR(i, 1) {
      store_fr<R>(agg, tl, load_fr<R>(x, 0));
      store_fr<R>(carry, 0, Fp<R>::zero());
      if (tl + 1 == ntiles) { store_fr<R>(inc, tl, load_fr<R>(x, 0)); divt_flag_store(ctl + 2 + tl, 2u); }
      else divt_flag_store(ctl + 2 + tl, 1u);
    }
    PCGPU_BLOCK_SYNC();
    if (tl + 1 != ntiles) {
      // window w covers tiles tl + 1 + 32 w + j, j < 32; term_j = Z^j * (inclusive or aggregate value); the first tile that
      // shows an inclusive value ends the walk.  `done` and the running sums live in shared memory (misc / carry / terms).
      for (uint32_t w = 0;; w++) {
        PCGPU_BLOCK_FOR(j, DIVT_WINDOW) {
          const uint32_t tj = tl + 1 + w * DIVT_WINDOW + j;
          uint32_t f = 2;
          Fp<R> v = Fp<R>::zero();
          if (tj < ntiles) {
            f = divt_flag_load(ctl + 2 + tj);
            for (uint32_t spin = 0; f == 0 && spin < DIVT_SPIN_LIMIT; spin++) f = divt_flag_load(ctl + 2 + tj);
            if (f == 0) { rt::atomic_or(ctl + 1, 1u); f = 2; }            // give up rather than hang: the caller sees PCGPU_E_CUDA
            else v = fp_mul<R>(load_fr<R>(pw, DIVT_POW_ZT + j), load_fr_cg<R>(f == 2 ? inc : agg, tj));
          }
          misc[1 + j] = f;
          store_fr<R>(terms, j, v);
        }
        PCGPU_BLOCK_SYNC();
        PCGPU_BLOCK_FOR(i, 1) {
          Fp<R> sum = Fp<R>::zero();
          uint32_t done = 0;
          for (uint32_t j = 0; j < DIVT_WINDOW && !done; j++) { sum = fp_add<R>(sum, load_fr<R>(terms, j)); done = misc[1 + j] == 2; }
          // carry += (Z^32)^w * sum: the factor is kept in scanB-free space: y[0] holds (Z^32)^w (set to one at w = 0)
          Fp<R> f = w ? load_fr<R>(y, 0) : Fp<R>::one();
          store_fr<R>(carry, 0, fp_add<R>(load_fr<R>(carry, 0), w ? fp_mul<R>(f, sum) : sum));
          store_fr<R>(y, 0, fp_mul<R>(f, load_fr<R>(pw, DIVT_POW_ZT + DIVT_WINDOW)));
          misc[34] = done;
        }
        PCGPU_BLOCK_SYNC();
        if (misc[34]) break;
      }
      PCGPU_BLOCK_FOR(i, 1) {
        // inclusive value = E_0 + Z * carry
        Fp<R> v = fp_add<R>(load_fr<R>(x, 0), fp_mul<R>(load_fr<R>(pw, DIVT_POW_W + DIVT_THREADS), load_fr<R>(carry, 0)));
        store_fr<R>(inc, tl, v);
        divt_flag_store(ctl + 2 + tl, 2u);
      }
    }
    // ---- 5. fix-up: the value entering run t is E_(t+1) + W^(THREADS-1-t) * carry; t_i = local_i + z^(L-i) * that ----
    PCGPU_BLOCK_FOR(t, DIVT_THREADS) {
      Fp<R> c = fp_mul<R>(load_fr<R>(pw, DIVT_POW_W + (DIVT_THREADS - 1 - t)), load_fr<R>(carry, 0));
      if (t + 1 < DIVT_THREADS) c = fp_add<R>(c, load_fr<R>(x, t + 1));
      for (uint32_t i = 0; i < DIVT_L; i++) {
        const uint32_t e = t * DIVT_L + i;
        sts(tile, e, fp_add<R>(lds(tile, e), fp_mul<R>(load_fr<R>(pw, DIVT_POW_Z + DIVT_L - i), c)));
      }
    }
    PCGPU_BLOCK_SYNC();
    // ---- 6. shared memory -> q (shifted by one coefficient), remainder ----
    u32x4 *q16 = reinterpret_cast<u32x4 *>(q), *rem16 = reinterpret_cast<u32x4 *>(rem);
    PCGPU_BLOCK_FOR(g, 2 * DIVT_TILE) {
      const uint32_t e = g >> 1, h = g & 1;
      const size_t idx = base + e;
      if (idx >= n) continue;
      if (idx == 0) rem16[h] = tile[gpos(e, h)];
      else q16[2 * (idx - 1) + h] = tile[gpos(e, h)];
    }
  }
};

// How one division by (X - z) of n coefficients runs, decided before its first launch: the path and the layout of its scratch
// (offsets in 32-bit words from the start of the scratch).
//   tiles: powers (DIVT_POW_COUNT elements) at 0 | tile aggregates | tile inclusive values | control words (2 + ntiles)
//   tree:  level factors (DIV_MAX_LEVELS elements) at 0 | per level: the nodes' local values, then their carries
enum { DIV_PATH_NONE, DIV_PATH_TILES, DIV_PATH_TREE };
struct DivPlan {
  size_t n;
  int path;                   // DIV_PATH_NONE for n = 0 (no kernel: the remainder is zero)
  uint32_t ntiles;            // tiles
  size_t agg, inc, ctl;       // tiles
  int levels;                 // tree
  size_t cnt[DIV_MAX_LEVELS], local[DIV_MAX_LEVELS], carry[DIV_MAX_LEVELS];   // tree: nodes and offsets per level
  size_t words;               // the scratch the division needs
};

// One pass up to 2^21 coefficients; beyond that the level tree's fewer products per coefficient win.
// PCGPU_DIV_MODE = tile | tree forces one.
inline DivPlan div_plan(size_t n) {
  DivPlan d{};
  d.n = n;
  bool tiles = n <= ((size_t)1 << 21);
  if (const char *e = getenv("PCGPU_DIV_MODE")) tiles = e[0] == 't' && e[1] == 'i';
  if (n == 0) {
    d.path = DIV_PATH_NONE;
  } else if (tiles) {
    d.path = DIV_PATH_TILES;
    d.ntiles = (uint32_t)((n + DIVT_TILE - 1) / DIVT_TILE);
    d.agg = 8 * DIVT_POW_COUNT; d.inc = d.agg + 8 * (size_t)d.ntiles; d.ctl = d.inc + 8 * (size_t)d.ntiles;
    d.words = d.ctl + 2 + d.ntiles;
  } else {
    d.path = DIV_PATH_TREE;
    size_t cur = 8 * DIV_MAX_LEVELS;
    for (size_t c = (n + DIV_K - 1) / DIV_K;; c = (c + DIV_F - 1) / DIV_F) {
      d.cnt[d.levels] = c; d.local[d.levels] = cur; cur += 8 * c; d.carry[d.levels] = cur; cur += 8 * c;
      d.levels++;
      if (c <= DIV_F || d.levels == DIV_MAX_LEVELS) break;
    }
    d.words = cur;
  }
  return d;
}

// The one-pass kernel's look-back is a BOUNDED spin: a tile that never sees its predecessor publish (which would take a lost
// block, i.e. a device fault) gives up, raises ctl[1] and lets the kernel finish -- never a hang.  Callers read the word back
// here, with the plan the division ran, once the stream is idle and turn it into an error code instead of returning a wrong
// quotient.
inline int fr_div_check(const DivPlan &d, const uint32_t *scratch, rt::stream_t st) {
  if (d.path != DIV_PATH_TILES) return rt::OK;
  uint32_t h = 0;
  int rc = rt::copy_d2h(&h, scratch + d.ctl + 1, sizeof h, st);
  if (!rc) rc = rt::stream_sync(st);
  if (rc) return rc;
  return h ? rt::E_CUDA : rt::OK;
}

// p: d.n coefficients, q: d.n - 1 coefficients, rem: 1 element, z: 1 element, scratch: d.words; all device.
template <class R>
inline int fr_div_linear(const DivPlan &d, const uint32_t *p, const uint32_t *z, uint32_t *q, uint32_t *rem,
                         uint32_t *scratch, rt::stream_t st) {
  const size_t n = d.n;
  int rc;
  if (d.path == DIV_PATH_NONE) return rt::dev_memset(rem, 0, 32, st);
  if (d.path == DIV_PATH_TILES) {
    // one pass: powers (one small launch), control words cleared, tiles chained by a decoupled look-back
    uint32_t *pw = scratch, *ctl = scratch + d.ctl;
    if ((rc = rt::dev_memset(ctl, 0, (2 + (size_t)d.ntiles) * 4, st))) return rc;
    if ((rc = rt::launch<64>(DivTilePowersBody<R>{z, pw}, DIVT_POW_COUNT, st))) return rc;
    return rt::launch_blocks<DIVT_THREADS>(DivTileBody<R>{p, n, z, pw, q, rem, ctl, scratch + d.agg, scratch + d.inc, d.ntiles},
                                           d.ntiles, divt_smem_bytes(), st);
  }
  const int levels = d.levels;
  const size_t *cnt = d.cnt;
  uint32_t *zp = scratch, *local[DIV_MAX_LEVELS], *carry[DIV_MAX_LEVELS];
  for (int l = 0; l < levels; l++) { local[l] = scratch + d.local[l]; carry[l] = scratch + d.carry[l]; }
  if ((rc = rt::launch<32>(DivPowersBody<R>{z, zp, (uint32_t)levels}, 1, st))) return rc;
  if ((rc = rt::launch<128>(DivChunkLocalBody<R>{p, n, z, local[0]}, cnt[0], st))) return rc;
  for (int l = 1; l < levels; l++)
    if ((rc = rt::launch<64>(DivFoldBody<R>{local[l - 1], cnt[l - 1], zp + 8 * (l - 1), local[l]}, cnt[l], st))) return rc;
  // root: one thread walks the top level (<= DIV_F nodes unless DIV_MAX_LEVELS was hit)
  if ((rc = rt::launch<32>(DivCarryBody<R>{local[levels - 1], cnt[levels - 1], zp + 8 * (levels - 1), nullptr, carry[levels - 1], rem}, 1, st))) return rc;
  for (int l = levels - 1; l >= 1; l--)
    if ((rc = rt::launch<64>(DivCarryBody<R>{local[l - 1], cnt[l - 1], zp + 8 * (l - 1), carry[l], carry[l - 1], nullptr}, cnt[l], st))) return rc;
  return rt::launch<128>(DivChunkWriteBody<R>{p, n, z, carry[0], q}, cnt[0], st);
}

// ---------------------------------------------------------------------------------------------
// inner product: strided per-thread partial sums (coalesced), then block-level shared-memory trees
// ---------------------------------------------------------------------------------------------
enum { IP_THREADS = 262144, IP_BLOCK = 256, IP_CHUNK = 1024 };   // IP_THREADS: the most partial sums a call produces (scratch sizing)
template <class R>
struct IpPartialBody {
  const uint32_t *a; const uint32_t *b; size_t n; uint32_t *partial; uint32_t T;   // T threads, thread t owns t, t + T, t + 2T, ...
  PCGPU_KERNEL_DEV void operator()(size_t t) const {
    // two elements per iteration: four independent loads in flight and ONE Montgomery reduction for the pair
    // (fr_dot2 = a0 b0 + a1 b1 with a single reduction where 3r < 2^256: 192 instead of 256 wide multiplies per pair)
    Fp<R> acc = Fp<R>::zero();
    size_t i = t;
    for (; i + T < n; i += 2 * (size_t)T) {
      const Fp<R> a0 = load_fr<R>(a, i), b0 = load_fr<R>(b, i), a1 = load_fr<R>(a, i + T), b1 = load_fr<R>(b, i + T);
      acc = fp_add<R>(acc, fr_dot2<R>(a0, b0, a1, b1));
    }
    if (i < n) acc = fp_add<R>(acc, fp_mul<R>(load_fr<R>(a, i), load_fr<R>(b, i)));
    store_fr<R>(partial, t, acc);
  }
};
// block b sums in[b * chunk .. min(m, (b + 1) * chunk)) into out[b]: strided per-thread partial sums, then a shared-memory tree
template <class R>
struct FrBlockSumBody {
  const uint32_t *in; size_t m; uint32_t *out; uint32_t chunk;
  PCGPU_KERNEL_DEV void operator()(size_t b, uint32_t *smem) const {
    PCGPU_BLOCK_FOR(i, IP_BLOCK) {
      const size_t lo = b * (size_t)chunk, hi = lo + chunk < m ? lo + chunk : m;
      Fp<R> v = Fp<R>::zero();
      for (size_t idx = lo + i; idx < hi; idx += IP_BLOCK) v = fp_add<R>(v, load_fr<R>(in, idx));
#pragma unroll
      for (int l = 0; l < 8; l++) smem[l * IP_BLOCK + i] = v.l[l];
    }
    PCGPU_BLOCK_SYNC();
    for (uint32_t half = IP_BLOCK / 2; half >= 1; half >>= 1) {
      PCGPU_BLOCK_FOR(i, half) {
        Fp<R> x, y;
#pragma unroll
        for (int l = 0; l < 8; l++) { x.l[l] = smem[l * IP_BLOCK + i]; y.l[l] = smem[l * IP_BLOCK + i + half]; }
        x = fp_add<R>(x, y);
#pragma unroll
        for (int l = 0; l < 8; l++) smem[l * IP_BLOCK + i] = x.l[l];
      }
      PCGPU_BLOCK_SYNC();
    }
    PCGPU_BLOCK_FOR(i, 1) {
      Fp<R> v;
#pragma unroll
      for (int l = 0; l < 8; l++) v.l[l] = smem[l * IP_BLOCK];
      store_fr<R>(out, b, v);
    }
  }
};
// scratch: (IP_THREADS + IP_THREADS / IP_BLOCK) elements.  The thread count follows n (two elements per thread per iteration, at
// most IP_THREADS: 2^22 elements keep ~55 warps per SM streaming instead of 14), the partial sums are folded in one or two
// block-tree launches.
template <class R>
inline int fr_inner_product(const uint32_t *a, const uint32_t *b, size_t n, uint32_t *out, uint32_t *scratch, rt::stream_t st) {
  int rc;
  size_t T = ((n + 1) / 2 + IP_CHUNK - 1) / IP_CHUNK * IP_CHUNK;
  if (T < IP_CHUNK) T = IP_CHUNK;
  if (T > IP_THREADS) T = IP_THREADS;
  const size_t nblk = T / IP_CHUNK;
  uint32_t *lvl1 = scratch + 8 * (size_t)IP_THREADS;
  if ((rc = rt::launch<128>(IpPartialBody<R>{a, b, n, scratch, (uint32_t)T}, T, st))) return rc;
  if (nblk == 1) return rt::launch_blocks<IP_BLOCK>(FrBlockSumBody<R>{scratch, T, out, IP_CHUNK}, 1, IP_BLOCK * 32, st);
  if ((rc = rt::launch_blocks<IP_BLOCK>(FrBlockSumBody<R>{scratch, T, lvl1, IP_CHUNK}, nblk, IP_BLOCK * 32, st))) return rc;
  return rt::launch_blocks<IP_BLOCK>(FrBlockSumBody<R>{lvl1, nblk, out, (uint32_t)nblk}, 1, IP_BLOCK * 32, st);
}

// ---------------------------------------------------------------------------------------------
// row product  out_p[c] = sum_r v[r] * M_p[r*cols + c]  for `count` matrices M_p of rows x cols (Matrix::row_mul, utils.rs:127-146)
// One thread per (matrix, row span, column): coalesced across columns.  When the columns alone cannot fill the device (Hyrax's
// 2^11 x (2^11 + 1) block at cfg4 is 2049 threads) the rows are cut into `splits` spans whose partial sums a second pass adds.
// ---------------------------------------------------------------------------------------------
enum { ROWMUL_THREADS = 1 << 17, ROWMUL_MIN_SPAN = 16, ROWMUL_MAX_SPLITS = 1024 };
struct RowMulPlan {
  size_t rows, cols, count;
  uint32_t splits;   // row spans per matrix (1: one pass straight into out)
  size_t span;       // rows per span
  size_t partial;    // Fr elements of partial-sum scratch (0 when splits == 1)
};
// the fewest spans (a power of two) that give ROWMUL_THREADS threads, while every span keeps >= ROWMUL_MIN_SPAN rows
inline RowMulPlan row_mul_plan(size_t rows, size_t cols, size_t count) {
  RowMulPlan p{rows, cols, count, 1, rows, 0};
  while (p.splits < ROWMUL_MAX_SPLITS && count * cols * p.splits < (size_t)ROWMUL_THREADS && rows / (2 * (size_t)p.splits) >= ROWMUL_MIN_SPAN)
    p.splits *= 2;
  p.span = (rows + p.splits - 1) / p.splits;
  if (p.splits > 1) p.partial = count * cols * p.splits;
  return p;
}

template <class R>
struct FrRowMulBody {
  const uint32_t *v; const uint32_t *const *mats; RowMulPlan p; uint32_t *out; size_t out_stride; uint32_t *partial;
  PCGPU_KERNEL_DEV void operator()(size_t t) const {
    const size_t c = t % p.cols, s = (t / p.cols) % p.splits, q = t / (p.cols * p.splits);
    const uint32_t *m = mats[q];
    const size_t r0 = s * p.span, r1 = r0 + p.span < p.rows ? r0 + p.span : p.rows;
    Fp<R> acc = Fp<R>::zero();
    size_t r = r0;
    for (; r + 2 <= r1; r += 2)      // pairs of rows: one reduction per two products (fr_dot2)
      acc = fp_add<R>(acc, fr_dot2<R>(load_fr<R>(v, r), load_fr<R>(m, r * p.cols + c), load_fr<R>(v, r + 1), load_fr<R>(m, (r + 1) * p.cols + c)));
    if (r < r1) acc = fp_add<R>(acc, fp_mul<R>(load_fr<R>(v, r), load_fr<R>(m, r * p.cols + c)));
    if (p.splits == 1) store_fr<R>(out, q * out_stride + c, acc);
    else store_fr<R>(partial, t, acc);
  }
};
template <class R>
struct FrRowMulSumBody {
  const uint32_t *partial; RowMulPlan p; uint32_t *out; size_t out_stride;
  PCGPU_KERNEL_DEV void operator()(size_t t) const {
    const size_t c = t % p.cols, q = t / p.cols;
    Fp<R> acc = Fp<R>::zero();
    for (uint32_t s = 0; s < p.splits; s++) acc = fp_add<R>(acc, load_fr<R>(partial, (q * p.splits + s) * p.cols + c));
    store_fr<R>(out, q * out_stride + c, acc);
  }
};
// v: p.rows elements; mats: device array of p.count device pointers; out: matrix q's row product at out + q * out_stride elements;
// partial: p.partial elements of scratch
template <class R>
inline int fr_row_mul_run(const RowMulPlan &p, const uint32_t *v, const uint32_t *const *mats, uint32_t *out, size_t out_stride,
                          uint32_t *partial, rt::stream_t st) {
  int rc;
  if ((rc = rt::launch<128>(FrRowMulBody<R>{v, mats, p, out, out_stride, partial}, p.count * p.cols * p.splits, st))) return rc;
  if (p.splits == 1) return rt::OK;
  return rt::launch<128>(FrRowMulSumBody<R>{partial, p, out, out_stride}, p.count * p.cols, st);
}

// err |= 1 when an element of v (n Montgomery or canonical Fr, as stored) is not below r
template <class R>
struct FrBelowModulusBody {
  const uint32_t *v; uint32_t *err;
  PCGPU_KERNEL_DEV void operator()(size_t i) const {
    const Fp<R> s = load_fr<R>(v, i);
    bool lt_r = false, decided = false;
    for (int j = 7; j >= 0; j--) if (!decided && s.l[j] != R::mod(j)) { lt_r = s.l[j] < R::mod(j); decided = true; }
    if (!lt_r) rt::atomic_or(err, 1u);
  }
};

}  // namespace pcgpu
