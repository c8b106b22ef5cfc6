// SRS-side kernels: window-folding tables built once at registration, and fixed-base batch
// multiplication (KZG10::setup's g.batch_mul(&powers_of_beta), kzg10/mod.rs:76 -- used here to
// produce synthetic SRSs on the device for tests and benchmarks).
//
// Table group k holds 2^(c*k) * P_i (affine).  With all W groups present every Pippenger window
// shares ONE bucket set (window w of scalar i adds group-w's copy of base i), so the MSM tail needs
// no doublings and the bucket reduction shrinks from W*2^(c-1) to 2^(c-1) buckets.  Cost: W x the
// SRS footprint (1.6 GB for 2^20 BLS12-381 bases at c = 16 -- small against 80 GB of HBM3).
#pragma once
#include "ec.cuh"
#include "msm.cuh"
#include "rt.cuh"

namespace pcgpu {

enum : size_t { SRS_PRECOMPUTE_MIN_N = 1u << 12 };

inline uint32_t srs_precompute_window(size_t n) {
  if (const char *e = getenv("PCGPU_SRS_C")) { int v = atoi(e); if (v >= 8 && v <= 22) return (uint32_t)v; }   // tuning knob
  uint32_t lg = ilog2_floor(n ? n : 1);
  if (lg >= 18) return 17;   // 255 / 17 = 15 windows (load_scalar halves the scalar range, no 16th carry window): 6 % fewer
                             // additions than c = 16
  if (lg >= 15) return 14;
  return 12;
}

// rows of the base array whose ABI infinity byte is set are zeroed: (0, 0) is the device's identity encoding (ec.cuh)
struct SrsZeroIdentityBody {
  uint32_t *tables; const uint8_t *inf; uint32_t words;
  PCGPU_KERNEL_DEV void operator()(size_t i) const {
    if (inf[i]) for (uint32_t k = 0; k < words; k++) tables[i * (size_t)words + k] = 0;
  }
};

template <class C>
struct SrsGroupsBody {   // raw bases (packed x||y) -> all W groups in the aligned table layout (group 0 = the bases themselves)
  const Affine<C> *raw; uint32_t *folded; size_t n; uint32_t c; uint32_t groups; uint32_t pt_words, y_words;
  PCGPU_KERNEL_DEV void operator()(size_t i) const {
    Affine<C> a = load_affine<C>(raw + i);
    store_table_point<C>(folded, i, pt_words, y_words, a);
    for (uint32_t k = 1; k < groups; k++) {
      XYZZ<C> p = xyzz_dbl_affine<C>(a);
      for (uint32_t j = 1; j < c; j++) p = xyzz_dbl<C>(p);
      a = xyzz_to_affine<C>(p);
      store_table_point<C>(folded, (size_t)k * n + i, pt_words, y_words, a);
    }
  }
};

template <class C>
inline int srs_build_groups(const Affine<C> *raw, uint32_t *folded, size_t n, uint32_t c, uint32_t groups, rt::stream_t st) {
  return rt::launch<128>(SrsGroupsBody<C>{raw, folded, n, c, groups, aligned_pt_words<C>(), aligned_y_words<C>()}, n, st);
}

// out[i] = k_i * P for canonical scalars k_i (thread per scalar, 4-bit fixed window over a table of
// 1..15 multiples of 2^(4j) P built by the same kernel family).
template <class C>
struct FixedBaseTableBody {  // thread j builds row j: {d * 16^j * P : d = 1..15}
  Affine<C> base; Affine<C> *table;
  PCGPU_KERNEL_DEV void operator()(size_t j) const {
    XYZZ<C> w = xyzz_from_affine<C>(base);
    for (size_t k = 0; k < 4 * j; k++) w = xyzz_dbl<C>(w);
    XYZZ<C> acc = w;
    for (uint32_t d = 1; d <= 15; d++) {
      table[j * 15 + (d - 1)] = xyzz_to_affine<C>(acc);
      xyzz_add<C>(acc, w);
    }
  }
};

template <class C>
struct FixedBaseMulBody {
  const Affine<C> *table; const uint32_t *scalars; Affine<C> *out;
  PCGPU_KERNEL_DEV void operator()(size_t i) const {
    uint32_t k[8];
    load_scalar_plain<C>(scalars, i, false, k);
    XYZZ<C> acc = XYZZ<C>::inf();
    for (uint32_t j = 0; j < 64; j++) {
      uint32_t d = (k[j >> 3] >> ((j & 7) * 4)) & 15;
      if (d) { Affine<C> a = load_affine<C>(table + j * 15 + (d - 1)); xyzz_madd<C>(acc, a, false); }
    }
    out[i] = xyzz_to_affine<C>(acc);
  }
};

// ---------------------------------------------------------------------------------------------
// Batched MSM over SHARED bases (HyraxPC::commit: one Pedersen commitment per matrix row, all rows over the
// same com_key -- hyrax/mod.rs:233-242): fixed-base comb.  comb[(j*W + w)*NBk + d-1] = d * 2^(c w) * G_j for
// d in 1..2^(c-1), so a row costs n*W mixed additions and no bucket work at all.  Signed digits halve the table.
// ---------------------------------------------------------------------------------------------
struct CombGeom {
  uint32_t n_bases, c, W, NBk;  // NBk = 2^(c-1) table entries per (base, window)
  uint32_t n, count;            // row length, number of rows
  uint32_t segs, seg_len;       // each row is split into `segs` segments of `seg_len` scalars
  uint32_t scalar_bits, scalars_mont;
};

// fp_inv_gcd-based projective -> affine (the table build is setup work, but at c = 14 it is 3 * 10^8 conversions: the
// binary-GCD inverse on the otherwise idle ALU pipe instead of a 380-multiplication Fermat inverse per entry)
template <class C>
PCGPU_DEV Affine<C> comb_to_affine(const XYZZ<C> &p, const uint32_t *pow2) {
  using Q = typename C::Fq;
  if (p.is_inf()) return Affine<C>::inf();
  Fp<Q> inv = fp_inv_gcd<Q>(fp_mul<Q>(p.zz, p.zzz), pow2);
  Affine<C> a;
  a.x = fp_mul<Q>(p.x, fp_mul<Q>(inv, p.zzz));
  a.y = fp_mul<Q>(p.y, fp_mul<Q>(inv, p.zz));
  return a;
}

// thread (j, w, q) fills entries d = q * COMB_CHUNK + 1 .. of row (j, w): start point by double-and-add, then mixed additions
enum { COMB_CHUNK = 256 };
template <class C>
struct CombTableBody {
  const Affine<C> *bases; CombGeom g; Affine<C> *table; const uint32_t *pow2; uint32_t chunks;   // chunks per row
  PCGPU_KERNEL_DEV void operator()(size_t t) const {
    const uint32_t q = (uint32_t)(t % chunks);
    const size_t jw = t / chunks;
    const uint32_t j = (uint32_t)(jw / g.W), w = (uint32_t)(jw % g.W);
    XYZZ<C> p = xyzz_from_affine<C>(load_affine<C>(bases + j));
    for (uint32_t k = 0; k < w * g.c; k++) p = xyzz_dbl<C>(p);
    const Affine<C> pa = comb_to_affine<C>(p, pow2);             // 2^(c w) G_j, affine: the additions below are mixed
    const uint32_t d0 = q * COMB_CHUNK + 1, d1 = d0 + COMB_CHUNK - 1 < g.NBk ? d0 + COMB_CHUNK - 1 : g.NBk;
    XYZZ<C> acc = XYZZ<C>::inf();
    for (int b = 31; b >= 0; b--) {                              // acc = d0 * pa
      acc = xyzz_dbl<C>(acc);
      if ((d0 >> b) & 1) xyzz_madd<C>(acc, pa, false);
    }
    Affine<C> *row = table + jw * (size_t)g.NBk;
    for (uint32_t d = d0; d <= d1; d++) {
      row[d - 1] = comb_to_affine<C>(acc, pow2);
      xyzz_madd<C>(acc, pa, false);
    }
  }
};

template <class C>
struct CombAccumulateBody {
  const Affine<C> *table; const uint32_t *scalars; CombGeom g; XYZZ<C> *partial; uint32_t *err;
  PCGPU_KERNEL_DEV void operator()(size_t t) const {
    uint32_t row = (uint32_t)(t / g.segs), seg = (uint32_t)(t % g.segs);
    uint32_t lo = seg * g.seg_len, hi = lo + g.seg_len < g.n ? lo + g.seg_len : g.n;
    MsmGeom mg; mg.c = g.c; mg.W = g.W;
    XYZZ<C> acc = XYZZ<C>::inf();
    const Affine<C> *tab = table; const CombGeom gg = g;
    for (uint32_t i = lo; i < hi; i++) {
      uint32_t k[8];
      bool flip;   // load_scalar halves the scalar range, so W = ceil(bits / c) windows carry every digit
      if (!load_scalar<C>(scalars, (size_t)row * g.n + i, g.scalars_mont != 0, k, &flip)) { rt::atomic_or(err, 1u); continue; }
      for_each_digit(k, mg, [&](uint32_t w, uint32_t mag, bool neg) {
        Affine<C> a = load_affine<C>(tab + ((size_t)i * gg.W + w) * gg.NBk + (mag - 1));
        xyzz_madd<C>(acc, a, neg != flip);
      });
    }
    store_xyzz<C>(partial + t, acc);
  }
};

template <class C>
struct CombRowSumBody {
  const XYZZ<C> *partial; uint32_t segs; Affine<C> *out; const uint32_t *pow2;
  PCGPU_KERNEL_DEV void operator()(size_t row) const {
    XYZZ<C> acc = XYZZ<C>::inf();
    for (uint32_t s = 0; s < segs; s++) { XYZZ<C> p = load_xyzz<C>(partial + row * segs + s); xyzz_add<C>(acc, p); }
    out[row] = comb_to_affine<C>(acc, pow2);
  }
};

}  // namespace pcgpu
