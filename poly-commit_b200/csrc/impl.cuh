// Host-side implementation templates behind the C ABI (include/pcgpu.h).  Host logic only: argument checks that mirror the
// reference's error behaviour, staging of host buffers, stage timing, and curve dispatch.
//
// Compiled by nvcc for sm_90a into libpcgpu.so (the product).  The same file is also compiled by
// g++ with -DPCGPU_EMUL into tests/host_emul/libpcgpu_hostcheck.so, a unit-test harness that runs
// the kernel bodies serially; the package never loads that library.
#pragma once
#include <algorithm>
#include <memory>
#include <mutex>
#include <new>
#include <type_traits>
#include <vector>

#include "../../include/pcgpu.h"
#include "frops.cuh"
#include "host_ec.hpp"
#include "host_glv.hpp"
#include "ntt.cuh"
#include "ipa.cuh"
#include <chrono>
#include "msm.cuh"
#include "srs.cuh"
#include "wire.cuh"
#include "msm_small.cuh"
#include "peer.cuh"
#include "hash.cuh"
#include "sprs.cuh"
#include "field_ops.cuh"
#include "mlpc.cuh"

using namespace pcgpu;

// ---------------------------------------------------------------------------------------------
// profiling (CUDA events on the launching stream)
// ---------------------------------------------------------------------------------------------
enum { PROF_STAGES = 17 };
struct Prof {
  bool on = false;
  double ms[PROF_STAGES] = {0};
  uint64_t cnt[PROF_STAGES] = {0};
#ifndef PCGPU_EMUL
  cudaEvent_t ev[PROF_STAGES][2];
  bool created = false, pending[PROF_STAGES] = {false};
  void ensure() {
    if (created) return;
    for (int s = 0; s < PROF_STAGES; s++) { cudaEventCreate(&ev[s][0]); cudaEventCreate(&ev[s][1]); }
    created = true;
  }
  void begin(int s, rt::stream_t st) { if (on) { ensure(); collect_one(s); cudaEventRecord(ev[s][0], st); } }
  void end(int s, rt::stream_t st) { if (on) { cudaEventRecord(ev[s][1], st); pending[s] = true; } }
  void collect_one(int s) {
    if (!pending[s]) return;
    cudaEventSynchronize(ev[s][1]);
    float t = 0; cudaEventElapsedTime(&t, ev[s][0], ev[s][1]);
    ms[s] += t; cnt[s]++; pending[s] = false;
  }
  void collect() { if (on) for (int s = 0; s < PROF_STAGES; s++) collect_one(s); }
  void destroy() { if (created) for (int s = 0; s < PROF_STAGES; s++) { cudaEventDestroy(ev[s][0]); cudaEventDestroy(ev[s][1]); } created = false; }
#else
  void begin(int, rt::stream_t) {}
  void end(int, rt::stream_t) {}
  void collect() {}
  void destroy() {}
#endif
  void reset() { for (int s = 0; s < PROF_STAGES; s++) { ms[s] = 0; cnt[s] = 0; } }
};

struct pcgpu_srs {
  int curve;
  size_t n;          // bases per table group
  uint32_t c;        // window bits the groups were built for (0: raw bases only)
  uint32_t groups;   // table groups (1: raw bases)
  void *d_tables;    // the n raw bases, packed x||y
  void *d_folded;    // window-folded tables: groups * n records in the aligned layout (PCGPU_SRS_PRECOMPUTE) or null
  void *d_comb;      // fixed-base comb tables (PCGPU_SRS_COMB) or null
  uint32_t comb_c;   // comb window bits
};

enum { PCGPU_MAX_PLANES = 512 };  // S * c of any geometry msm_geometry produces (W <= 32 windows of <= 22 bits, S <= W)

// Page-locked landing zone of msm_issue's asynchronous copies: the S*c plane sums, packed, then msm_run's error words.
struct PinnedZone {
  unsigned char planes[PCGPU_MAX_PLANES * sizeof(XYZZ<Bls12381G2>)];   // sized for the largest XYZZ
  uint32_t err[MSM_ERR_WORDS];
};

// A context's own device words.
struct DeviceWords {
  XYZZ<Bls12381> peer_partial;       // msm_peer_impl: a partial finished on the host, pushed as a one-plane record (largest G1)
  uint32_t peer_timeout;             // PeerWaitBody: non-zero when a peer missed the deadline
  unsigned long long last_nonzero;   // FrLastNonzeroBody: one past the last non-zero coefficient
  uint32_t selftest_bad;             // FieldSelfTestBody: mismatch count
};

struct pcgpu_ctx {
  int device;
  rt::stream_t own_stream, stream;
  rt::Arena msm_arena, stage;
  rt::Arena ipa_arena;             // state of the (one) InnerProductArgPC::open in progress on this context; reused across opens
  bool ipa_active = false;
  uint32_t pair_tdiv = 1;          // set by the batch entry points while several pipelines are in flight (msm_run)
  DeviceWords *d_words = nullptr;
  Prof prof;
  uint32_t *d_pow2[3] = {nullptr, nullptr, nullptr};  // fp_inv_gcd tables (Fq), per curve
  std::vector<pcgpu_ctx *> siblings;  // extra contexts on the same device for pcgpu_kzg_commit_batch
  std::vector<NttPlan> ntt_plans;  // twiddle tables, cached per (curve, logn, direction)
  PinnedZone *h_pinned = nullptr;
  rt::event_t ev_upload;           // "inputs are on the device": lets a sibling context's stream start on them
  bool ev_ok = false;
  uint64_t last_geom[PCGPU_GEOM_FIELDS] = {0};   // path / geometry of the most recent MSM (pcgpu_msm_last_geometry)
  std::mutex mu;
};

#ifndef PCGPU_EMUL
#define SET_DEVICE(ctx) do { if (cudaSetDevice((ctx)->device) != cudaSuccess) return PCGPU_E_CUDA; } while (0)
#else
#define SET_DEVICE(ctx) do { } while (0)
#endif

#define DISPATCH_CURVE(curve, CALL)                 \
  switch (curve) {                                  \
    case PCGPU_BLS12_381: { using C = Bls12381; CALL; } \
    case PCGPU_BN254: { using C = Bn254; CALL; }    \
    case PCGPU_PALLAS: { using C = Pallas; CALL; }  \
    default: return PCGPU_E_BADARG;                 \
  }

// the groups an MSM key can hold: the three G1s and the two G2s (include/pcgpu.h group ids)
#define DISPATCH_GROUP(group, CALL)                          \
  switch (group) {                                           \
    case PCGPU_BLS12_381: { using C = Bls12381; CALL; }      \
    case PCGPU_BN254: { using C = Bn254; CALL; }             \
    case PCGPU_PALLAS: { using C = Pallas; CALL; }           \
    case PCGPU_BLS12_381_G2: { using C = Bls12381G2; CALL; } \
    case PCGPU_BN254_G2: { using C = Bn254G2; CALL; }        \
    default: return PCGPU_E_BADARG;                          \
  }

// the G2 group of a pairing curve id (MultilinearPC, pcgpu_diag_field_op which = 2)
#define DISPATCH_PAIRING_G2(curve, CALL)                 \
  switch (curve) {                                       \
    case PCGPU_BLS12_381: { using C = Bls12381G2; CALL; } \
    case PCGPU_BN254: { using C = Bn254G2; CALL; }        \
    default: return PCGPU_E_BADARG;                      \
  }

// The operands of one call that pass through the context's staging arena.  Each operand is declared once, by what it is:
//   in       with PCGPU_DEVICE_PTRS the caller's pointer as is, else an arena buffer filled from the host
//   host_in  always a host pointer: an arena buffer filled from it
//   out      with PCGPU_DEVICE_PTRS and a non-null destination the caller's pointer, else an arena buffer, copied back when
//            the flag is clear and the destination is non-null
//   inout    in and out over one buffer
//   scratch  an arena buffer
// upload() reserves the arena once from the declared sizes, points every operand at its buffer and queues the host-to-device
// copies; download() queues the copies back.  Copies go on the context's stream in declaration order; nothing synchronises.
// Every arena buffer is at least one 256-byte granule, so a zero-length operand still gets a valid, distinct pointer; zero-byte
// copies are skipped.
class Staging {
 public:
  Staging(pcgpu_ctx *ctx, uint32_t flags) : ctx_(ctx), dev_((flags & PCGPU_DEVICE_PTRS) != 0) {}
  template <class P> void in(P &d, const void *src, size_t bytes) { add(d, dev_, src, nullptr, bytes, TO_DEV); }
  template <class P> void host_in(P &d, const void *src, size_t bytes) { add(d, false, src, nullptr, bytes, TO_DEV); }
  template <class P> void out(P &d, void *dst, size_t bytes) { add(d, dev_ && dst, dst, dev_ ? nullptr : dst, bytes, TO_HOST); }
  template <class P> void inout(P &d, void *buf, size_t bytes) { add(d, dev_, buf, buf, bytes, TO_DEV | TO_HOST); }
  template <class P> void scratch(P &d, size_t bytes) { add(d, false, nullptr, nullptr, bytes, 0); }
  int upload();
  int download();

 private:
  enum { TO_DEV = 1, TO_HOST = 2, MAX_OPS = 8 };
  struct Op { void *slot; void (*set)(void *slot, void *p); const void *src; void *dst; size_t bytes; int copy; char *buf; };
  template <class P> void add(P &d, bool callers, const void *src, void *dst, size_t bytes, int copy) {
    if (callers) { d = static_cast<P>(const_cast<void *>(src)); return; }
    if (n_ == MAX_OPS) { overflow_ = true; return; }
    ops_[n_++] = Op{&d, [](void *slot, void *p) { *static_cast<P *>(slot) = static_cast<P>(p); }, src, dst, bytes, copy, nullptr};
  }
  pcgpu_ctx *ctx_;
  bool dev_, overflow_ = false;
  int n_ = 0;
  Op ops_[MAX_OPS];
};

inline int Staging::upload() {
  if (overflow_) return PCGPU_E_BADARG;
  int rc = ctx_->stage.carve([&](auto &&buf) { for (int i = 0; i < n_; i++) buf(ops_[i].buf, ops_[i].bytes); });
  if (rc) return rc;
  for (int i = 0; i < n_; i++) {
    const Op &o = ops_[i];
    o.set(o.slot, o.buf);
    if ((o.copy & TO_DEV) && o.bytes && (rc = rt::copy_h2d(o.buf, o.src, o.bytes, ctx_->stream))) return rc;
  }
  return PCGPU_OK;
}

inline int Staging::download() {
  int rc;
  for (int i = 0; i < n_; i++) {
    const Op &o = ops_[i];
    if ((o.copy & TO_HOST) && o.dst && o.bytes && (rc = rt::copy_d2h(o.dst, o.buf, o.bytes, ctx_->stream))) return rc;
  }
  return PCGPU_OK;
}

// ---------------------------------------------------------------------------------------------
// SRS
// ---------------------------------------------------------------------------------------------
template <class C> static int ensure_pow2(pcgpu_ctx *ctx);

// comb window bits: the widest window whose tables (n * W * 2^(c-1) points) fit the budget: PCGPU_COMB_MAX_GB if set, else
// 40 % of the device memory that is free right now, at most 72 GB (wider windows mean fewer bucket additions per commit;
// the table is built once per key)
inline uint32_t comb_window_bits(size_t n, size_t point_bytes) {
  if (const char *e = getenv("PCGPU_COMB_C")) { int v = atoi(e); if (v >= 4 && v <= 16) return (uint32_t)v; }
  double cap = 24e9;
#ifdef PCGPU_EMUL
  const double max_entries = 65536.0;          // the serial emulation builds every entry with a GCD inversion
#else
  const double max_entries = 1.2e9;            // ~2 s of table construction
  size_t free_b = 0, total_b = 0;
  if (cudaMemGetInfo(&free_b, &total_b) == cudaSuccess) { cap = 0.4 * (double)free_b; if (cap > 72e9) cap = 72e9; }
#endif
  if (const char *e = getenv("PCGPU_COMB_MAX_GB")) { double v = atof(e); if (v > 0) cap = v * 1e9; }
  uint32_t best = 4;
  for (uint32_t c = 4; c <= 16; c++) {
    double entries = (double)n * ((255 + c - 1) / c) * (double)(1u << (c - 1));
    if (entries * (double)point_bytes <= cap && entries <= max_entries) best = c;
  }
  return best;
}

template <class C>
int srs_register_impl(pcgpu_ctx *ctx, const void *bases, const uint8_t *inf, size_t n, uint32_t flags, pcgpu_srs *srs) {
  const size_t psz = sizeof(Affine<C>);
  uint32_t groups = 1, c = 0;
  if (C::EXT == 2 && (flags & (PCGPU_SRS_PRECOMPUTE | PCGPU_SRS_COMB))) return PCGPU_E_BADARG;   // G2 keys hold raw bases only
  if ((flags & PCGPU_SRS_PRECOMPUTE) && n > 0) {
    c = srs_precompute_window(n);
    groups = (C::Fr::BITS + c - 1) / c;   // one table group per window (msm_geometry's W)
  }
  int rc = rt::dev_malloc(&srs->d_tables, psz * (n ? n : 1));
  if (rc) return rc;
  if (groups > 1 && (rc = rt::dev_malloc(&srs->d_folded, (size_t)aligned_pt_words<C>() * 4 * n * groups))) return rc;
  rt::stream_t st = ctx->stream;
  if (n) {
    if (flags & PCGPU_DEVICE_PTRS) rc = rt::copy_d2d(srs->d_tables, bases, psz * n, st);
    else rc = rt::copy_h2d(srs->d_tables, bases, psz * n, st);
    if (rc) return rc;
    if (inf) {   // identity bases become the device's (0, 0) encoding -- one kernel, for host and device flag arrays alike
      const uint8_t *d_inf;
      Staging io(ctx, flags);
      io.in(d_inf, inf, n);
      if ((rc = io.upload())) return rc;
      if ((rc = rt::launch<256>(SrsZeroIdentityBody{(uint32_t *)srs->d_tables, d_inf, (uint32_t)(psz / 4)}, n, st))) return rc;
    }
    if constexpr (C::EXT == 1) {
    if (groups > 1 && (rc = srs_build_groups<C>((const Affine<C> *)srs->d_tables, (uint32_t *)srs->d_folded, n, c, groups, st))) return rc;
    if (flags & PCGPU_SRS_COMB) {
      CombGeom cg; memset(&cg, 0, sizeof cg);
      cg.n_bases = (uint32_t)n; cg.c = comb_window_bits(n, psz); cg.W = (C::Fr::BITS + cg.c - 1) / cg.c; cg.NBk = 1u << (cg.c - 1);
      if ((rc = rt::dev_malloc(&srs->d_comb, psz * n * cg.W * cg.NBk))) return rc;
      srs->comb_c = cg.c;
      if ((rc = ensure_pow2<C>(ctx))) return rc;
      const uint32_t chunks = (cg.NBk + COMB_CHUNK - 1) / COMB_CHUNK;
      if ((rc = rt::launch<64>(CombTableBody<C>{(const Affine<C> *)srs->d_tables, cg, (Affine<C> *)srs->d_comb, ctx->d_pow2[C::ID], chunks},
                               n * cg.W * chunks, st))) return rc;
    }
    }
  }
  srs->c = c; srs->groups = groups;
  return rt::stream_sync(st);
}




// ---------------------------------------------------------------------------------------------
// helpers
// ---------------------------------------------------------------------------------------------
// Small MSMs (msm_small.cuh): up to SMALL_MAX_PROB problems of <= SMALL_MAX_N terms in one launch; one point per window
// comes back and the host finishes with the doublings.  PCGPU_MSM_SMALL=0 forces the bucket pipeline (tests, A/B timing).
inline bool msm_small_enabled() {
  const char *e = getenv("PCGPU_MSM_SMALL");
  return !(e && e[0] == '0');
}
template <class C>
int msm_small_to_host(pcgpu_ctx *ctx, const MsmSmallProblem<C> *probs, uint32_t nprob, bool mont, host::HXYZZ<C> *out) {
  using R = typename C::Fr;
  constexpr uint32_t W = small_windows<R>();
  rt::stream_t st = ctx->stream;
  int rc;
  if (nprob == 0 || nprob > SMALL_MAX_PROB) return PCGPU_E_BADARG;
  uint32_t nmax = 0;
  for (uint32_t p = 0; p < nprob; p++) nmax = probs[p].n > nmax ? probs[p].n : nmax;
  // blocks per window: 1 below 512 terms, 3 up to SMALL_MAX_N, 6 beyond (the IPA's l / r commitments of 8192 terms: a block's
  // share stays at <= 1366 terms, which is what bounds its chain of dependent additions and its digit buffer)
  if (nmax > 2 * SMALL_MAX_N) return PCGPU_E_BADARG;
  const uint32_t split = nmax > SMALL_MAX_N ? 2 * SMALL_SPLIT : (nmax >= SMALL_SPLIT_MIN_N ? SMALL_SPLIT : 1);
  memset(ctx->last_geom, 0, sizeof ctx->last_geom);
  ctx->last_geom[PCGPU_GEOM_PATH] = PCGPU_MSM_PATH_SMALL; ctx->last_geom[PCGPU_GEOM_SPLIT] = split; ctx->last_geom[PCGPU_GEOM_N] = nmax;
  const size_t npts = (size_t)nprob * W * split;
  uint32_t *d_err; XYZZ<C> *d_out;
  if ((rc = ctx->msm_arena.carve([&](auto &&buf) { buf(d_err, 1); buf(d_out, npts); }))) return rc;
  if ((rc = rt::dev_memset(d_err, 0, sizeof *d_err, st))) return rc;
  MsmSmallBody<C> body;
  memset(&body, 0, sizeof body);
  for (uint32_t p = 0; p < nprob; p++) body.prob[p] = probs[p];
  body.mont = mont ? 1u : 0u; body.split = split; body.out = d_out; body.err = d_err;
  ctx->prof.begin(4, st);
  if ((rc = rt::launch_blocks<SMALL_BLOCK>(body, npts, msm_small_smem<C>(), st))) return rc;
  ctx->prof.end(4, st);
  static_assert(sizeof(host::HXYZZ<C>) == sizeof(XYZZ<C>), "host/device point layouts must agree");
  std::vector<host::HXYZZ<C>> U(npts);
  uint32_t herr = 0;
  if ((rc = rt::copy_d2h(U.data(), d_out, U.size() * sizeof(XYZZ<C>), st))) return rc;
  if ((rc = rt::copy_d2h(&herr, d_err, sizeof herr, st))) return rc;
  if ((rc = rt::stream_sync(st))) return rc;
  ctx->prof.collect();
  if (herr) return PCGPU_E_RANGE;
  auto t0 = std::chrono::steady_clock::now();
  for (size_t v = 0; v < (size_t)nprob * W && split > 1; v++) {       // fold the partial window sums of the split blocks
    host::HXYZZ<C> a = U[v * split];
    for (uint32_t q = 1; q < split; q++) a = host::padd<C>(a, U[v * split + q]);
    U[v] = a;
  }
  for (uint32_t p = 0; p < nprob; p++) out[p] = host::combine_windows<C>(U.data() + (size_t)p * W, W, SMALL_C);
  if (ctx->prof.on) {
    ctx->prof.ms[6] += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    ctx->prof.cnt[6]++;
  }
  return PCGPU_OK;
}

// Device half of one bucket-pipeline MSM (n > SMALL_MAX_N or the small path disabled): picks the geometry, runs msm_run on
// the context's stream and returns (asynchronously) the compact S*c bit-plane sums and the error words.
template <class C>
int msm_device_planes(pcgpu_ctx *ctx, const pcgpu_srs *srs, size_t base_offset, const uint32_t *d_scalars, size_t n,
                             bool mont, MsmGeom *g_out, const XYZZ<C> **d_planes, size_t *stride, uint32_t **d_err) {
  rt::stream_t st = ctx->stream;
  uint32_t c, groups;
  const uint32_t *tables = (const uint32_t *)srs->d_tables;
  uint32_t pt_words = 2 * coord_words<typename C::F>(), y_words = coord_words<typename C::F>();
  if (srs->groups > 1 && n >= SRS_PRECOMPUTE_MIN_N) {
    c = srs->c; groups = srs->groups;
    tables = (const uint32_t *)srs->d_folded; pt_words = aligned_pt_words<C>(); y_words = aligned_y_words<C>();
  } else {
    c = msm_pick_c(n); groups = 1;
    if (const char *e = getenv("PCGPU_MSM_C")) { int v = atoi(e); if (v >= 8 && v <= 22) c = (uint32_t)v; }   // tuning / test knob
  }
  MsmGeom g = msm_geometry(n, c, groups, C::Fr::BITS, mont, srs->n, base_offset);
  g.pt_words = pt_words; g.y_words = y_words; g.pair_tdiv = ctx->pair_tdiv;
  int rc;
  // batched-affine rounds while buckets hold >= 64 points and a round still gives every thread >= 16 additions
  {
    size_t Tmax = 0, entries = (size_t)g.n * g.W;
    uint32_t R = 0;
    if constexpr (C::EXT == 1) {   // G2: no batched-affine rounds (R = 0)
      if ((rc = msm_pair_oneshot_threads<C>(&Tmax))) return rc;
      size_t avg = entries / g.TB;
      while (R < 8 && (avg >> R) >= 4 && (entries >> (R + 1)) >= 16 * Tmax) R++;
      if (const char *e = getenv("PCGPU_MSM_AFFINE_ROUNDS")) { int v = atoi(e); if (v >= 0 && v <= 12) R = (uint32_t)v; }
    }
    g.affine_rounds = R;
    uint64_t *lg = ctx->last_geom;
    memset(lg, 0, sizeof ctx->last_geom);
    lg[PCGPU_GEOM_PATH] = PCGPU_MSM_PATH_BUCKETS; lg[PCGPU_GEOM_N] = g.n; lg[PCGPU_GEOM_C] = g.c; lg[PCGPU_GEOM_W] = g.W;
    lg[PCGPU_GEOM_G] = g.G; lg[PCGPU_GEOM_R] = R; lg[PCGPU_GEOM_WAVE] = Tmax; lg[PCGPU_GEOM_ENTRIES] = entries;
    lg[PCGPU_GEOM_HEAVY] = UINT64_MAX;   // msm_collect fills it in from the pipeline's error words
  }
  if (g.affine_rounds && (rc = ensure_pow2<C>(ctx))) return rc;
  *g_out = g;
  uint32_t T = 0, tdiv = 0;
  rc = msm_run<C>(tables, g, d_scalars, ctx->msm_arena, d_planes, stride, d_err, st, ctx->prof, ctx->d_pow2[C::ID], &T, &tdiv);
  ctx->last_geom[PCGPU_GEOM_T] = T; ctx->last_geom[PCGPU_GEOM_TDIV] = tdiv;
  return rc;
}

// One MSM in two halves so that a caller can keep several pipelines in flight from one host thread:
//   msm_issue    launches the device pipeline on the context's stream and queues the copy of the S*c bit-plane sums (and the
//                error words) into the context's pinned zone -- returns without waiting
//   msm_collect  waits for that stream and combines the planes on the host (host_ec.hpp)
// MSMs below the small-path threshold complete inside msm_issue.
template <class C>
struct MsmPending {
  bool done = true;            // result already in `ready`
  host::HXYZZ<C> ready;
  MsmGeom g;
  size_t np = 0;
};

template <class C>
int msm_issue(pcgpu_ctx *ctx, const pcgpu_srs *srs, size_t base_offset, const uint32_t *d_scalars, size_t n, bool mont,
              MsmPending<C> *p) {
  rt::stream_t st = ctx->stream;
  p->done = true; p->ready = host::HXYZZ<C>::inf(); p->np = 0;
  if (n == 0) { memset(ctx->last_geom, 0, sizeof ctx->last_geom); return PCGPU_OK; }
  if (n <= SMALL_MAX_N && msm_small_enabled()) {
    MsmSmallProblem<C> pr{(const Affine<C> *)srs->d_tables + base_offset, d_scalars, nullptr, nullptr, (uint32_t)n};
    return msm_small_to_host<C>(ctx, &pr, 1, mont, &p->ready);
  }
  const XYZZ<C> *d_planes = nullptr; size_t stride = 0; uint32_t *d_err = nullptr;
  int rc = msm_device_planes<C>(ctx, srs, base_offset, d_scalars, n, mont, &p->g, &d_planes, &stride, &d_err);
  if (rc) return rc;
  p->np = (size_t)p->g.S * p->g.c;   // one-level: c planes per set; two-level: (h+1) + (c-1-h) = c planes per set as well
  static_assert(sizeof(host::HXYZZ<C>) == sizeof(XYZZ<C>), "host/device point layouts must agree");
  static_assert(PCGPU_MAX_PLANES * sizeof(XYZZ<C>) <= sizeof(PinnedZone::planes), "the plane sums must fit the pinned zone");
  if (p->np > PCGPU_MAX_PLANES || !ctx->h_pinned) return PCGPU_E_BADARG;
  PinnedZone *hp = ctx->h_pinned;
  if ((rc = rt::copy_d2h_2d(hp->planes, sizeof(XYZZ<C>), d_planes, stride * sizeof(XYZZ<C>), sizeof(XYZZ<C>), p->np, st))) return rc;
  if ((rc = rt::copy_d2h(hp->err, d_err, sizeof hp->err, st))) return rc;
  p->done = false;
  return PCGPU_OK;
}

template <class C>
int msm_collect(pcgpu_ctx *ctx, MsmPending<C> *p, host::HXYZZ<C> *out) {
  if (p->done) { *out = p->ready; return PCGPU_OK; }
  int rc = rt::stream_sync(ctx->stream);
  if (rc) return rc;
  ctx->prof.collect();
  const PinnedZone *hp = ctx->h_pinned;
  ctx->last_geom[PCGPU_GEOM_HEAVY] = hp->err[MSM_ERR_HEAVY];
  if (hp->err[MSM_ERR_RANGE]) return PCGPU_E_RANGE;
  auto t0 = std::chrono::steady_clock::now();
  const host::HXYZZ<C> *planes = (const host::HXYZZ<C> *)hp->planes;
  *out = p->g.h_split ? host::combine_bit_planes_2level<C>(planes, p->g.S, p->g.c, p->g.h_split)
                      : host::combine_bit_planes<C>(planes, p->g.S, p->g.c);
  if (ctx->prof.on) {
    ctx->prof.ms[6] += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    ctx->prof.cnt[6]++;
  }
  p->done = true; p->ready = *out;
  return PCGPU_OK;
}

// One MSM, synchronous.  d_scalars: device, n x 8 u32.
template <class C>
int msm_to_host(pcgpu_ctx *ctx, const pcgpu_srs *srs, size_t base_offset, const uint32_t *d_scalars, size_t n,
                bool mont, host::HXYZZ<C> *out) {
  MsmPending<C> p;
  int rc = msm_issue<C>(ctx, srs, base_offset, d_scalars, n, mont, &p);
  if (rc) return rc;
  return msm_collect<C>(ctx, &p, out);
}

// the n scalars (32 bytes each) of an MSM on the device: the caller's (PCGPU_DEVICE_PTRS) or a staged copy
static int stage_scalars(pcgpu_ctx *ctx, const void *scalars, size_t n, uint32_t flags, const uint32_t **d_scalars) {
  *d_scalars = nullptr;
  if (!n) return PCGPU_OK;
  Staging io(ctx, flags);
  io.in(*d_scalars, scalars, n * 32);
  return io.upload();
}

// ---------------------------------------------------------------------------------------------
// MSM entry points
// ---------------------------------------------------------------------------------------------
template <class C>
int msm_impl(pcgpu_ctx *ctx, const pcgpu_srs *srs, size_t base_offset, const void *scalars, size_t n, uint32_t flags,
             void *out_xy, uint8_t *out_inf, void *out_xyzz) {
  if (base_offset > srs->n || n > srs->n - base_offset) return PCGPU_E_LEN;
  int rc;
  const uint32_t *d_scalars;
  if ((rc = stage_scalars(ctx, scalars, n, flags, &d_scalars))) return rc;
  host::HXYZZ<C> r;
  if ((rc = msm_to_host<C>(ctx, srs, base_offset, d_scalars, n, (flags & PCGPU_SCALARS_MONT) != 0, &r))) return rc;
  if (out_xyzz) { memcpy(out_xyzz, &r, sizeof r); return PCGPU_OK; }
  host::to_affine<C>(r, out_xy, out_inf);
  return PCGPU_OK;
}

// ---------------------------------------------------------------------------------------------
// index-range-sharded MSM with the point-sum fused into the pipeline tail (peer.cuh; SURVEY.md 8e partitioning B)
// ---------------------------------------------------------------------------------------------
static const long long PEER_WAIT_CYCLES = 6000000000ll;   // ~3 s at 1.9 GHz: a missing peer becomes PCGPU_E_PEER, not a hang

template <class C>
int msm_peer_impl(pcgpu_ctx *ctx, const pcgpu_srs *srs, size_t base_offset, const void *scalars, size_t n, uint32_t flags,
                  void *const *win, uint32_t rank, uint32_t world, uint64_t epoch, void *out_xy, uint8_t *out_inf) {
  if (base_offset > srs->n || n > srs->n - base_offset) return PCGPU_E_LEN;
  rt::stream_t st = ctx->stream;
  const bool mont = (flags & PCGPU_SCALARS_MONT) != 0;
  int rc;
  const uint32_t *d_scalars;
  if ((rc = stage_scalars(ctx, scalars, n, flags, &d_scalars))) return rc;
  MsmPeerPushBody push;
  memset(&push, 0, sizeof push);
  for (uint32_t d = 0; d < world; d++) push.win[d] = (char *)win[d];
  push.rank = rank; push.world = world; push.epoch = epoch;
  uint32_t *d_timeout = &ctx->d_words->peer_timeout;
  bool pipeline = n > SMALL_MAX_N || (n > 0 && !msm_small_enabled());
  MsmGeom g;
  if (pipeline) {
    const XYZZ<C> *d_planes = nullptr; size_t stride = 0; uint32_t *d_err = nullptr;
    if ((rc = msm_device_planes<C>(ctx, srs, base_offset, d_scalars, n, mont, &g, &d_planes, &stride, &d_err))) return rc;
    const size_t np = (size_t)g.S * g.c;
    if (sizeof(PeerRecordHeader) + np * sizeof(XYZZ<C>) <= (size_t)PEER_RECORD_BYTES && stride == 1) {
      push.planes = (const uint32_t *)d_planes; push.plane_words = (uint32_t)(np * sizeof(XYZZ<C>) / 4);
      push.hdr.np = (uint32_t)np; push.hdr.S = g.S; push.hdr.c = g.c; push.hdr.h_split = g.h_split; push.d_err = d_err;
    } else {
      pipeline = false;   // record too large for a slot (no window folding): send the combined partial instead
    }
  }
  if (!pipeline) {
    // small or unfolded MSM: this rank's partial is finished on the host and pushed as a one-plane record
    host::HXYZZ<C> part;
    if ((rc = msm_to_host<C>(ctx, srs, base_offset, d_scalars, n, mont, &part))) return rc;
    static_assert(sizeof(XYZZ<C>) <= sizeof(DeviceWords::peer_partial), "the partial must fit its device slot");
    XYZZ<C> *d_one = (XYZZ<C> *)&ctx->d_words->peer_partial;
    if ((rc = rt::copy_h2d(d_one, &part, sizeof part, st))) return rc;
    push.planes = (const uint32_t *)d_one; push.plane_words = sizeof(XYZZ<C>) / 4;
    push.hdr.np = 1; push.hdr.S = 1; push.hdr.c = 1; push.hdr.h_split = 0; push.d_err = nullptr;
  }
  if ((rc = rt::dev_memset(d_timeout, 0, 4, st))) return rc;
  ctx->prof.begin(13, st);
  if ((rc = rt::launch_blocks<128>(push, world, 0, st))) return rc;
  if ((rc = rt::launch<32>(PeerWaitBody{(const char *)win[rank], world, (uint32_t)PEER_FLAG_OFFSET, epoch, PEER_WAIT_CYCLES, d_timeout}, world, st))) return rc;
  ctx->prof.end(13, st);
  // ONE copy brings every rank's record back
  std::unique_ptr<char[]> rec(new (std::nothrow) char[(size_t)world * PEER_RECORD_BYTES]);
  if (!rec) return PCGPU_E_OOM;
  uint32_t timed_out = 0;
  if ((rc = rt::copy_d2h(rec.get(), win[rank], (size_t)world * PEER_RECORD_BYTES, st))) return rc;
  if ((rc = rt::copy_d2h(&timed_out, d_timeout, 4, st))) return rc;
  if ((rc = rt::stream_sync(st))) return rc;
  ctx->prof.collect();
  if (timed_out) return PCGPU_E_PEER;
  host::HXYZZ<C> acc = host::HXYZZ<C>::inf();
  for (uint32_t r = 0; r < world; r++) {
    const char *p = rec.get() + (size_t)r * PEER_RECORD_BYTES;
    PeerRecordHeader h;
    memcpy(&h, p, sizeof h);
    if (h.err) return PCGPU_E_RANGE;
    if (h.np == 0 || h.np > PCGPU_MAX_PLANES || sizeof h + (size_t)h.np * sizeof(XYZZ<C>) > (size_t)PEER_RECORD_BYTES || h.np != h.S * h.c) return PCGPU_E_PEER;
    host::HXYZZ<C> planes[PEER_RECORD_BYTES / sizeof(XYZZ<C>) + 1];
    memcpy(planes, p + sizeof h, (size_t)h.np * sizeof(XYZZ<C>));
    acc = host::padd<C>(acc, h.h_split ? host::combine_bit_planes_2level<C>(planes, h.S, h.c, h.h_split)
                                       : host::combine_bit_planes<C>(planes, h.S, h.c));
  }
  host::to_affine<C>(acc, out_xy, out_inf);
  return PCGPU_OK;
}

// point-sum of XYZZ partials: a handful of additions and one inversion -- host work (host_ec.hpp)
template <class C>
int g1_sum_impl(pcgpu_ctx *, const void *xyzz, size_t count, void *out_xy, uint8_t *out_inf) {
  host::HXYZZ<C> acc = host::HXYZZ<C>::inf();
  for (size_t i = 0; i < count; i++) {
    host::HXYZZ<C> p;
    memcpy(&p, (const char *)xyzz + i * sizeof p, sizeof p);
    acc = host::padd<C>(acc, p);
  }
  host::to_affine<C>(acc, out_xy, out_inf);
  return PCGPU_OK;
}

// `count` MSMs over shared bases (hyrax/mod.rs:233-242)
template <class C>
int msm_batch_impl(pcgpu_ctx *ctx, const pcgpu_srs *srs, const void *scalars, size_t n, size_t count, uint32_t flags,
                   void *out_xy, uint8_t *out_inf) {
  if (n > srs->n) return PCGPU_E_LEN;
  rt::stream_t st = ctx->stream;
  int rc;
  const size_t psz = sizeof(Affine<C>);
  const bool mont = (flags & PCGPU_SCALARS_MONT) != 0;
  if (count == 0) return PCGPU_OK;
  if (!srs->d_comb || n == 0) {  // no comb tables: run the rows through the single-MSM pipeline
    for (size_t r = 0; r < count; r++) {
      rc = msm_impl<C>(ctx, srs, 0, (const char *)scalars + r * n * 32, n, flags, (char *)out_xy + r * psz,
                       out_inf ? out_inf + r : nullptr, nullptr);
      if (rc) return rc;
    }
    return PCGPU_OK;
  }
  CombGeom g; memset(&g, 0, sizeof g);
  g.n_bases = (uint32_t)srs->n; g.c = srs->comb_c; g.W = (C::Fr::BITS + g.c - 1) / g.c; g.NBk = 1u << (g.c - 1);
  g.n = (uint32_t)n; g.count = (uint32_t)count;
  g.seg_len = 64; if (count < 4096) { while (g.seg_len > 8 && count * ((n + g.seg_len - 1) / g.seg_len) < 65536) g.seg_len /= 2; }
  g.segs = (uint32_t)((n + g.seg_len - 1) / g.seg_len);
  g.scalar_bits = C::Fr::BITS; g.scalars_mont = mont ? 1 : 0;
  size_t ntasks = count * g.segs;
  uint64_t *lg = ctx->last_geom;
  memset(lg, 0, sizeof ctx->last_geom);
  lg[PCGPU_GEOM_PATH] = PCGPU_MSM_PATH_COMB; lg[PCGPU_GEOM_N] = n; lg[PCGPU_GEOM_C] = g.c; lg[PCGPU_GEOM_W] = g.W;
  lg[PCGPU_GEOM_SPLIT] = g.seg_len; lg[PCGPU_GEOM_ENTRIES] = ntasks;
  uint32_t *d_err; XYZZ<C> *partial; Affine<C> *d_out; const uint32_t *d_s;
  Staging io(ctx, flags);
  io.scratch(d_err, 64);
  io.scratch(partial, ntasks * sizeof(XYZZ<C>));
  io.scratch(d_out, count * psz);
  io.in(d_s, scalars, count * n * 32);
  if ((rc = io.upload())) return rc;
  if ((rc = rt::dev_memset(d_err, 0, 64, st))) return rc;
  ctx->prof.begin(10, st);
  if ((rc = rt::launch<128>(CombAccumulateBody<C>{(const Affine<C> *)srs->d_comb, d_s, g, partial, d_err}, ntasks, st))) return rc;
  if ((rc = ensure_pow2<C>(ctx))) return rc;
  if ((rc = rt::launch<64>(CombRowSumBody<C>{partial, g.segs, d_out, ctx->d_pow2[C::ID]}, count, st))) return rc;
  ctx->prof.end(10, st);
  std::vector<Affine<C>> h(count);
  uint32_t herr = 0;
  if ((rc = rt::copy_d2h(h.data(), d_out, count * psz, st))) return rc;
  if ((rc = rt::copy_d2h(&herr, d_err, 4, st))) return rc;
  if ((rc = rt::stream_sync(st))) return rc;
  ctx->prof.collect();
  if (herr) return PCGPU_E_RANGE;
  for (size_t r = 0; r < count; r++) {
    bool inf = h[r].is_inf();
    memcpy((char *)out_xy + r * psz, &h[r], psz);
    if (out_inf) out_inf[r] = inf ? 1 : 0;
  }
  return PCGPU_OK;
}

template <class C>
int fixed_base_impl(pcgpu_ctx *ctx, const void *base_xy, const void *scalars, size_t n, uint32_t flags, void *out_xy) {
  rt::stream_t st = ctx->stream;
  int rc;
  Affine<C> *table, *d_o; const uint32_t *d_s;
  Staging io(ctx, flags);
  io.scratch(table, 64 * 15 * sizeof(Affine<C>));
  io.in(d_s, scalars, n * 32);
  io.out(d_o, out_xy, n * sizeof(Affine<C>));
  if ((rc = io.upload())) return rc;
  Affine<C> base;
  memcpy(&base, base_xy, sizeof base);
  if ((rc = rt::launch<64>(FixedBaseTableBody<C>{base, table}, 64, st))) return rc;
  if ((rc = rt::launch<128>(FixedBaseMulBody<C>{table, d_s, d_o}, n, st))) return rc;
  if ((rc = io.download())) return rc;
  return rt::stream_sync(st);
}

// ---------------------------------------------------------------------------------------------
// MultilinearPC (mlpc.cuh): committer key with pair-folded G2 bases, open = fold chain + nv G2 MSMs
// ---------------------------------------------------------------------------------------------
struct pcgpu_mlpc {
  int curve;        // the pairing curve (PCGPU_BLS12_381 / PCGPU_BN254)
  uint32_t nv;
  pcgpu_srs key;    // every level's folded bases, level i at mlpc_level_offset(nv, i); key.curve is the G2 group id
};

template <class C>
int mlpc_register_impl(pcgpu_ctx *ctx, uint32_t nv, const void *const *powers_of_h, const uint8_t *const *inf, uint32_t flags,
                       pcgpu_mlpc *m) {
  const size_t psz = sizeof(Affine<C>), n0 = (size_t)1 << nv;
  rt::stream_t st = ctx->stream;
  int rc;
  for (uint32_t i = 0; i < nv; i++) if (!powers_of_h[i]) return PCGPU_E_BADARG;
  if ((rc = rt::dev_malloc(&m->key.d_tables, psz * (n0 - 1)))) return rc;
  Affine<C> *raw; uint8_t *d_inf;
  Staging io(ctx, 0);
  io.scratch(raw, psz * n0);
  io.scratch(d_inf, n0);
  if ((rc = io.upload())) return rc;
  for (uint32_t i = 0; i < nv; i++) {
    const size_t len = n0 >> i;
    if (flags & PCGPU_DEVICE_PTRS) rc = rt::copy_d2d(raw, powers_of_h[i], psz * len, st);
    else rc = rt::copy_h2d(raw, powers_of_h[i], psz * len, st);
    if (rc) return rc;
    if (inf && inf[i]) {
      if (flags & PCGPU_DEVICE_PTRS) rc = rt::copy_d2d(d_inf, inf[i], len, st);
      else rc = rt::copy_h2d(d_inf, inf[i], len, st);
      if (rc) return rc;
      if ((rc = rt::launch<256>(SrsZeroIdentityBody{(uint32_t *)raw, d_inf, (uint32_t)(psz / 4)}, len, st))) return rc;
    }
    Affine<C> *out = (Affine<C> *)m->key.d_tables + mlpc_level_offset(nv, i);
    if ((rc = rt::launch<128>(PairFoldBasesBody<C>{raw, out}, len / 2, st))) return rc;
    if ((rc = rt::stream_sync(st))) return rc;   // the next level's upload overwrites raw
  }
  m->key.n = n0 - 1; m->key.c = 0; m->key.groups = 1;
  return PCGPU_OK;
}

template <class C>
int mlpc_open_impl(pcgpu_ctx *ctx, const pcgpu_mlpc *m, const void *evals, size_t n, const void *point, uint32_t flags,
                   void *out_xy, uint8_t *out_inf, void *out_value) {
  using R = typename C::Fr;
  const uint32_t nv = m->nv;
  const size_t n0 = (size_t)1 << nv, psz = sizeof(Affine<C>);
  if (n != n0) return PCGPU_E_LEN;   // "Invalid size of polynomial" (multilinear_pc/mod.rs:136)
  rt::stream_t st = ctx->stream;
  int rc;
  const uint32_t *d_ev, *d_pt; uint32_t *d_q, *d_ra, *d_rb;
  Staging io(ctx, flags);
  io.in(d_ev, evals, n0 * 32);
  io.host_in(d_pt, point, (size_t)nv * 32);
  io.scratch(d_q, (n0 - 1) * 32);
  io.scratch(d_ra, n0 / 2 * 32);
  io.scratch(d_rb, n0 / 2 * 32);
  if ((rc = io.upload())) return rc;
  ctx->prof.begin(16, st);
  const uint32_t *r = d_ev;
  for (uint32_t i = 0; i < nv; i++) {
    uint32_t *r_out = (i & 1) ? d_rb : d_ra;
    if ((rc = rt::launch<256>(MlpcFoldBody<R>{r, d_pt, i, d_q + mlpc_level_offset(nv, i) * 8, r_out}, n0 >> (i + 1), st))) return rc;
    r = r_out;
  }
  ctx->prof.end(16, st);
  uint32_t value[8];
  if ((rc = rt::copy_d2h(value, r, 32, st))) return rc;
  if ((rc = rt::stream_sync(st))) return rc;
  ctx->prof.collect();
  if (out_value) memcpy(out_value, value, 32);
  for (uint32_t i = 0; i < nv; i++) {   // the levels are independent now: level i is sum_b q_i[b] H'_i[b]
    const size_t off = mlpc_level_offset(nv, i);
    host::HXYZZ<C> res;
    if ((rc = msm_to_host<C>(ctx, &m->key, off, d_q + off * 8, n0 >> (i + 1), true, &res))) return rc;
    host::to_affine<C>(res, (char *)out_xy + i * psz, out_inf ? out_inf + i : nullptr);
  }
  return PCGPU_OK;
}


// ---------------------------------------------------------------------------------------------
// Fr vector entry points
// ---------------------------------------------------------------------------------------------
template <class C>
int fr_from_mont_impl(pcgpu_ctx *ctx, const void *in, void *out, size_t n, uint32_t flags) {
  using R = typename C::Fr;
  rt::stream_t st = ctx->stream;
  int rc;
  if (n == 0) return PCGPU_OK;
  const uint32_t *d_in; uint32_t *d_out;
  Staging io(ctx, flags);
  io.in(d_in, in, n * 32);
  io.out(d_out, out, n * 32);
  if ((rc = io.upload())) return rc;
  if ((rc = rt::launch<256>(FrFromMontBody<R>{d_in, d_out}, n, st))) return rc;
  if ((rc = io.download())) return rc;
  return rt::stream_sync(st);
}

template <class C>
int fr_mul_impl(pcgpu_ctx *ctx, const void *a, const void *b, void *out, size_t n, uint32_t flags) {
  using R = typename C::Fr;
  rt::stream_t st = ctx->stream;
  int rc;
  if (n == 0) return PCGPU_OK;
  const uint32_t *d_a, *d_b; uint32_t *d_o;
  Staging io(ctx, flags);
  io.in(d_a, a, n * 32);
  io.in(d_b, b, n * 32);
  io.out(d_o, out, n * 32);
  if ((rc = io.upload())) return rc;
  if ((rc = rt::launch<256>(FrMulBody<R>{d_a, d_b, d_o}, n, st))) return rc;
  if ((rc = io.download())) return rc;
  return rt::stream_sync(st);
}

template <class C>
int fr_axpy_impl(pcgpu_ctx *ctx, void *y, const void *c, const void *x, size_t n, uint32_t flags) {
  using R = typename C::Fr;
  rt::stream_t st = ctx->stream;
  int rc;
  if (n == 0) return PCGPU_OK;
  const uint32_t *d_c, *d_x; uint32_t *d_y;
  Staging io(ctx, flags);
  io.host_in(d_c, c, 32);
  io.inout(d_y, y, n * 32);
  io.in(d_x, x, n * 32);
  if ((rc = io.upload())) return rc;
  ctx->prof.begin(8, st);
  if ((rc = rt::launch<256>(FrAxpyBody<R>{d_y, d_c, d_x}, n, st))) return rc;
  ctx->prof.end(8, st);
  if ((rc = io.download())) return rc;
  rc = rt::stream_sync(st);
  ctx->prof.collect();
  return rc;
}


template <class C>
int fr_div_impl(pcgpu_ctx *ctx, const void *p, size_t n, const void *z, void *q, void *rem, uint32_t flags) {
  using R = typename C::Fr;
  rt::stream_t st = ctx->stream;
  int rc;
  const uint32_t *d_z, *d_p; uint32_t *d_rem, *scratch, *d_q;
  Staging io(ctx, flags);
  io.host_in(d_z, z, 32);
  io.scratch(d_rem, 32);
  io.scratch(scratch, div_scratch_words(n) * 4);
  io.in(d_p, p, n * 32);
  io.out(d_q, q, n > 1 ? (n - 1) * 32 : 0);
  if ((rc = io.upload())) return rc;
  ctx->prof.begin(7, st);
  if ((rc = fr_div_linear<R>(d_p, n, d_z, d_q, d_rem, scratch, st))) return rc;
  ctx->prof.end(7, st);
  if ((rc = io.download())) return rc;
  uint32_t hrem[8];
  if ((rc = rt::copy_d2h(hrem, d_rem, 32, st))) return rc;
  if ((rc = rt::stream_sync(st))) return rc;
  if ((rc = fr_div_check(scratch, n, st))) return rc;
  if (rem) memcpy(rem, hrem, 32);
  ctx->prof.collect();
  return PCGPU_OK;
}


template <class C>
int fr_ip_impl(pcgpu_ctx *ctx, const void *a, const void *b, size_t n, void *out, uint32_t flags) {
  using R = typename C::Fr;
  rt::stream_t st = ctx->stream;
  int rc;
  uint32_t *scratch, *d_out; const uint32_t *d_a, *d_b;
  Staging io(ctx, flags);
  io.scratch(scratch, (IP_THREADS + IP_THREADS / IP_BLOCK + 8) * 32);
  io.scratch(d_out, 32);
  io.in(d_a, a, n * 32);
  io.in(d_b, b, n * 32);
  if ((rc = io.upload())) return rc;
  if ((rc = fr_inner_product<R>(d_a, d_b, n, d_out, scratch, st))) return rc;
  if ((rc = rt::copy_d2h(out, d_out, 32, st))) return rc;
  return rt::stream_sync(st);
}


template <class C>
int fr_row_mul_impl(pcgpu_ctx *ctx, const void *v, const void *m, size_t rows, size_t cols, void *out, uint32_t flags) {
  using R = typename C::Fr;
  rt::stream_t st = ctx->stream;
  int rc;
  if (cols == 0) return PCGPU_OK;
  const uint32_t *dv, *dm; uint32_t *dout;
  Staging io(ctx, flags);
  io.in(dv, v, rows * 32);
  io.in(dm, m, rows * cols * 32);
  io.out(dout, out, cols * 32);
  if ((rc = io.upload())) return rc;
  if ((rc = rt::launch<128>(FrRowMulBody<R>{dv, dm, rows, cols, dout}, cols, st))) return rc;
  if ((rc = io.download())) return rc;
  return rt::stream_sync(st);
}


// ---------------------------------------------------------------------------------------------
// KZG10 fused calls
// ---------------------------------------------------------------------------------------------
static int device_trim_trailing_zeros(pcgpu_ctx *ctx, const void *d_coeffs, size_t *n);
static size_t trim_trailing_zeros(const void *coeffs, size_t n) {
  const uint64_t *c = (const uint64_t *)coeffs;
  while (n > 0 && !(c[4 * (n - 1)] | c[4 * (n - 1) + 1] | c[4 * (n - 1) + 2] | c[4 * (n - 1) + 3])) n--;
  return n;
}

template <class C>
int kzg_commit_impl(pcgpu_ctx *ctx, const pcgpu_srs *pg, const void *coeffs, size_t n, const pcgpu_srs *gamma,
                           const void *blind, size_t n_blind, uint32_t flags, void *out_xy, uint8_t *out_inf) {
  bool dev = (flags & PCGPU_DEVICE_PTRS) != 0;
  if (!dev) { n = trim_trailing_zeros(coeffs, n); n_blind = trim_trailing_zeros(blind, n_blind); }
  else { int trc; if ((trc = device_trim_trailing_zeros(ctx, coeffs, &n)) || (trc = device_trim_trailing_zeros(ctx, blind, &n_blind))) return trc; }
  if (n > pg->n) return PCGPU_E_DEGREE;                      // check_degree_is_too_large, kzg10/mod.rs:163
  if (n_blind && (!gamma || n_blind > gamma->n)) return PCGPU_E_HIDING;  // check_hiding_bound, :190-193
  int rc;
  const uint32_t *d_c, *d_b;
  Staging io(ctx, flags);
  io.in(d_c, coeffs, n * 32);
  io.in(d_b, blind, n_blind * 32);
  if ((rc = io.upload())) return rc;
  host::HXYZZ<C> comm, rnd;
  if ((rc = msm_to_host<C>(ctx, pg, 0, d_c, n, true, &comm))) return rc;            // :175-178
  if (n_blind) {
    if ((rc = msm_to_host<C>(ctx, gamma, 0, d_b, n_blind, true, &rnd))) return rc;  // :199-203
    comm = host::padd<C>(comm, rnd);                                                  // :206
  }
  host::to_affine<C>(comm, out_xy, out_inf);                                           // :209
  return PCGPU_OK;
}


template <class C>
int kzg_open_impl(pcgpu_ctx *ctx, const pcgpu_srs *pg, const void *coeffs, size_t n, const void *z,
                         const pcgpu_srs *gamma, const void *blind, size_t n_blind, uint32_t flags, void *out_xy,
                         uint8_t *out_inf, void *out_random_v) {
  using R = typename C::Fr;
  bool dev = (flags & PCGPU_DEVICE_PTRS) != 0;
  if (!dev) { n = trim_trailing_zeros(coeffs, n); n_blind = trim_trailing_zeros(blind, n_blind); }
  else { int trc; if ((trc = device_trim_trailing_zeros(ctx, coeffs, &n)) || (trc = device_trim_trailing_zeros(ctx, blind, &n_blind))) return trc; }
  if (n > pg->n) return PCGPU_E_DEGREE;  // kzg10/mod.rs:292
  if (n_blind && (!gamma || n_blind - 1 > gamma->n)) return PCGPU_E_HIDING;
  rt::stream_t st = ctx->stream;
  int rc;
  const uint32_t *d_z, *d_c, *d_b; uint32_t *d_rem, *d_rv, *scratch, *d_q, *d_bq;
  Staging io(ctx, flags);
  io.host_in(d_z, z, 32);
  io.scratch(d_rem, 32);
  io.scratch(d_rv, 32);
  io.scratch(scratch, div_scratch_words(n > n_blind ? n : n_blind) * 4);
  io.scratch(d_q, n * 32);
  io.scratch(d_bq, n_blind * 32);
  io.in(d_c, coeffs, n * 32);
  io.in(d_b, blind, n_blind * 32);
  if ((rc = io.upload())) return rc;
  // witness = p / (X - z)   (kzg10/mod.rs:222-226)
  ctx->prof.begin(7, st);
  if ((rc = fr_div_linear<R>(d_c, n, d_z, d_q, d_rem, scratch, st))) return rc;
  ctx->prof.end(7, st);
  host::HXYZZ<C> w, rw;
  if ((rc = msm_to_host<C>(ctx, pg, 0, d_q, n ? n - 1 : 0, true, &w))) return rc;     // :255-258
  if ((rc = fr_div_check(scratch, n, st))) return rc;
  if (n_blind) {
    if ((rc = fr_div_linear<R>(d_b, n_blind, d_z, d_bq, d_rv, scratch, st))) return rc;  // rem = blind(z), :264
    if ((rc = msm_to_host<C>(ctx, gamma, 0, d_bq, n_blind - 1, true, &rw))) return rc;  // :270-273
    if ((rc = fr_div_check(scratch, n_blind, st))) return rc;
    if (out_random_v) {
      if ((rc = rt::copy_d2h(out_random_v, d_rv, 32, st))) return rc;
      if ((rc = rt::stream_sync(st))) return rc;
    }
    w = host::padd<C>(w, rw);
  }
  host::to_affine<C>(w, out_xy, out_inf);                                              // :281
  return PCGPU_OK;
}



// length of the polynomial without its trailing zero coefficients, for coefficients that live on the device
// (DensePolynomial truncates them; the host path does the same scan in trim_trailing_zeros).  One 32-byte read in the common
// case of a non-zero leading coefficient, otherwise a scan kernel.
struct FrLastNonzeroBody {
  const uint32_t *v; size_t n; unsigned long long *last_plus_one;
  PCGPU_KERNEL_DEV void operator()(size_t i) const {
    const uint32_t *e = v + 8 * i;
    uint32_t o = 0;
    for (int l = 0; l < 8; l++) o |= e[l];
    if (o) {
#ifdef __CUDA_ARCH__
      atomicMax(last_plus_one, (unsigned long long)(i + 1));
#else
      if (*last_plus_one < i + 1) *last_plus_one = i + 1;
#endif
    }
  }
};
static int device_trim_trailing_zeros(pcgpu_ctx *ctx, const void *d_coeffs, size_t *n) {
  rt::stream_t st = ctx->stream;
  int rc;
  while (*n > 0) {
    uint64_t top[4];
    if ((rc = rt::copy_d2h(top, (const char *)d_coeffs + (*n - 1) * 32, 32, st))) return rc;
    if ((rc = rt::stream_sync(st))) return rc;
    if (top[0] | top[1] | top[2] | top[3]) return PCGPU_OK;
    unsigned long long *d_last = &ctx->d_words->last_nonzero;
    if ((rc = rt::dev_memset(d_last, 0, sizeof *d_last, st))) return rc;
    if ((rc = rt::launch<256>(FrLastNonzeroBody{(const uint32_t *)d_coeffs, *n, d_last}, *n, st))) return rc;
    unsigned long long h = 0;
    if ((rc = rt::copy_d2h(&h, d_last, 8, st))) return rc;
    if ((rc = rt::stream_sync(st))) return rc;
    *n = (size_t)h;
    return PCGPU_OK;
  }
  return PCGPU_OK;
}

// KZG10::commit followed by KZG10::open of the SAME polynomial (what a Marlin prover does per polynomial: commit,
// marlin_pc/mod.rs:192-241, then open, :245-336) in one call: the coefficients are uploaded ONCE, the commitment MSM runs
// on `ctx`'s stream while the witness division and the witness MSM run on the sibling context `sib`'s stream, so the
// latency-bound stages of one pipeline hide under the multiply-bound stages of the other.  Non-hiding path only (the caller
// falls back to the two separate calls when blinding polynomials are present).
template <class C>
int kzg_commit_open_impl(pcgpu_ctx *ctx, pcgpu_ctx *sib, const pcgpu_srs *pg, const void *coeffs, size_t n, const void *z,
                         uint32_t flags, void *out_c_xy, uint8_t *out_c_inf, void *out_w_xy, uint8_t *out_w_inf) {
  using R = typename C::Fr;
  const bool dev = (flags & PCGPU_DEVICE_PTRS) != 0;
  int rc;
  if (!dev) n = trim_trailing_zeros(coeffs, n);
  else if ((rc = device_trim_trailing_zeros(ctx, coeffs, &n))) return rc;
  if (n > pg->n) return PCGPU_E_DEGREE;                      // kzg10/mod.rs:163, :292
  rt::stream_t sa = ctx->stream, sb = sib->stream;
  const uint32_t *d_c, *d_z; uint32_t *d_rem, *scratch, *d_q;
  Staging a(ctx, flags), b(sib, flags);   // the coefficients on ctx's stream, the witness side on sib's
  a.in(d_c, coeffs, n * 32);
  b.host_in(d_z, z, 32);
  b.scratch(d_rem, 32);
  b.scratch(scratch, div_scratch_words(n) * 4);
  b.scratch(d_q, n * 32);
  if ((rc = a.upload()) || (rc = b.upload())) return rc;
  if (!ctx->ev_ok) { if ((rc = rt::event_create(&ctx->ev_upload))) return rc; ctx->ev_ok = true; }
  if ((rc = rt::event_record(ctx->ev_upload, sa))) return rc;
  if ((rc = rt::stream_wait_event(sb, ctx->ev_upload))) return rc;
  MsmPending<C> pc, pw;
  // witness side first: its division is short and its MSM then overlaps the commitment's
  sib->prof.begin(7, sb);
  if ((rc = fr_div_linear<R>(d_c, n, d_z, d_q, d_rem, scratch, sb))) return rc;      // kzg10/mod.rs:222-226
  sib->prof.end(7, sb);
  if ((rc = msm_issue<C>(ctx, pg, 0, d_c, n, true, &pc))) return rc;                 // :175-178
  if ((rc = msm_issue<C>(sib, pg, 0, d_q, n ? n - 1 : 0, true, &pw))) return rc;     // :255-258
  host::HXYZZ<C> comm, w;
  if ((rc = msm_collect<C>(ctx, &pc, &comm))) return rc;
  if ((rc = msm_collect<C>(sib, &pw, &w))) return rc;
  if ((rc = fr_div_check(scratch, n, sb))) return rc;
  host::to_affine<C>(comm, out_c_xy, out_c_inf);                                      // :209
  host::to_affine<C>(w, out_w_xy, out_w_inf);                                         // :281
  return PCGPU_OK;
}

// ---------------------------------------------------------------------------------------------
// IPA halving loop (device-resident)
// ---------------------------------------------------------------------------------------------
// Device buffers are carved from the context's IPA arena by ipa_begin.
struct pcgpu_ipa {
  int curve; size_t n0, n;
  void *d_key;               // n0 affine points (folded in place until the key is frozen)
  uint32_t *d_coeffs, *d_z;  // n0 Fr each
  uint32_t *d_ip_scratch;    // fr_inner_product's scratch
  uint32_t *d_point;         // the evaluation point z (1 Fr)
  uint32_t *d_ip;            // <coeffs_r, z_l>, <coeffs_l, z_r> (2 Fr)
  uint32_t *d_ch, *d_chi;    // the round's challenge and its inverse (1 Fr each)
  void *d_h;                 // h' (one affine point)
  pcgpu_srs view;            // non-owning SRS view over d_key for the MSM pipeline
  size_t frozen_m;           // 0: the key is folded explicitly; else the key stays at frozen_m points (ipa.cuh, "late rounds")
  uint32_t *d_w, *d_sl, *d_sr;   // frozen key: the weights and the l / r MSM scalars (SMALL_MAX_N Fr each)
};

template <class C>
static int ensure_pow2(pcgpu_ctx *ctx) {
  using QP = typename C::Fq;
  if (ctx->d_pow2[C::ID]) return PCGPU_OK;
  int rc;
  if ((rc = rt::dev_malloc((void **)&ctx->d_pow2[C::ID], pow2_table_bytes<QP>()))) return rc;
  return rt::launch<32>(Pow2TableBody<QP>{ctx->d_pow2[C::ID]}, 1, ctx->stream);
}

#ifndef PCGPU_IPA_FOLD_MIN_BLOCKS
#define PCGPU_IPA_FOLD_MIN_BLOCKS 2
#endif
enum { IPA_FOLD_MIN_BLOCKS = PCGPU_IPA_FOLD_MIN_BLOCKS };
// freeze the key at its current length (<= SMALL_MAX_N): weights start at one
template <class C>
static int ipa_freeze(pcgpu_ctx *ctx, pcgpu_ipa *st) {
  using R = typename C::Fr;
  st->frozen_m = st->n;
  return rt::launch<128>(FrFillOneBody<R>{st->d_w}, st->n, ctx->stream);
}
inline bool ipa_freeze_enabled() {
  const char *e = getenv("PCGPU_IPA_FREEZE");
  return msm_small_enabled() && !(e && e[0] == '0');
}

template <class C>
int ipa_begin_impl(pcgpu_ctx *ctx, const void *key_xy, size_t n, const void *coeffs, size_t n_coeffs, const void *point,
                   uint32_t flags, pcgpu_ipa *st) {
  using R = typename C::Fr;
  rt::stream_t s = ctx->stream;
  int rc;
  bool dev = (flags & PCGPU_DEVICE_PTRS) != 0;
  st->curve = C::ID; st->n0 = st->n = n; st->frozen_m = 0;
  if ((rc = ensure_pow2<C>(ctx))) return rc;
  // one arena per context, grown on demand and kept: an open costs no cudaMalloc / cudaFree after the first
  if (ctx->ipa_active) return PCGPU_E_BADARG;          // one halving loop at a time per context
  Affine<C> *key, *h;
  rc = ctx->ipa_arena.carve([&](auto &&buf) {
    buf(key, n); buf(st->d_coeffs, 8 * n); buf(st->d_z, 8 * n); buf(st->d_ip_scratch, 8 * (IP_THREADS + IP_THREADS / IP_BLOCK));
    buf(st->d_point, 8); buf(st->d_ip, 2 * 8); buf(st->d_ch, 8); buf(st->d_chi, 8); buf(h, 1);
    buf(st->d_w, 8 * SMALL_MAX_N); buf(st->d_sl, 8 * SMALL_MAX_N); buf(st->d_sr, 8 * SMALL_MAX_N);
  });
  if (rc) return rc;
  st->d_key = key; st->d_h = h;
  ctx->ipa_active = true;
  if ((rc = dev ? rt::copy_d2d(st->d_key, key_xy, n * sizeof(Affine<C>), s) : rt::copy_h2d(st->d_key, key_xy, n * sizeof(Affine<C>), s))) return rc;
  if ((rc = rt::dev_memset(st->d_coeffs, 0, n * 32, s))) return rc;
  if (n_coeffs && (rc = dev ? rt::copy_d2d(st->d_coeffs, coeffs, n_coeffs * 32, s) : rt::copy_h2d(st->d_coeffs, coeffs, n_coeffs * 32, s))) return rc;
  if ((rc = rt::copy_h2d(st->d_point, point, 32, s))) return rc;
  if ((rc = rt::launch<128>(FrPowersBody<R>{st->d_point, st->d_z}, n, s))) return rc;
  st->view.curve = C::ID; st->view.n = n; st->view.c = 0; st->view.groups = 1; st->view.d_tables = st->d_key; st->view.d_folded = nullptr;
  st->view.d_comb = nullptr; st->view.comb_c = 0;
  if (n <= SMALL_MAX_N && n > 1 && ipa_freeze_enabled() && (rc = ipa_freeze<C>(ctx, st))) return rc;
  return rt::stream_sync(s);
}

template <class C>
int ipa_round_lr_impl(pcgpu_ctx *ctx, pcgpu_ctx *sib, pcgpu_ipa *st, const void *h_prime_xy, void *out_l_xy, uint8_t *out_l_inf,
                      void *out_r_xy, uint8_t *out_r_inf) {
  using R = typename C::Fr;
  rt::stream_t s = ctx->stream;
  int rc;
  size_t m = st->n / 2;
  if (m == 0) return PCGPU_E_BADARG;
  const uint32_t *cl = st->d_coeffs, *cr = st->d_coeffs + 8 * m, *zl = st->d_z, *zr = st->d_z + 8 * m;
  uint32_t *d_ip = st->d_ip, *scr = st->d_ip_scratch;
  const Affine<C> *d_h = (const Affine<C> *)st->d_h;
  uint64_t ip_m[2][4], ip_c[2][4];
  if (st->frozen_m) {
    // frozen key: both commitments are frozen_m-term MSMs over the same points, scalars expanded on the device
    const size_t M = st->frozen_m;
    if ((rc = fr_inner_product<R>(cr, zl, m, d_ip, scr, s))) return rc;
    if ((rc = fr_inner_product<R>(cl, zr, m, d_ip + 8, scr, s))) return rc;
    if ((rc = rt::copy_h2d(st->d_h, h_prime_xy, sizeof(Affine<C>), s))) return rc;
    if ((rc = rt::launch<128>(IpaFrozenScalarsBody<R>{st->d_w, st->d_coeffs, (uint32_t)st->n, st->d_sl, st->d_sr}, M, s))) return rc;
    const Affine<C> *key = (const Affine<C> *)st->d_key;
    MsmSmallProblem<C> pr[2] = {{key, st->d_sl, d_h, d_ip, (uint32_t)M}, {key, st->d_sr, d_h, d_ip + 8, (uint32_t)M}};
    host::HXYZZ<C> lr[2];
    if ((rc = msm_small_to_host<C>(ctx, pr, 2, true, lr))) return rc;
    host::to_affine<C>(lr[0], out_l_xy, out_l_inf);
    host::to_affine<C>(lr[1], out_r_xy, out_r_inf);
    return PCGPU_OK;
  }
  if (m <= 2 * SMALL_MAX_N && msm_small_enabled()) {
    // rounds of <= 8192-term commitments (the bucket pipeline's fixed cost dominates at this size): both commitments, each with its  + h' * <.,.>  term, in ONE launch; the inner products never leave HBM
    if ((rc = fr_inner_product<R>(cr, zl, m, d_ip, scr, s))) return rc;
    if ((rc = fr_inner_product<R>(cl, zr, m, d_ip + 8, scr, s))) return rc;
    if ((rc = rt::copy_h2d(st->d_h, h_prime_xy, sizeof(Affine<C>), s))) return rc;
    const Affine<C> *key = (const Affine<C> *)st->view.d_tables;
    MsmSmallProblem<C> pr[2] = {{key, cr, d_h, d_ip, (uint32_t)m},          // cm_commit(key_l, coeffs_r) + h' <c_r, z_l>
                                {key + m, cl, d_h, d_ip + 8, (uint32_t)m}};  // cm_commit(key_r, coeffs_l) + h' <c_l, z_r>
    host::HXYZZ<C> lr[2];
    if ((rc = msm_small_to_host<C>(ctx, pr, 2, true, lr))) return rc;
    host::to_affine<C>(lr[0], out_l_xy, out_l_inf);
    host::to_affine<C>(lr[1], out_r_xy, out_r_inf);
    return PCGPU_OK;
  }
  // <coeffs_r, z_l>, <coeffs_l, z_r> (results fetched after the MSMs have been queued), then the two commitments: cm_commit(key_l,
  // coeffs_r) on this context's stream and cm_commit(key_r, coeffs_l) on the sibling's, so their latency-bound stages overlap
  if ((rc = fr_inner_product<R>(cr, zl, m, d_ip, scr, s))) return rc;
  if ((rc = fr_inner_product<R>(cl, zr, m, d_ip + 8, scr, s))) return rc;   // stream order: the first product is complete
  if ((rc = rt::copy_d2h(ip_m[0], d_ip, 32, s))) return rc;
  if ((rc = rt::copy_d2h(ip_m[1], d_ip + 8, 32, s))) return rc;
  host::HXYZZ<C> l, r;
  if (sib) {
    MsmPending<C> pl, pr;
    if ((rc = msm_issue<C>(ctx, &st->view, 0, cr, m, true, &pl))) return rc;
    if ((rc = msm_issue<C>(sib, &st->view, m, cl, m, true, &pr))) return rc;
    if ((rc = msm_collect<C>(ctx, &pl, &l))) return rc;
    if ((rc = msm_collect<C>(sib, &pr, &r))) return rc;
  } else {
    if ((rc = msm_to_host<C>(ctx, &st->view, 0, cr, m, true, &l))) return rc;  // cm_commit(key_l, coeffs_r)
    if ((rc = msm_to_host<C>(ctx, &st->view, m, cl, m, true, &r))) return rc;  // cm_commit(key_r, coeffs_l)
  }
  if ((rc = rt::stream_sync(s))) return rc;
  host::fr_from_mont_host<R>(ip_m[0], ip_c[0]);
  host::fr_from_mont_host<R>(ip_m[1], ip_c[1]);
  l = host::padd<C>(l, host::pmul_affine<C>(h_prime_xy, ip_c[0]));
  r = host::padd<C>(r, host::pmul_affine<C>(h_prime_xy, ip_c[1]));
  host::to_affine<C>(l, out_l_xy, out_l_inf);
  host::to_affine<C>(r, out_r_xy, out_r_inf);
  return PCGPU_OK;
}

template <class C>
int ipa_round_fold_impl(pcgpu_ctx *ctx, pcgpu_ipa *st, const void *challenge, const void *challenge_inv) {
  using R = typename C::Fr;
  rt::stream_t s = ctx->stream;
  int rc;
  size_t m = st->n / 2;
  if (m == 0) return PCGPU_E_BADARG;
  if ((rc = rt::copy_h2d(st->d_ch, challenge, 32, s))) return rc;
  if ((rc = rt::copy_h2d(st->d_chi, challenge_inv, 32, s))) return rc;
  if ((rc = rt::launch<256>(FrAxpyBody<R>{st->d_coeffs, st->d_chi, st->d_coeffs + 8 * m}, m, s))) return rc;  // :691-693
  if ((rc = rt::launch<256>(FrAxpyBody<R>{st->d_z, st->d_ch, st->d_z + 8 * m}, m, s))) return rc;              // :695-697
  if (st->frozen_m) {   // the key's fold is a multiplication of the weights (ipa.cuh)
    if ((rc = rt::launch<128>(IpaFrozenWeightBody<R>{st->d_w, st->d_ch, (uint32_t)st->n}, st->frozen_m, s))) return rc;
    st->n = m;
    return rt::stream_sync(s);
  }
  uint64_t canon[4];
  host::fr_from_mont_host<R>(challenge, canon);
  host::GlvSplit gs;
  gs.ok = false;
  if (C::Fq::COFACTOR_ONE) {                       // phi acts as lambda on the whole curve only when the cofactor is 1
    const char *e = getenv("PCGPU_IPA_GLV");
    if (!(e && e[0] == '0')) gs = host::glv_decompose<C>(canon);
  }
  if (gs.ok) {
    G1FoldGlvBody<C> gb; gb.key = (Affine<C> *)st->d_key; gb.m = (uint32_t)m;
    memcpy(gb.u1_nz, gs.u1_nz, sizeof gb.u1_nz); memcpy(gb.u1_sg, gs.u1_sg, sizeof gb.u1_sg);
    memcpy(gb.u2_nz, gs.u2_nz, sizeof gb.u2_nz); memcpy(gb.u2_sg, gs.u2_sg, sizeof gb.u2_sg);
    gb.neg1 = gs.neg1; gb.neg2 = gs.neg2; gb.ncols = gs.jsf_len; gb.pow2 = ctx->d_pow2[C::ID];
    // registers: 190 uncapped (2 blocks of 128 threads per SM); 3 or 4 resident blocks cap them at 168 / 128 (PCGPU_IPA_FOLD_OCC)
    int occ = IPA_FOLD_MIN_BLOCKS;
    if (const char *e = getenv("PCGPU_IPA_FOLD_OCC")) { int v = atoi(e); if (v >= 2 && v <= 4) occ = v; }
    if (occ == 2) rc = rt::launch<128>(gb, m, s);
    else if (occ == 3) rc = rt::launch_occ<128, 3>(gb, m, s);
    else rc = rt::launch_occ<128, 4>(gb, m, s);
    if (rc) return rc;                                                                                      // :699-707
  } else {
    G1FoldBody<C> fb; fb.key = (Affine<C> *)st->d_key; fb.m = (uint32_t)m;
    memcpy(fb.chal, canon, 32); fb.pow2 = ctx->d_pow2[C::ID];
    if ((rc = rt::launch<128>(fb, m, s))) return rc;                                                        // :699-707
  }
  st->n = m; st->view.n = m;
  if (m <= SMALL_MAX_N && m > 1 && ipa_freeze_enabled() && (rc = ipa_freeze<C>(ctx, st))) return rc;
  return rt::stream_sync(s);
}

template <class C>
int ipa_finish_impl(pcgpu_ctx *ctx, pcgpu_ipa *st, void *out_final_key_xy, void *out_c) {
  rt::stream_t s = ctx->stream;
  int rc;
  if (out_final_key_xy && st->frozen_m) {   // final_comm_key = sum_j w[j] B[j]
    MsmSmallProblem<C> pr{(const Affine<C> *)st->d_key, st->d_w, nullptr, nullptr, (uint32_t)st->frozen_m};
    host::HXYZZ<C> k;
    if ((rc = msm_small_to_host<C>(ctx, &pr, 1, true, &k))) return rc;
    uint8_t inf = 0;
    host::to_affine<C>(k, out_final_key_xy, &inf);
  } else if (out_final_key_xy && (rc = rt::copy_d2h(out_final_key_xy, st->d_key, sizeof(Affine<C>), s))) return rc;
  if (out_c && (rc = rt::copy_d2h(out_c, st->d_coeffs, 32, s))) return rc;
  return rt::stream_sync(s);
}

template <class C>
int ipa_check_final_key_impl(pcgpu_ctx *ctx, const pcgpu_srs *key, const void *challenges, uint32_t log_d, void *out_xy,
                             uint8_t *out_inf) {
  using R = typename C::Fr;
  if (log_d > 26) return PCGPU_E_BADARG;
  size_t n = (size_t)1 << log_d;
  if (n > key->n) return PCGPU_E_LEN;
  rt::stream_t st = ctx->stream;
  int rc;
  const uint32_t *d_ch; uint32_t *d_co;
  Staging io(ctx, 0);
  io.host_in(d_ch, challenges, (size_t)log_d * 32);
  io.scratch(d_co, n * 32);
  if ((rc = io.upload())) return rc;
  if ((rc = rt::launch<256>(FrCheckCoeffsBody<R>{d_ch, log_d, d_co}, n, st))) return rc;
  host::HXYZZ<C> r;
  if ((rc = msm_to_host<C>(ctx, key, 0, d_co, n, true, &r))) return rc;
  host::to_affine<C>(r, out_xy, out_inf);
  return PCGPU_OK;
}

// ---------------------------------------------------------------------------------------------
// NTT
// ---------------------------------------------------------------------------------------------
// the context's twiddle tables for (curve, logn, direction), built on first use
template <class C>
static int ntt_plan(pcgpu_ctx *ctx, uint32_t logn, int inverse, const NttPlan **plan) {
  for (const NttPlan &p : ctx->ntt_plans)
    if (p.curve == C::ID && p.logn == logn && p.inverse == inverse) { *plan = &p; return PCGPU_OK; }
  NttPlan p;
  int rc = ntt_build_plan<typename C::Fr>(p, C::ID, logn, inverse, ctx->stream);
  if (rc) return rc;
  ctx->ntt_plans.push_back(p);
  *plan = &ctx->ntt_plans.back();
  return PCGPU_OK;
}

template <class C>
int ntt_impl(pcgpu_ctx *ctx, const void *in, size_t n_in, uint32_t logn, uint32_t flags, void *out) {
  using R = typename C::Fr;
  if (!ntt_supported(logn) || logn > (uint32_t)R::TWO_ADICITY) return PCGPU_E_BADARG;
  const size_t N = (size_t)1 << logn;
  if (n_in > N) return PCGPU_E_LEN;
  rt::stream_t st = ctx->stream;
  int rc, inverse = (flags & PCGPU_NTT_INVERSE) ? 1 : 0;
  const NttPlan *plan;
  if ((rc = ntt_plan<C>(ctx, logn, inverse, &plan))) return rc;
  uint32_t *tmp, *d_out; const uint32_t *d_in;
  Staging io(ctx, flags);
  io.scratch(tmp, N * 32);
  io.in(d_in, in, n_in * 32);
  io.out(d_out, out, N * 32);
  if ((rc = io.upload())) return rc;
  ctx->prof.begin(9, st);
  if ((rc = ntt_run<R>(*plan, d_in, n_in, d_out, tmp, st))) return rc;
  ctx->prof.end(9, st);
  if ((rc = io.download())) return rc;
  rc = rt::stream_sync(st);
  ctx->prof.collect();
  return rc;
}

template <class C>
int ntt_pass1_peer_impl(pcgpu_ctx *ctx, uint32_t logn, uint32_t flags, size_t lo, size_t count, const void *in, size_t n_in,
                        void *const *dst, uint32_t world) {
  using R = typename C::Fr;
  if (!ntt_supported(logn) || logn > (uint32_t)R::TWO_ADICITY || world == 0 || world > NTT_MAX_PEERS) return PCGPU_E_BADARG;
  uint32_t m1, m2;
  ntt_split(logn, &m1, &m2);
  if (m2 == 0 || (((size_t)1 << m1) % world) != 0) return PCGPU_E_BADARG;
  const size_t N2 = (size_t)1 << m2;
  if (lo > N2 || count > N2 - lo) return PCGPU_E_LEN;
  for (uint32_t d = 0; d < world; d++) if (!dst[d]) return PCGPU_E_BADARG;
  rt::stream_t st = ctx->stream;
  int rc, inverse = (flags & PCGPU_NTT_INVERSE) ? 1 : 0;
  const NttPlan *plan;
  if ((rc = ntt_plan<C>(ctx, logn, inverse, &plan))) return rc;
  if (count && (rc = ntt_run_pass1_peer<R>(*plan, lo, count, (const uint32_t *)in, n_in, (uint32_t *const *)dst, world, st))) return rc;
  return rt::stream_sync(st);
}

template <class C>
int ntt_batch_impl(pcgpu_ctx *ctx, const void *in, size_t n_in, size_t count, uint32_t logn, uint32_t flags, void *out) {
  using R = typename C::Fr;
  if (!ntt_supported(logn) || logn > (uint32_t)R::TWO_ADICITY) return PCGPU_E_BADARG;
  const size_t N = (size_t)1 << logn;
  if (n_in > N) return PCGPU_E_LEN;
  if (count == 0) return PCGPU_OK;
  if (count > ((size_t)1 << 40) / N) return PCGPU_E_BADARG;
  rt::stream_t st = ctx->stream;
  int rc, inverse = (flags & PCGPU_NTT_INVERSE) ? 1 : 0;
  const NttPlan *plan;
  if ((rc = ntt_plan<C>(ctx, logn, inverse, &plan))) return rc;
  uint32_t *tmp, *tmp_rows = nullptr, *d_out; const uint32_t *d_in;
  Staging io(ctx, flags);
  io.scratch(tmp, N * 32);
  if (plan->m2) io.scratch(tmp_rows, count * N * 32);   // rows longer than one block pass: scratch for all rows so both passes are single launches
  io.in(d_in, in, count * n_in * 32);
  io.out(d_out, out, count * N * 32);
  if ((rc = io.upload())) return rc;
  ctx->prof.begin(9, st);
  if ((rc = ntt_run_batch<R>(*plan, d_in, n_in, count, d_out, tmp, st, tmp_rows))) return rc;
  ctx->prof.end(9, st);
  if ((rc = io.download())) return rc;
  rc = rt::stream_sync(st);
  ctx->prof.collect();
  return rc;
}

template <class C>
int ntt_pass_impl(pcgpu_ctx *ctx, uint32_t logn, uint32_t flags, int which, size_t lo, size_t count, const void *in, size_t n_in,
                  void *out) {
  using R = typename C::Fr;
  if (!ntt_supported(logn) || logn > (uint32_t)R::TWO_ADICITY || (which != 1 && which != 2)) return PCGPU_E_BADARG;
  uint32_t m1, m2;
  ntt_split(logn, &m1, &m2);
  if (m2 == 0) return PCGPU_E_BADARG;
  const size_t lim = which == 1 ? ((size_t)1 << m2) : ((size_t)1 << m1);
  if (lo > lim || count > lim - lo) return PCGPU_E_LEN;
  rt::stream_t st = ctx->stream;
  int rc, inverse = (flags & PCGPU_NTT_INVERSE) ? 1 : 0;
  const NttPlan *plan;
  if ((rc = ntt_plan<C>(ctx, logn, inverse, &plan))) return rc;
  if (count && (rc = ntt_run_pass<R>(*plan, which, lo, count, (const uint32_t *)in, n_in, (uint32_t *)out, st))) return rc;
  return rt::stream_sync(st);
}

// ---------------------------------------------------------------------------------------------
// linear-code commitments: column hashes + Merkle tree (hash.cuh), fused behind the row encoding
// ---------------------------------------------------------------------------------------------
static inline uint64_t next_pow2_u64(uint64_t v) { uint64_t p = 1; while (p < v) p <<= 1; return p; }

template <class C>
static int hash_columns_device(const uint32_t *d_mat, size_t n_rows, size_t n_cols, int hash, bool mont, uint32_t *d_leaves, rt::stream_t st) {
  using R = typename C::Fr;
  if (hash == HASH_BLAKE2S) return rt::launch<64>(ColumnHashBody<R, Blake2s>{d_mat, n_rows, n_cols, d_leaves, mont ? 1 : 0}, n_cols, st);
  if (hash == HASH_SHA256) return rt::launch<64>(ColumnHashBody<R, Sha256>{d_mat, n_rows, n_cols, d_leaves, mont ? 1 : 0}, n_cols, st);
  return PCGPU_E_BADARG;
}

template <class C>
int lincode_hash_columns_impl(pcgpu_ctx *ctx, const void *mat, size_t n_rows, size_t n_cols, int hash, uint32_t flags, uint8_t *out_leaves) {
  rt::stream_t st = ctx->stream;
  int rc;
  if (n_cols == 0) return PCGPU_OK;
  const uint32_t *d_m; uint32_t *d_l;
  Staging io(ctx, flags);
  io.in(d_m, mat, n_rows * n_cols * 32);
  io.out(d_l, out_leaves, n_cols * 32);
  if ((rc = io.upload())) return rc;
  if ((rc = hash_columns_device<C>(d_m, n_rows, n_cols, hash, true, d_l, st))) return rc;
  if ((rc = io.download())) return rc;
  return rt::stream_sync(st);
}

inline int merkle_tree_impl(pcgpu_ctx *ctx, const uint8_t *leaves, size_t n_leaves, uint32_t flags, uint8_t *out_nodes, uint8_t *out_root) {
  rt::stream_t st = ctx->stream;
  if (n_leaves < 2) return PCGPU_E_BADARG;          // ark-crypto-primitives' MerkleTree::new needs at least two leaves
  const uint64_t P = next_pow2_u64(n_leaves);
  int rc;
  uint32_t *d_nodes; const uint32_t *d_leaves;
  Staging io(ctx, flags);
  io.out(d_nodes, out_nodes, (P - 1) * 32);
  io.in(d_leaves, leaves, n_leaves * 32);
  if ((rc = io.upload())) return rc;
  if ((rc = merkle_build(d_leaves, n_leaves, P, d_nodes, st))) return rc;
  if ((rc = io.download())) return rc;
  if (out_root && (rc = rt::copy_d2h(out_root, d_nodes, 32, st))) return rc;
  return rt::stream_sync(st);
}

// compute_matrices' row encoding + column hashes + Merkle tree without leaving the device (linear_codes/mod.rs:247-275)
template <class C>
int lincode_commit_impl(pcgpu_ctx *ctx, const void *mat, size_t n_rows, size_t n_cols, uint32_t log_ext, int hash, uint32_t flags,
                        void *out_ext, uint8_t *out_leaves, uint8_t *out_nodes, uint8_t *out_root) {
  using R = typename C::Fr;
  if (!ntt_supported(log_ext) || log_ext > (uint32_t)R::TWO_ADICITY) return PCGPU_E_BADARG;
  const size_t N = (size_t)1 << log_ext;
  if (n_cols > N) return PCGPU_E_LEN;
  if (N < 2 || n_rows == 0) return PCGPU_E_BADARG;
  if (n_rows > ((size_t)1 << 40) / N) return PCGPU_E_BADARG;
  rt::stream_t st = ctx->stream;
  int rc;
  const NttPlan *plan;
  if ((rc = ntt_plan<C>(ctx, log_ext, 0, &plan))) return rc;
  const uint64_t P = N;   // the extended width is a power of two already
  uint32_t *tmp, *tmp_rows = nullptr, *d_ext, *d_leaves, *d_nodes; const uint32_t *d_in;
  Staging io(ctx, flags);
  io.scratch(tmp, N * 32);
  if (plan->m2) io.scratch(tmp_rows, n_rows * N * 32);
  io.out(d_ext, out_ext, n_rows * N * 32);
  io.out(d_leaves, out_leaves, N * 32);
  io.out(d_nodes, out_nodes, (P - 1) * 32);
  io.in(d_in, mat, n_rows * n_cols * 32);
  if ((rc = io.upload())) return rc;
  ctx->prof.begin(9, st);
  if ((rc = ntt_run_batch<R>(*plan, d_in, n_cols, n_rows, d_ext, tmp, st, tmp_rows))) return rc;
  ctx->prof.end(9, st);
  ctx->prof.begin(14, st);
  if ((rc = hash_columns_device<C>(d_ext, n_rows, N, hash, true, d_leaves, st))) return rc;
  if ((rc = merkle_build(d_leaves, N, P, d_nodes, st))) return rc;
  ctx->prof.end(14, st);
  if ((rc = io.download())) return rc;
  if (out_root && (rc = rt::copy_d2h(out_root, d_nodes, 32, st))) return rc;
  rc = rt::stream_sync(st);
  ctx->prof.collect();
  return rc;
}

// ---------------------------------------------------------------------------------------------
// Brakedown: the sparse row encoding (sprs.cuh) in front of the same column hashes + tree
// ---------------------------------------------------------------------------------------------
// BrakedownPCParams' code (linear_codes/brakedown.rs:146-203) on the device.  start / end as brakedown.rs:168-181; the
// Reed-Solomon bounds as multilinear_brakedown/mod.rs:71-73 (with the unwrap_or defaults when there are no levels).
struct pcgpu_brakedown {
  int curve;
  uint64_t m, m_ext, levels;
  std::vector<uint64_t> a_dims, b_dims, start, end;   // 3L, 3L, L, L
  uint64_t rss, rsie, rsoe;
  uint32_t *d_mem;                                    // every matrix: ind_ptr | col_ind | val, one allocation
  std::vector<SprsLevel> a_lev, b_lev;
};

template <class R>
static bool fr_words_reduced(const uint32_t *w) {
  for (int i = R::N - 1; i >= 0; i--)
    if (w[i] != R::mod(i)) return w[i] < R::mod(i);
  return false;
}

// Checks one SprsMat (n rows, m columns, at most nnz_cap nonzeros) and packs the nonzeros whose row index is < lim as
// 32-bit offsets / indices + Montgomery words.  BADARG: ind_ptr not starting at 0, not monotone, past nnz_cap or 2^32;
// col_ind >= n.  RANGE: a value that is not a reduced field element.
template <class R>
static int sprs_pack(uint64_t n, uint64_t m, uint64_t nnz_cap, const uint64_t *ind_ptr, const uint64_t *col_ind, const void *val,
                     uint64_t lim, std::vector<uint32_t> &ptr, std::vector<uint32_t> &col, std::vector<uint32_t> &vals) {
  if (!ind_ptr || ind_ptr[0] != 0) return PCGPU_E_BADARG;
  for (uint64_t j = 0; j < m; j++)
    if (ind_ptr[j + 1] < ind_ptr[j]) return PCGPU_E_BADARG;
  const uint64_t nnz = ind_ptr[m];
  if (nnz > nnz_cap || nnz >= ((uint64_t)1 << 32)) return PCGPU_E_BADARG;
  if (nnz && (!col_ind || !val)) return PCGPU_E_BADARG;
  const uint32_t *w = (const uint32_t *)val;
  for (uint64_t k = 0; k < nnz; k++) {
    if (col_ind[k] >= n) return PCGPU_E_BADARG;
    if (!fr_words_reduced<R>(w + 8 * k)) return PCGPU_E_RANGE;
  }
  ptr.assign(m + 1, 0);
  col.clear(); vals.clear();
  for (uint64_t j = 0; j < m; j++) {
    for (uint64_t k = ind_ptr[j]; k < ind_ptr[j + 1]; k++) {
      if (col_ind[k] >= lim) continue;
      col.push_back((uint32_t)col_ind[k]);
      vals.insert(vals.end(), w + 8 * k, w + 8 * k + 8);
    }
    ptr[j + 1] = (uint32_t)col.size();
  }
  return PCGPU_OK;
}

template <class C>
int brakedown_register_impl(pcgpu_ctx *ctx, uint64_t m, uint64_t m_ext, uint64_t L, const uint64_t *a_dims, const uint64_t *b_dims,
                            const uint64_t *const *ind_ptr, const uint64_t *const *col_ind, const void *const *val, pcgpu_brakedown *bd) {
  using R = typename C::Fr;
  if (m == 0 || L > SPRS_MAX_LEVELS || (L && (!a_dims || !b_dims || !ind_ptr || !col_ind || !val))) return PCGPU_E_BADARG;
  bd->curve = C::ID; bd->m = m; bd->m_ext = m_ext; bd->levels = L;
  bd->a_dims.assign(a_dims, a_dims + 3 * L); bd->b_dims.assign(b_dims, b_dims + 3 * L);
  // shapes: A_0 reads the message, A_i reads what A_{i-1} wrote, B_i reads [start[i], end[i]), m_ext = codeword_len
  // (brakedown.rs:292-299; without levels the caller's ceil_mul(m, rho_inv), which only has to hold the message)
  if (L) {
    if (a_dims[0] != m) return PCGPU_E_BADARG;
    uint64_t s = 0, cw = 0;
    for (uint64_t i = 0; i < L; i++) {
      if (i + 1 < L && a_dims[3 * i + 1] != a_dims[3 * (i + 1)]) return PCGPU_E_BADARG;
      if (a_dims[3 * i + 1] == 0 || b_dims[3 * i] == 0) return PCGPU_E_BADARG;
      s += a_dims[3 * i]; cw += a_dims[3 * i] + b_dims[3 * i + 1];
      bd->start.push_back(s);
    }
    cw += b_dims[3 * (L - 1)];
    if (m_ext != cw) return PCGPU_E_BADARG;
    uint64_t e = m_ext;
    for (uint64_t i = 0; i < L; i++) {
      e -= b_dims[3 * i + 1];
      bd->end.push_back(e);
      if (e < bd->start[i] || b_dims[3 * i] != e - bd->start[i]) return PCGPU_E_BADARG;
    }
    bd->rss = bd->start.back(); bd->rsie = bd->rss + a_dims[3 * (L - 1) + 1]; bd->rsoe = bd->end.back();
  } else {
    if (m_ext < m) return PCGPU_E_BADARG;
    bd->rss = 0; bd->rsie = m; bd->rsoe = m_ext;
  }
  if (bd->rsoe < bd->rsie) return PCGPU_E_BADARG;   // the Reed-Solomon step must have room for its input
  // pack: A_0..A_{L-1}, B_0..B_{L-1}.  B_i's nonzeros at rows >= rsoe - start[i] read the deeper levels' outputs, which are
  // still zero when B_i runs (the ascending loop of mod.rs:77-80), so they are dropped here.
  std::vector<std::vector<uint32_t>> P(2 * L), Cc(2 * L), V(2 * L);
  for (uint64_t q = 0; q < 2 * L; q++) {
    const uint64_t i = q % L;
    const uint64_t *d = q < L ? a_dims + 3 * i : b_dims + 3 * i;
    const uint64_t lim = q < L ? d[0] : bd->rsoe - bd->start[i];
    const uint64_t cap = (d[2] && d[0] > UINT64_MAX / d[2]) ? UINT64_MAX : d[0] * d[2];
    int rc = sprs_pack<R>(d[0], d[1], cap, ind_ptr[q], col_ind[q], val[q], lim, P[q], Cc[q], V[q]);
    if (rc) return rc;
  }
  size_t words = 0;
  for (uint64_t q = 0; q < 2 * L; q++) words += P[q].size() + Cc[q].size() + V[q].size() + 8;   // +8: keep 32-byte alignment
  int rc = rt::dev_malloc((void **)&bd->d_mem, words * 4 + 64);
  if (rc) return rc;
  rt::stream_t st = ctx->stream;
  uint32_t *p = bd->d_mem;
  uint64_t b_first = 0;
  for (uint64_t q = 0; q < 2 * L; q++) {
    const uint64_t i = q % L;
    SprsLevel lv;
    uint32_t *dv = p;                     // values first: 32-byte aligned loads
    if (!V[q].empty() && (rc = rt::copy_h2d(dv, V[q].data(), V[q].size() * 4, st))) return rc;
    p += V[q].size();
    uint32_t *dp = p;
    if ((rc = rt::copy_h2d(dp, P[q].data(), P[q].size() * 4, st))) return rc;
    p += P[q].size();
    uint32_t *dc = p;
    if (!Cc[q].empty() && (rc = rt::copy_h2d(dc, Cc[q].data(), Cc[q].size() * 4, st))) return rc;
    p += Cc[q].size();
    p += (8 - (size_t)(p - bd->d_mem) % 8) % 8;
    lv.ind_ptr = dp; lv.col_ind = dc; lv.val = dv;
    if (q < L) {
      lv.in_base = bd->start[i] - a_dims[3 * i]; lv.out_base = bd->start[i]; lv.cols = a_dims[3 * i + 1]; lv.first = 0;
      bd->a_lev.push_back(lv);
    } else {
      lv.in_base = bd->start[i]; lv.out_base = bd->end[i]; lv.cols = b_dims[3 * i + 1];
      bd->b_lev.push_back(lv);
    }
  }
  // the B launch enumerates its output columns from the deepest level (lowest positions) up
  std::sort(bd->b_lev.begin(), bd->b_lev.end(), [](const SprsLevel &x, const SprsLevel &y) { return x.out_base < y.out_base; });
  for (SprsLevel &lv : bd->b_lev) { lv.first = b_first; b_first += lv.cols; }
  return rt::stream_sync(st);
}

// encode every row of d_in (n_rows x m, row-major) into d_out (n_rows x m_ext, row-major).
//   work: rsoe * n_rows elements, element-major; rs: (rsie - rss) * n_rows elements
template <class C>
static int brakedown_encode_device(const pcgpu_brakedown *bd, const uint32_t *d_in, uint64_t n_rows, uint32_t *work, uint32_t *rs,
                                   uint32_t *d_out, rt::stream_t st) {
  using R = typename C::Fr;
  const uint64_t n = n_rows, m_ext = bd->m_ext;
  int rc;
  // cw = msg
  if ((rc = rt::launch<128>(FrStridedCopyBody{d_in, 1, bd->m, work, n, 1, n}, bd->m * n, st))) return rc;
  // A levels, each on what the previous one appended
  for (const SprsLevel &lv : bd->a_lev) {
    SprsRowMulBody<R> b{};
    b.lev[0] = lv; b.nlev = 1;
    b.src = work; b.src_es = n; b.src_rs = 1; b.dst = work; b.dst_es = n; b.dst_rs = 1; b.n_rows = n;
    if ((rc = rt::launch<128>(b, lv.cols * n, st))) return rc;
  }
  // Reed-Solomon in place over cw[rss..rsoe]: its input cw[rss..rsie] is copied aside first
  const uint64_t n_in = bd->rsie - bd->rss;
  if ((rc = rt::copy_d2d(rs, work + bd->rss * n * 8, n_in * n * 32, st))) return rc;
  if ((rc = rt::launch<128>(NaiveRsBody<R>{rs, n_in, work, bd->rss, n}, (bd->rsoe - bd->rss) * n, st))) return rc;
  // every B level against the buffer as it stands now, straight into the row-major output
  if (!bd->b_lev.empty()) {
    SprsRowMulBody<R> b{};
    for (size_t i = 0; i < bd->b_lev.size(); i++) b.lev[i] = bd->b_lev[i];
    b.nlev = (uint32_t)bd->b_lev.size();
    b.src = work; b.src_es = n; b.src_rs = 1; b.dst = d_out; b.dst_es = 1; b.dst_rs = m_ext; b.n_rows = n;
    if ((rc = rt::launch<128>(b, (m_ext - bd->rsoe) * n, st))) return rc;
  }
  // cw[0..rsoe] to the row-major output
  return rt::launch<128>(FrStridedCopyBody{work, n, 1, d_out, 1, m_ext, n}, bd->rsoe * n, st);
}

// MultilinearBrakedown::encode over n_rows rows (compute_matrices, linear_codes/mod.rs:118-138) and, when `hash` >= 0, the
// column hashes and the tree of LinearCodePCS::commit (mod.rs:253-275)
template <class C>
int brakedown_commit_impl(pcgpu_ctx *ctx, const pcgpu_brakedown *bd, const void *mat, size_t n_rows, size_t n_cols, int hash,
                          uint32_t flags, void *out_ext, uint8_t *out_leaves, uint8_t *out_nodes, uint8_t *out_root) {
  if (n_cols != bd->m) return PCGPU_E_LEN;                   // Error::EncodingError
  if (n_rows == 0 || n_rows > ((size_t)1 << 40) / bd->m_ext) return PCGPU_E_BADARG;
  const bool tree = hash >= 0;
  if (tree && (hash > HASH_SHA256 || bd->m_ext < 2)) return PCGPU_E_BADARG;
  rt::stream_t st = ctx->stream;
  const uint64_t N = bd->m_ext, P = next_pow2_u64(N);
  int rc;
  // work: rsoe * n_rows elements, element-major; rs: (rsie - rss) * n_rows elements (brakedown_encode_device)
  uint32_t *work, *rs, *d_ext, *d_leaves = nullptr, *d_nodes = nullptr; const uint32_t *d_in;
  Staging io(ctx, flags);
  io.scratch(work, bd->rsoe * n_rows * 32);
  io.scratch(rs, (bd->rsie - bd->rss) * n_rows * 32);
  io.out(d_ext, out_ext, n_rows * N * 32);
  if (tree) {
    io.out(d_leaves, out_leaves, N * 32);
    io.out(d_nodes, out_nodes, (P - 1) * 32);
  }
  io.in(d_in, mat, n_rows * n_cols * 32);
  if ((rc = io.upload())) return rc;
  ctx->prof.begin(15, st);
  if ((rc = brakedown_encode_device<C>(bd, d_in, n_rows, work, rs, d_ext, st))) return rc;
  ctx->prof.end(15, st);
  if (tree) {
    ctx->prof.begin(14, st);
    if ((rc = hash_columns_device<C>(d_ext, n_rows, N, hash, true, d_leaves, st))) return rc;
    if ((rc = merkle_build(d_leaves, N, P, d_nodes, st))) return rc;
    ctx->prof.end(14, st);
  }
  if ((rc = io.download())) return rc;
  if (tree && out_root && (rc = rt::copy_d2h(out_root, d_nodes, 32, st))) return rc;
  rc = rt::stream_sync(st);
  ctx->prof.collect();
  return rc;
}

// SprsMat::row_mul on `count` vectors (count x n, row-major) -> count x m.  The matrix is host data (checked, then staged);
// with PCGPU_DEVICE_PTRS v and out are device pointers.
template <class C>
int fr_sprs_row_mul_impl(pcgpu_ctx *ctx, size_t n, size_t m, const uint64_t *ind_ptr, const uint64_t *col_ind, const void *val,
                         const void *v, size_t count, uint32_t flags, void *out) {
  using R = typename C::Fr;
  std::vector<uint32_t> P, Cc, V;
  int rc;
  if ((rc = sprs_pack<R>(n, m, UINT64_MAX, ind_ptr, col_ind, val, n, P, Cc, V))) return rc;
  if (m == 0 || count == 0) return PCGPU_OK;
  rt::stream_t st = ctx->stream;
  const uint32_t *dv, *dp, *dc, *d_v; uint32_t *d_o;
  Staging io(ctx, flags);
  io.host_in(dv, V.data(), V.size() * 4);
  io.host_in(dp, P.data(), P.size() * 4);
  io.host_in(dc, Cc.data(), Cc.size() * 4);
  io.in(d_v, v, count * n * 32);
  io.out(d_o, out, count * m * 32);
  if ((rc = io.upload())) return rc;
  SprsRowMulBody<R> b{};
  b.lev[0] = SprsLevel{dp, dc, dv, 0, 0, m, 0}; b.nlev = 1;
  b.src = d_v; b.src_es = 1; b.src_rs = n; b.dst = d_o; b.dst_es = 1; b.dst_rs = m; b.n_rows = count;
  if ((rc = rt::launch<128>(b, m * count, st))) return rc;
  if ((rc = io.download())) return rc;
  return rt::stream_sync(st);
}

// ---------------------------------------------------------------------------------------------
// G1 wire formats (wire.cuh)
// ---------------------------------------------------------------------------------------------
template <class C>
int g1_serialize_impl(pcgpu_ctx *ctx, const void *xy, const uint8_t *inf, size_t n, uint32_t flags, uint8_t *out) {
  constexpr size_t PT = 2 * C::Fq::N * 4;
  rt::stream_t st = ctx->stream;
  const int comp = (flags & PCGPU_WIRE_COMPRESSED) ? 1 : 0;
  const size_t sz = wire_size<C>(comp != 0);
  int rc;
  if (n == 0) return PCGPU_OK;
  const uint32_t *d_xy; const uint8_t *d_inf = nullptr; uint8_t *d_out;
  Staging io(ctx, flags);
  io.in(d_xy, xy, n * PT);
  if (inf) io.in(d_inf, inf, n);
  io.out(d_out, out, n * sz);
  if ((rc = io.upload())) return rc;
  if ((rc = rt::launch<128>(G1EncodeBody<C>{d_xy, d_inf, d_out, comp}, n, st))) return rc;
  if ((rc = io.download())) return rc;
  return rt::stream_sync(st);
}

template <class C>
int g1_deserialize_impl(pcgpu_ctx *ctx, const uint8_t *bytes, size_t n, uint32_t flags, void *out_xy, uint8_t *out_inf,
                        size_t *first_bad, int *reason) {
  constexpr size_t PT = 2 * C::Fq::N * 4;
  rt::stream_t st = ctx->stream;
  const int comp = (flags & PCGPU_WIRE_COMPRESSED) ? 1 : 0, validate = (flags & PCGPU_WIRE_NO_VALIDATE) ? 0 : 1;
  const size_t sz = wire_size<C>(comp != 0);
  int rc;
  if (n == 0) return PCGPU_OK;
  uint8_t *d_status, *d_inf; const uint8_t *d_bytes; uint32_t *d_xy;
  Staging io(ctx, flags);
  io.scratch(d_status, n);
  io.in(d_bytes, bytes, n * sz);
  io.out(d_xy, out_xy, n * PT);
  io.out(d_inf, out_inf, n);
  if ((rc = io.upload())) return rc;
  if ((rc = rt::launch<128>(G1DecodeBody<C>{d_bytes, d_xy, d_inf, d_status, comp, validate}, n, st))) return rc;
  std::vector<uint8_t> status(n);
  if ((rc = rt::copy_d2h(status.data(), d_status, n, st))) return rc;
  if ((rc = io.download())) return rc;
  if ((rc = rt::stream_sync(st))) return rc;
  for (size_t i = 0; i < n; i++)
    if (status[i]) {
      if (first_bad) *first_bad = i;
      if (reason) *reason = status[i];
      return PCGPU_E_INVALID;
    }
  return PCGPU_OK;
}

template <class C>
int g1_sample_generators_impl(pcgpu_ctx *ctx, const uint8_t *name, size_t name_len, uint64_t first, size_t n, uint32_t flags, void *out_xy) {
  constexpr size_t PT = 2 * C::Fq::N * 4;
  if (name_len > SAMPLE_NAME_MAX) return PCGPU_E_BADARG;
  if (n == 0) return PCGPU_OK;
  rt::stream_t st = ctx->stream;
  int rc;
  SampleGeneratorsBody<C> b;
  memset(&b, 0, sizeof b);
  memcpy(b.name, name, name_len);
  b.name_len = (uint32_t)name_len; b.first = first;
  Staging io(ctx, flags);
  io.out(b.out_xy, out_xy, n * PT);
  if ((rc = io.upload())) return rc;
  if ((rc = rt::launch<128>(b, n, st))) return rc;
  if ((rc = io.download())) return rc;
  return rt::stream_sync(st);
}

// ---------------------------------------------------------------------------------------------
// device self-test of the field layer
// ---------------------------------------------------------------------------------------------
template <class P>
struct FieldSelfTestBody {
  uint64_t seed; uint32_t *bad;
  static PCGPU_DEV uint64_t mix(uint64_t x) {  // splitmix64
    x += 0x9e3779b97f4a7c15ull; x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull; x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
    return x ^ (x >> 31);
  }
  PCGPU_KERNEL_DEV void operator()(size_t i) const {
    Fp<P> a, b;
    uint64_t s = seed + 0x1000003ull * i;
    for (int j = 0; j < P::N; j += 2) {
      s = mix(s); a.l[j] = (uint32_t)s; a.l[j + 1] = (uint32_t)(s >> 32);
      s = mix(s); b.l[j] = (uint32_t)s; b.l[j + 1] = (uint32_t)(s >> 32);
    }
    // force the operands below p: clear the top bits, then one conditional subtraction
    const uint32_t topmask = (P::BITS % 32) ? ((1u << (P::BITS % 32)) - 1) : 0xffffffffu;
    a.l[P::N - 1] &= topmask; b.l[P::N - 1] &= topmask;
    fp_reduce_once<P>(a.l); fp_reduce_once<P>(b.l);
    if (i % 7 == 0) a = fp_neg<P>(Fp<P>::one());      // p - R
    if (i % 11 == 0) b = fp_sub<P>(Fp<P>::zero(), Fp<P>::one());
    Fp<P> x = mont_mul<P>(a, b), y = mont_mul_ref<P>(a, b);
    uint32_t wrong = (x != y) ? 1u : 0u;
    Fp<P> c = fp_sub<P>(fp_add<P>(a, b), b);
    wrong += (c != a) ? 1u : 0u;
    if (i < 64 && !a.is_zero()) {
      Fp<P> inv = fp_inv<P>(a);
      wrong += (mont_mul<P>(a, inv) != Fp<P>::one()) ? 1u : 0u;
    }
    if (wrong) rt::atomic_add(bad, wrong);
  }
};

// pcgpu_diag_field_op: FieldOpBody on the device, host operands staged through the context's arena
template <class C, class P>
static int diag_field_op_run(pcgpu_ctx *ctx, int op, const void *a, const void *b, void *out, size_t n) {
  rt::stream_t st = ctx->stream;
  const size_t bytes = n * P::N * 4;
  int rc;
  const bool fr_table = op == 8 && !std::is_same<P, typename C::Fq>::value;   // no kernel inverts in Fr by binary GCD
  const uint32_t *da, *db; uint32_t *dout, *t = nullptr;
  Staging io(ctx, 0);
  io.host_in(da, a, bytes);
  io.host_in(db, b, bytes);
  io.out(dout, out, bytes);
  if (fr_table) io.scratch(t, pow2_table_bytes<P>());   // a table for this call only
  if ((rc = io.upload())) return rc;
  const uint32_t *pow2 = nullptr;
  if (op == 8) {
    if (!fr_table) {                     // the table the pair rounds use
      if ((rc = ensure_pow2<C>(ctx))) return rc;
      pow2 = ctx->d_pow2[C::ID];
    } else {
      if ((rc = rt::launch<32>(Pow2TableBody<P>{t}, 1, st))) return rc;
      pow2 = t;
    }
  }
  if ((rc = rt::launch<128>(FieldOpBody<P>{da, db, dout, pow2, op}, n, st))) return rc;
  if ((rc = io.download())) return rc;
  return rt::stream_sync(st);
}

// which = 2: Fq2 of a pairing curve (C is its G2 group)
template <class C>
int diag_fq2_op_impl(pcgpu_ctx *ctx, int op, const void *a, const void *b, void *out, size_t n) {
  using P = typename C::Fq;
  if (op != 0 && op != 2 && op != 3 && op != 4 && op != 5 && op != 9) return PCGPU_E_BADARG;
  if (n == 0) return PCGPU_OK;
  rt::stream_t st = ctx->stream;
  const size_t bytes = n * Fq2<P>::WORDS * 4;
  int rc;
  const uint32_t *da, *db; uint32_t *dout;
  Staging io(ctx, 0);
  io.host_in(da, a, bytes);
  io.host_in(db, b, bytes);
  io.out(dout, out, bytes);
  if ((rc = io.upload())) return rc;
  if ((rc = rt::launch<128>(Fq2OpBody<P>{da, db, dout, op}, n, st))) return rc;
  if ((rc = io.download())) return rc;
  return rt::stream_sync(st);
}

template <class C>
int diag_field_op_impl(pcgpu_ctx *ctx, int which, int op, const void *a, const void *b, void *out, size_t n) {
  if (n == 0) return PCGPU_OK;
  return which == 0 ? diag_field_op_run<C, typename C::Fq>(ctx, op, a, b, out, n)
                    : diag_field_op_run<C, typename C::Fr>(ctx, op, a, b, out, n);
}

template <class C>
int selftest_field_impl(pcgpu_ctx *ctx, uint64_t seed, size_t n, uint64_t *mismatches) {
  rt::stream_t st = ctx->stream;
  int rc;
  uint32_t *d_bad = &ctx->d_words->selftest_bad;
  if ((rc = rt::dev_memset(d_bad, 0, sizeof *d_bad, st))) return rc;
  if ((rc = rt::launch<128>(FieldSelfTestBody<typename C::Fq>{seed, d_bad}, n, st))) return rc;
  if ((rc = rt::launch<128>(FieldSelfTestBody<typename C::Fr>{seed ^ 0x5555, d_bad}, n, st))) return rc;
  uint32_t h = 0;
  if ((rc = rt::copy_d2h(&h, d_bad, 4, st))) return rc;
  if ((rc = rt::stream_sync(st))) return rc;
  *mismatches = h;
  return PCGPU_OK;
}

// ---------------------------------------------------------------------------------------------
// IMAD.WIDE peak microbenchmark
// ---------------------------------------------------------------------------------------------
struct ImadPeakBody {
  uint64_t *sink; uint32_t iters;
  PCGPU_KERNEL_DEV void operator()(size_t t) const {
    uint32_t lo[8], hi[8];
#pragma unroll
    for (int j = 0; j < 8; j++) { lo[j] = (uint32_t)t * 8u + j + 1u; hi[j] = (uint32_t)t ^ (0x9e3779b9u * (j + 1)); }
    const uint32_t y = (uint32_t)t | 0x80000001u;
    for (uint32_t i = 0; i < iters; i++) {
#pragma unroll
      for (int j = 0; j < 8; j++) {
        // (hi:lo)[j] += hi[j+3] * y -- the same mad.lo.cc / madc.hi pair the field multiplier is made of; ptxas fuses each
        // pair into one IMAD.WIDE.U32 with 64-bit accumulate.  8 independent chains per thread.
        uint32_t x = hi[(j + 3) & 7];
        lo[j] = mad_lo_cc(x, y, lo[j]);
        hi[j] = madc_hi(x, y, hi[j]);
      }
    }
    uint64_t acc = 0;
#pragma unroll
    for (int j = 0; j < 8; j++) acc ^= ((uint64_t)hi[j] << 32) | lo[j];
    sink[t] = acc;
  }
};

inline int measure_imad_peak_impl(pcgpu_ctx *ctx, double *ops_per_s) {
#ifdef PCGPU_EMUL
  (void)ctx; *ops_per_s = 0; return PCGPU_OK;
#else
  rt::stream_t st = ctx->stream;
  int rc;
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
    return PCGPU_E_CUDA;
  const size_t threads = (size_t)sms * 2048;   // full occupancy: 2048 resident threads per SM
  const uint32_t iters = 4096;
  uint64_t *sink;
  Staging io(ctx, 0);
  io.scratch(sink, threads * 8);
  if ((rc = io.upload())) return rc;
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  if ((rc = rt::launch<256>(ImadPeakBody{sink, 64}, threads, st))) return rc;   // warm-up
  cudaEventRecord(e0, st);
  if ((rc = rt::launch<256>(ImadPeakBody{sink, iters}, threads, st))) return rc;
  cudaEventRecord(e1, st);
  if ((rc = rt::stream_sync(st))) return rc;
  float ms = 0; cudaEventElapsedTime(&ms, e0, e1);
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  *ops_per_s = (double)threads * iters * 8.0 / (ms * 1e-3);
  return PCGPU_OK;
#endif
}

// Explicit instantiation lists, one per translation-unit group so that the heavy kernels of one curve compile in parallel
// (inst_unit.cu is built once per (curve, group); `EXT` = extern declares, empty defines).  The three msm_* helpers are
// instantiated in ONE group and only declared elsewhere, so the Pippenger kernels are compiled exactly once per curve.
#define PCGPU_INST_PIPE(C, EXT)                                                                                            \
  EXT template int msm_device_planes<C>(pcgpu_ctx *, const pcgpu_srs *, size_t, const uint32_t *, size_t, bool, MsmGeom *, \
                                        const XYZZ<C> **, size_t *, uint32_t **);                                          \
  EXT template int msm_to_host<C>(pcgpu_ctx *, const pcgpu_srs *, size_t, const uint32_t *, size_t, bool, host::HXYZZ<C> *); \
  EXT template int msm_issue<C>(pcgpu_ctx *, const pcgpu_srs *, size_t, const uint32_t *, size_t, bool, MsmPending<C> *);   \
  EXT template int msm_collect<C>(pcgpu_ctx *, MsmPending<C> *, host::HXYZZ<C> *);
#define PCGPU_INST_PAIR1(C, EXT)                                                                                           \
  EXT template int pcgpu::msm_pair_round_oneshot<C>(bool, const uint32_t *, const MsmGeom &, const uint32_t *, const Affine<C> *, uint32_t *, \
                                             const uint32_t *, uint32_t, uint32_t *, const uint32_t *, Affine<C> *, rt::stream_t);   \
  EXT template int pcgpu::msm_pair_oneshot_threads<C>(size_t *);
#define PCGPU_INST_ACC(C, EXT)                                                                                             \
  EXT template int pcgpu::msm_accumulate_launch<C>(const uint32_t *, const MsmGeom &, const uint32_t *, const uint32_t *, const uint32_t *, \
                                            const uint32_t *, XYZZ<C> *, uint32_t *, const Affine<C> *, rt::stream_t);
#define PCGPU_INST_REDUCE(C, EXT)                                                                                          \
  EXT template int pcgpu::msm_reduce_launch<C>(const MsmGeom &, const uint32_t *, const XYZZ<C> *, XYZZ<C> *, XYZZ<C> *, XYZZ<C> *,    \
                                        const uint32_t *, const uint32_t *, rt::stream_t);
#define PCGPU_INST_SMALL(C, EXT)                                                                                           \
  EXT template int msm_small_to_host<C>(pcgpu_ctx *, const MsmSmallProblem<C> *, uint32_t, bool, host::HXYZZ<C> *);
#define PCGPU_INST_SRS(C, EXT)                                                                                             \
  EXT template int srs_register_impl<C>(pcgpu_ctx *, const void *, const uint8_t *, size_t, uint32_t, pcgpu_srs *);        \
  EXT template int msm_impl<C>(pcgpu_ctx *, const pcgpu_srs *, size_t, const void *, size_t, uint32_t, void *, uint8_t *, void *); \
  EXT template int g1_sum_impl<C>(pcgpu_ctx *, const void *, size_t, void *, uint8_t *);                                   \
  EXT template int fixed_base_impl<C>(pcgpu_ctx *, const void *, const void *, size_t, uint32_t, void *);                  \
  EXT template int kzg_commit_impl<C>(pcgpu_ctx *, const pcgpu_srs *, const void *, size_t, const pcgpu_srs *, const void *, \
                                      size_t, uint32_t, void *, uint8_t *);                                                \
  EXT template int kzg_open_impl<C>(pcgpu_ctx *, const pcgpu_srs *, const void *, size_t, const void *, const pcgpu_srs *, \
                                    const void *, size_t, uint32_t, void *, uint8_t *, void *); \
  EXT template int msm_batch_impl<C>(pcgpu_ctx *, const pcgpu_srs *, const void *, size_t, size_t, uint32_t, void *, uint8_t *); \
  EXT template int kzg_commit_open_impl<C>(pcgpu_ctx *, pcgpu_ctx *, const pcgpu_srs *, const void *, size_t, const void *, uint32_t, void *, uint8_t *, void *, uint8_t *); \
  EXT template int msm_peer_impl<C>(pcgpu_ctx *, const pcgpu_srs *, size_t, const void *, size_t, uint32_t, void *const *, uint32_t, uint32_t, uint64_t, void *, uint8_t *);
#define PCGPU_INST_FR(C, EXT)                                                                                              \
  EXT template int fr_from_mont_impl<C>(pcgpu_ctx *, const void *, void *, size_t, uint32_t);                              \
  EXT template int fr_axpy_impl<C>(pcgpu_ctx *, void *, const void *, const void *, size_t, uint32_t);                     \
  EXT template int fr_div_impl<C>(pcgpu_ctx *, const void *, size_t, const void *, void *, void *, uint32_t);              \
  EXT template int fr_ip_impl<C>(pcgpu_ctx *, const void *, const void *, size_t, void *, uint32_t);                       \
  EXT template int fr_row_mul_impl<C>(pcgpu_ctx *, const void *, const void *, size_t, size_t, void *, uint32_t);          \
  EXT template int fr_mul_impl<C>(pcgpu_ctx *, const void *, const void *, void *, size_t, uint32_t); \
  EXT template int selftest_field_impl<C>(pcgpu_ctx *, uint64_t, size_t, uint64_t *); \
  EXT template int diag_field_op_impl<C>(pcgpu_ctx *, int, int, const void *, const void *, void *, size_t); \
  EXT template int ntt_impl<C>(pcgpu_ctx *, const void *, size_t, uint32_t, uint32_t, void *); \
  EXT template int ntt_pass_impl<C>(pcgpu_ctx *, uint32_t, uint32_t, int, size_t, size_t, const void *, size_t, void *); \
  EXT template int ntt_batch_impl<C>(pcgpu_ctx *, const void *, size_t, size_t, uint32_t, uint32_t, void *); \
  EXT template int ntt_pass1_peer_impl<C>(pcgpu_ctx *, uint32_t, uint32_t, size_t, size_t, const void *, size_t, void *const *, uint32_t); \
  EXT template int lincode_hash_columns_impl<C>(pcgpu_ctx *, const void *, size_t, size_t, int, uint32_t, uint8_t *); \
  EXT template int lincode_commit_impl<C>(pcgpu_ctx *, const void *, size_t, size_t, uint32_t, int, uint32_t, void *, uint8_t *, uint8_t *, uint8_t *); \
  EXT template int brakedown_register_impl<C>(pcgpu_ctx *, uint64_t, uint64_t, uint64_t, const uint64_t *, const uint64_t *, \
                                              const uint64_t *const *, const uint64_t *const *, const void *const *, pcgpu_brakedown *); \
  EXT template int brakedown_commit_impl<C>(pcgpu_ctx *, const pcgpu_brakedown *, const void *, size_t, size_t, int, uint32_t, void *, \
                                            uint8_t *, uint8_t *, uint8_t *); \
  EXT template int fr_sprs_row_mul_impl<C>(pcgpu_ctx *, size_t, size_t, const uint64_t *, const uint64_t *, const void *, const void *, \
                                           size_t, uint32_t, void *);
#define PCGPU_INST_IPA(C, EXT)                                                                                             \
  EXT template int ipa_begin_impl<C>(pcgpu_ctx *, const void *, size_t, const void *, size_t, const void *, uint32_t, pcgpu_ipa *); \
  EXT template int ipa_round_lr_impl<C>(pcgpu_ctx *, pcgpu_ctx *, pcgpu_ipa *, const void *, void *, uint8_t *, void *, uint8_t *); \
  EXT template int ipa_round_fold_impl<C>(pcgpu_ctx *, pcgpu_ipa *, const void *, const void *); \
  EXT template int ipa_finish_impl<C>(pcgpu_ctx *, pcgpu_ipa *, void *, void *); \
  EXT template int ipa_check_final_key_impl<C>(pcgpu_ctx *, const pcgpu_srs *, const void *, uint32_t, void *, uint8_t *); \
  EXT template int g1_serialize_impl<C>(pcgpu_ctx *, const void *, const uint8_t *, size_t, uint32_t, uint8_t *); \
  EXT template int g1_deserialize_impl<C>(pcgpu_ctx *, const uint8_t *, size_t, uint32_t, void *, uint8_t *, size_t *, int *); \
  EXT template int g1_sample_generators_impl<C>(pcgpu_ctx *, const uint8_t *, size_t, uint64_t, size_t, uint32_t, void *);
// G2 groups (inst_unit.cu groups 10-12, pairing curves only): the bucket pipeline's point kernels, the small MSM and the G2 entry
// points; the pair-round kernels are never instantiated for G2
#define PCGPU_INST_G2(C, EXT)                                                                                              \
  EXT template int srs_register_impl<C>(pcgpu_ctx *, const void *, const uint8_t *, size_t, uint32_t, pcgpu_srs *);        \
  EXT template int msm_impl<C>(pcgpu_ctx *, const pcgpu_srs *, size_t, const void *, size_t, uint32_t, void *, uint8_t *, void *); \
  EXT template int fixed_base_impl<C>(pcgpu_ctx *, const void *, const void *, size_t, uint32_t, void *);                  \
  EXT template int diag_fq2_op_impl<C>(pcgpu_ctx *, int, const void *, const void *, void *, size_t);                      \
  EXT template int mlpc_register_impl<C>(pcgpu_ctx *, uint32_t, const void *const *, const uint8_t *const *, uint32_t, pcgpu_mlpc *); \
  EXT template int mlpc_open_impl<C>(pcgpu_ctx *, const pcgpu_mlpc *, const void *, size_t, const void *, uint32_t, void *, uint8_t *, void *);
#define PCGPU_INSTANTIATE_G2(C, EXT) \
  PCGPU_INST_ACC(C, EXT) PCGPU_INST_REDUCE(C, EXT) PCGPU_INST_PIPE(C, EXT) PCGPU_INST_SMALL(C, EXT) PCGPU_INST_G2(C, EXT)
#define PCGPU_INSTANTIATE(C, EXT) \
  PCGPU_INST_PAIR1(C, EXT) PCGPU_INST_ACC(C, EXT) PCGPU_INST_REDUCE(C, EXT) \
  PCGPU_INST_PIPE(C, EXT) PCGPU_INST_SMALL(C, EXT) PCGPU_INST_SRS(C, EXT) PCGPU_INST_FR(C, EXT) PCGPU_INST_IPA(C, EXT)
