// C ABI entry points (include/pcgpu.h): argument checks, locking, curve dispatch.
// The per-curve template instantiations live in inst_*.cu so the three curves compile in parallel.
#include <thread>

#include "impl.cuh"

// Nothing unwinds across the C ABI: every entry point runs inside this guard (std::vector / std::thread / new can throw).
static int ensure_siblings(pcgpu_ctx *ctx, size_t count);

template <class F>
static int guarded(F f) {
  try { return f(); }
  catch (const std::bad_alloc &) { return PCGPU_E_OOM; }
  catch (...) { return PCGPU_E_CUDA; }
}

// An entry point on one context: BADARG for a null context or when the argument checks found `bad_args`, else f() under the
// context's mutex with its device current, inside the guard.
template <class F>
static int on_ctx(pcgpu_ctx *ctx, bool bad_args, F f) {
  return guarded([&]() -> int {
    if (!ctx || bad_args) return PCGPU_E_BADARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    SET_DEVICE(ctx);
    return f();
  });
}

// x || y of one affine point of the curve (Montgomery limbs)
static size_t affine_bytes(int curve) { return (curve == PCGPU_BLS12_381 ? 6 : 4) * 16; }

// the device memory a handle owns (an IPA state's lives in its context's arena)
static void free_device(pcgpu_srs *srs) { rt::dev_free(srs->d_tables); rt::dev_free(srs->d_folded); rt::dev_free(srs->d_comb); }
static void free_device(pcgpu_mlpc *key) { free_device(&key->key); }
static void free_device(pcgpu_brakedown *code) { rt::dev_free(code->d_mem); }
static void free_device(pcgpu_ipa *) {}
static void free_device(pcgpu_g2_prepared *q) { rt::dev_free(q->d_lines); }
static void free_device(pcgpu_hyrax *h) { rt::dev_free(h->d_block); }

// Every creating entry point: *out is cleared whenever out is non-null, then make(handle) fills a fresh handle under the
// context's lock.  *out receives the handle only when make succeeds; on failure its device memory is freed and it is deleted.
template <class H, class F>
static int create(pcgpu_ctx *ctx, bool bad_args, H **out, F make) {
  if (out) *out = nullptr;
  return on_ctx(ctx, bad_args || !out, [&]() -> int {
    H *h = new (std::nothrow) H();
    if (!h) return PCGPU_E_OOM;
    int rc = make(h);
    if (rc) { free_device(h); delete h; return rc; }
    *out = h;
    return PCGPU_OK;
  });
}

// Frees a handle whose device memory work queued on the context may still read: waits for its stream first (no context:
// frees at once).
template <class H>
static void release_after_stream(pcgpu_ctx *ctx, H *h) {
  if (!h) return;
  std::unique_lock<std::mutex> lk;
  if (ctx) {
    lk = std::unique_lock<std::mutex>(ctx->mu);
#ifndef PCGPU_EMUL
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
#endif
  }
  free_device(h);
  delete h;
}

PCGPU_INSTANTIATE(Bls12381, extern)
PCGPU_INSTANTIATE(Bn254, extern)
PCGPU_INSTANTIATE(Pallas, extern)
PCGPU_INSTANTIATE_G2(Bls12381G2, extern)
PCGPU_INSTANTIATE_G2(Bn254G2, extern)
PCGPU_INST_PAIRING(Bls12381, extern)
PCGPU_INST_PAIRING(Bn254, extern)

extern "C" const char *pcgpu_strerror(int code) {
  switch (code) {
    case PCGPU_OK: return "ok";
    case PCGPU_E_CUDA: return "CUDA failure or no usable sm_90 device";
    case PCGPU_E_OOM: return "device memory allocation failed";
    case PCGPU_E_BADARG: return "bad argument";
    case PCGPU_E_LEN: return "length out of range (base_offset + n exceeds the registered bases, or the input is longer than the transform / slice)";
    case PCGPU_E_RANGE: return "canonical scalar out of range (not a reduced field element)";
    case PCGPU_E_DEGREE: return "TooManyCoefficients: polynomial degree too large for the powers";
    case PCGPU_E_HIDING: return "HidingBoundToolarge: blinding polynomial too large for powers_of_gamma_g";
    case PCGPU_E_INVALID: return "SerializationError: wire-format element failed to decode or validate";
    case PCGPU_E_PEER: return "multi-GPU exchange failed: a peer did not signal in time, or sent a malformed record";
    default: return "unknown error";
  }
}

extern "C" int pcgpu_init(int device, pcgpu_ctx **out) {
  return guarded([&]() -> int {
  if (!out) return PCGPU_E_BADARG;
  *out = nullptr;
#ifndef PCGPU_EMUL
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || device < 0 || device >= count) return PCGPU_E_CUDA;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return PCGPU_E_CUDA;
  if (prop.major != 9 || prop.minor != 0) return PCGPU_E_CUDA;  // built for sm_90a only; no other code path exists
  if (cudaSetDevice(device) != cudaSuccess) return PCGPU_E_CUDA;
  // L2 fetch granularity hint: round 0 of the pair rounds gathers the 64-byte x halves of table records in pass 1 and whole
  // 128-byte records in pass 2 (DESIGN.md section 5); at the default granularity every pass-1 miss moves a 128-byte line.
  if (const char *e = getenv("PCGPU_L2_FETCH_GRANULARITY")) {
    int v = atoi(e);
    if (v == 32 || v == 64 || v == 128) cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, (size_t)v);
  }
#endif
  pcgpu_ctx *ctx = new (std::nothrow) pcgpu_ctx();
  if (!ctx) return PCGPU_E_OOM;
  ctx->device = device;
#ifndef PCGPU_EMUL
  if (cudaStreamCreateWithFlags(&ctx->own_stream, cudaStreamNonBlocking) != cudaSuccess) { delete ctx; return PCGPU_E_CUDA; }
#else
  ctx->own_stream = nullptr;
#endif
  ctx->stream = ctx->own_stream;
  int rc = rt::dev_malloc((void **)&ctx->d_words, sizeof(DeviceWords));
  if (rc) { delete ctx; return rc; }
  if ((rc = rt::host_alloc_pinned((void **)&ctx->h_pinned, sizeof(PinnedZone)))) { rt::dev_free(ctx->d_words); delete ctx; return rc; }
  *out = ctx;
  return PCGPU_OK;
  });
}

extern "C" void pcgpu_destroy(pcgpu_ctx *ctx) {
  if (!ctx) return;
#ifndef PCGPU_EMUL
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
#endif
  ctx->prof.destroy();
  for (pcgpu_ctx *s : ctx->siblings) pcgpu_destroy(s);
  for (NttPlan &p : ctx->ntt_plans) rt::dev_free(p.base);
  for (int k = 0; k < 3; k++) rt::dev_free(ctx->d_pow2[k]);
  ctx->msm_arena.release();
  ctx->stage.release();
  ctx->ipa_arena.release();
  rt::dev_free(ctx->d_words);
  rt::host_free_pinned(ctx->h_pinned);
  if (ctx->ev_ok) rt::event_destroy(ctx->ev_upload);
#ifndef PCGPU_EMUL
  cudaStreamDestroy(ctx->own_stream);
#endif
  delete ctx;
}

extern "C" int pcgpu_set_stream(pcgpu_ctx *ctx, void *cuda_stream) {
  return guarded([&]() -> int {
  if (!ctx) return PCGPU_E_BADARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  ctx->stream = cuda_stream ? (rt::stream_t)cuda_stream : ctx->own_stream;
  return PCGPU_OK;
  });
}

extern "C" int pcgpu_profile_enable(pcgpu_ctx *ctx, int enable) {
  return on_ctx(ctx, false, [&]() -> int {
    ctx->prof.collect();
    ctx->prof.on = enable != 0;
    if (enable) ctx->prof.reset();
    return PCGPU_OK;
  });
}

extern "C" int pcgpu_profile_get(pcgpu_ctx *ctx, int stage, double *ms, uint64_t *count) {
  return on_ctx(ctx, stage < 0 || stage >= PROF_STAGES, [&]() -> int {
    ctx->prof.collect();
    if (ms) *ms = ctx->prof.ms[stage];
    if (count) *count = ctx->prof.cnt[stage];
    return PCGPU_OK;
  });
}

extern "C" int pcgpu_srs_register(pcgpu_ctx *ctx, int curve, const void *bases_xy, const uint8_t *inf, size_t n,
                                  uint32_t flags, pcgpu_srs **out) {
  return create(ctx, (n && !bases_xy) || n >= (1u << 26), out, [&](pcgpu_srs *srs) -> int {
    srs->curve = curve; srs->n = n;
    DISPATCH_GROUP(curve, return srs_register_impl<C>(ctx, bases_xy, inf, n, flags, srs));
  });
}

extern "C" void pcgpu_srs_release(pcgpu_ctx *ctx, pcgpu_srs *srs) { release_after_stream(ctx, srs); }

extern "C" size_t pcgpu_srs_len(const pcgpu_srs *srs) { return srs ? srs->n : 0; }
extern "C" int pcgpu_srs_curve(const pcgpu_srs *srs) { return srs ? srs->curve : -1; }

extern "C" int pcgpu_msm(pcgpu_ctx *ctx, const pcgpu_srs *srs, size_t base_offset, const void *scalars, size_t n,
                         uint32_t flags, void *out_xy, uint8_t *out_inf) {
  return on_ctx(ctx, !srs || (n && !scalars) || !out_xy, [&]() -> int {
    DISPATCH_GROUP(srs->curve, return msm_impl<C>(ctx, srs, base_offset, scalars, n, flags, out_xy, out_inf, nullptr));
  });
}

extern "C" int pcgpu_msm_partial(pcgpu_ctx *ctx, const pcgpu_srs *srs, size_t base_offset, const void *scalars, size_t n,
                                 uint32_t flags, void *out_xyzz) {
  return on_ctx(ctx, !srs || (n && !scalars) || !out_xyzz, [&]() -> int {
    DISPATCH_CURVE(srs->curve, return msm_impl<C>(ctx, srs, base_offset, scalars, n, flags, nullptr, nullptr, out_xyzz));
  });
}

extern "C" int pcgpu_g1_sum_xyzz(pcgpu_ctx *ctx, int curve, const void *xyzz, size_t count, void *out_xy, uint8_t *out_inf) {
  return on_ctx(ctx, (count && !xyzz) || !out_xy, [&]() -> int {
    DISPATCH_CURVE(curve, return g1_sum_impl<C>(ctx, xyzz, count, out_xy, out_inf));
  });
}

extern "C" int pcgpu_g1_fixed_base_mul(pcgpu_ctx *ctx, int curve, const void *base_xy, const void *scalars, size_t n,
                                       uint32_t flags, void *out_xy) {
  return on_ctx(ctx, !base_xy || (n && (!scalars || !out_xy)), [&]() -> int {
    DISPATCH_CURVE(curve, return fixed_base_impl<C>(ctx, base_xy, scalars, n, flags, out_xy));
  });
}

extern "C" int pcgpu_g2_fixed_base_mul(pcgpu_ctx *ctx, int group, const void *base_xy, const void *scalars, size_t n,
                                       uint32_t flags, void *out_xy) {
  return on_ctx(ctx, !base_xy || (n && (!scalars || !out_xy)), [&]() -> int {
    switch (group) {
      case PCGPU_BLS12_381_G2: return fixed_base_impl<Bls12381G2>(ctx, base_xy, scalars, n, flags, out_xy);
      case PCGPU_BN254_G2: return fixed_base_impl<Bn254G2>(ctx, base_xy, scalars, n, flags, out_xy);
      default: return PCGPU_E_BADARG;
    }
  });
}

// ---- MultilinearPC (mlpc.cuh) -------------------------------------------------------------------------------------------
extern "C" int pcgpu_mlpc_register(pcgpu_ctx *ctx, int curve, uint32_t nv, const void *const *powers_of_h, const uint8_t *const *inf,
                                   uint32_t flags, pcgpu_mlpc **out) {
  const bool bad_args = !powers_of_h || nv == 0 || nv > 25 || (flags & ~(uint32_t)PCGPU_DEVICE_PTRS);
  return create(ctx, bad_args, out, [&](pcgpu_mlpc *m) -> int {
    m->curve = curve; m->nv = nv;
    DISPATCH_PAIRING_G2(curve, return mlpc_register_impl<C>(ctx, nv, powers_of_h, inf, flags, m));
  });
}

extern "C" void pcgpu_mlpc_release(pcgpu_ctx *ctx, pcgpu_mlpc *key) { release_after_stream(ctx, key); }

extern "C" int pcgpu_mlpc_open(pcgpu_ctx *ctx, const pcgpu_mlpc *key, const void *evals, size_t n, const void *point, uint32_t flags,
                               void *out_proofs_xy, uint8_t *out_proofs_inf, void *out_value) {
  return on_ctx(ctx, !key || !evals || !point || !out_proofs_xy || (flags & ~(uint32_t)PCGPU_DEVICE_PTRS), [&]() -> int {
    DISPATCH_PAIRING_G2(key->curve, return mlpc_open_impl<C>(ctx, key, evals, n, point, flags, out_proofs_xy, out_proofs_inf, out_value));
  });
}

// ---- pairing (pairing.cuh) ----------------------------------------------------------------------------------------------
extern "C" int pcgpu_multi_pairing(pcgpu_ctx *ctx, int curve, const void *g1_xy, const uint8_t *g1_inf, const void *g2_xy,
                                   const uint8_t *g2_inf, size_t k, size_t count, uint32_t flags, void *out_gt, uint8_t *out_is_one) {
  const bool bad_args = k > PCGPU_PAIRING_MAX_K || (!out_gt && !out_is_one) || (k && count && (!g1_xy || !g2_xy)) ||
                        (flags & ~(uint32_t)PCGPU_DEVICE_PTRS);
  return on_ctx(ctx, bad_args, [&]() -> int {
    DISPATCH_PAIRING(curve, return multi_pairing_impl<C>(ctx, g1_xy, g1_inf, g2_xy, g2_inf, k, count, flags, out_gt, out_is_one));
  });
}

extern "C" int pcgpu_g2_prepare(pcgpu_ctx *ctx, int curve, const void *g2_xy, const uint8_t *g2_inf, size_t n, uint32_t flags,
                                pcgpu_g2_prepared **out) {
  const bool bad_args = (n && !g2_xy) || n > UINT32_MAX || (flags & ~(uint32_t)PCGPU_DEVICE_PTRS);
  return create(ctx, bad_args, out, [&](pcgpu_g2_prepared *q) -> int {
    q->curve = curve; q->n = n;
    DISPATCH_PAIRING(curve, return g2_prepare_impl<C>(ctx, g2_xy, g2_inf, n, flags, q));
  });
}

extern "C" void pcgpu_g2_prepared_release(pcgpu_ctx *ctx, pcgpu_g2_prepared *q) { release_after_stream(ctx, q); }

extern "C" int pcgpu_multi_pairing_prepared(pcgpu_ctx *ctx, int curve, const void *g1_xy, const uint8_t *g1_inf,
                                            const pcgpu_g2_prepared *q, const uint32_t *q_index, size_t k, size_t count,
                                            uint32_t flags, void *out_gt, uint8_t *out_is_one) {
  bool bad_args = !q || q->curve != curve || k > PCGPU_PAIRING_MAX_K || (!out_gt && !out_is_one) ||
                  (k && count && (!g1_xy || !q_index)) || (flags & ~(uint32_t)PCGPU_DEVICE_PTRS);
  if (!bad_args && k && count)   // every index names a prepared point before anything runs
    for (size_t i = 0; i < k * count && !bad_args; i++) bad_args = q_index[i] >= q->n;
  return on_ctx(ctx, bad_args, [&]() -> int {
    DISPATCH_PAIRING(curve, return multi_pairing_prepared_impl<C>(ctx, g1_xy, g1_inf, q, q_index, k, count, flags, out_gt, out_is_one));
  });
}

extern "C" int pcgpu_fr_from_mont(pcgpu_ctx *ctx, int curve, const void *in, void *out, size_t n, uint32_t flags) {
  return on_ctx(ctx, (n && (!in || !out)), [&]() -> int {
    DISPATCH_CURVE(curve, return fr_from_mont_impl<C>(ctx, in, out, n, flags));
  });
}

extern "C" int pcgpu_fr_axpy(pcgpu_ctx *ctx, int curve, void *y, const void *c, const void *x, size_t n, uint32_t flags) {
  return on_ctx(ctx, !c || (n && (!y || !x)), [&]() -> int {
    DISPATCH_CURVE(curve, return fr_axpy_impl<C>(ctx, y, c, x, n, flags));
  });
}

extern "C" int pcgpu_fr_div_linear(pcgpu_ctx *ctx, int curve, const void *p, size_t n, const void *z, void *q, void *rem,
                                   uint32_t flags) {
  return on_ctx(ctx, !z || (n && !p) || (n > 1 && !q), [&]() -> int {
    DISPATCH_CURVE(curve, return fr_div_impl<C>(ctx, p, n, z, q, rem, flags));
  });
}

extern "C" int pcgpu_fr_inner_product(pcgpu_ctx *ctx, int curve, const void *a, const void *b, size_t n, void *out,
                                      uint32_t flags) {
  return on_ctx(ctx, !out || (n && (!a || !b)), [&]() -> int {
    DISPATCH_CURVE(curve, return fr_ip_impl<C>(ctx, a, b, n, out, flags));
  });
}

extern "C" int pcgpu_fr_row_mul(pcgpu_ctx *ctx, int curve, const void *v, const void *m, size_t rows, size_t cols, void *out,
                                uint32_t flags) {
  return on_ctx(ctx, (cols && !out) || (rows && cols && (!v || !m)), [&]() -> int {
    DISPATCH_CURVE(curve, return fr_row_mul_impl<C>(ctx, v, m, rows, cols, out, flags));
  });
}

extern "C" int pcgpu_kzg_commit(pcgpu_ctx *ctx, const pcgpu_srs *powers_of_g, const void *coeffs, size_t n,
                                const pcgpu_srs *powers_of_gamma_g, const void *blind, size_t n_blind, uint32_t flags,
                                void *out_xy, uint8_t *out_inf) {
  return on_ctx(ctx, !powers_of_g || (n && !coeffs) || (n_blind && !blind) || !out_xy ||
                         (powers_of_gamma_g && powers_of_gamma_g->curve != powers_of_g->curve), [&]() -> int {
    DISPATCH_CURVE(powers_of_g->curve,
                   return kzg_commit_impl<C>(ctx, powers_of_g, coeffs, n, powers_of_gamma_g, blind, n_blind, flags, out_xy, out_inf));
  });
}

extern "C" int pcgpu_kzg_open(pcgpu_ctx *ctx, const pcgpu_srs *powers_of_g, const void *coeffs, size_t n, const void *z,
                              const pcgpu_srs *powers_of_gamma_g, const void *blind, size_t n_blind, uint32_t flags,
                              void *out_w_xy, uint8_t *out_w_inf, void *out_random_v) {
  return on_ctx(ctx, !powers_of_g || !z || (n && !coeffs) || (n_blind && !blind) || !out_w_xy ||
                         (powers_of_gamma_g && powers_of_gamma_g->curve != powers_of_g->curve), [&]() -> int {
    DISPATCH_CURVE(powers_of_g->curve, return kzg_open_impl<C>(ctx, powers_of_g, coeffs, n, z, powers_of_gamma_g, blind,
                                                               n_blind, flags, out_w_xy, out_w_inf, out_random_v));
  });
}

extern "C" int pcgpu_selftest_field(pcgpu_ctx *ctx, int curve, uint64_t seed, size_t n, uint64_t *mismatches) {
  return on_ctx(ctx, !mismatches, [&]() -> int {
    DISPATCH_CURVE(curve, return selftest_field_impl<C>(ctx, seed, n, mismatches));
  });
}

extern "C" int pcgpu_msm_last_geometry(pcgpu_ctx *ctx, uint64_t *out, size_t len) {
  return guarded([&]() -> int {
  if (!ctx || (len && !out)) return PCGPU_E_BADARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  for (size_t i = 0; i < len && i < (size_t)PCGPU_GEOM_FIELDS; i++) out[i] = ctx->last_geom[i];
  return PCGPU_OK;
  });
}

extern "C" int pcgpu_diag_field_op(pcgpu_ctx *ctx, int curve, int which, int op, const void *a, const void *b, void *out, size_t n) {
  return on_ctx(ctx, which < 0 || which > 3 || op < 0 || op > (which == 3 ? 11 : 9) || (n && (!a || !b || !out)), [&]() -> int {
    if (which == 2) { DISPATCH_PAIRING_G2(curve, return diag_fq2_op_impl<C>(ctx, op, a, b, out, n)); }
    if (which == 3) { DISPATCH_PAIRING(curve, return diag_fq12_op_impl<C>(ctx, op, a, b, out, n)); }
    DISPATCH_CURVE(curve, return diag_field_op_impl<C>(ctx, which, op, a, b, out, n));
  });
}

extern "C" uint64_t pcgpu_launch_count(void) { return rt::launch_counter().load(); }

extern "C" int pcgpu_ntt(pcgpu_ctx *ctx, int curve, const void *in, size_t n_in, uint32_t logn, uint32_t flags, void *out) {
  return on_ctx(ctx, !out || (n_in && !in), [&]() -> int {
    DISPATCH_CURVE(curve, return ntt_impl<C>(ctx, in, n_in, logn, flags, out));
  });
}

extern "C" int pcgpu_msm_batch(pcgpu_ctx *ctx, const pcgpu_srs *srs, const void *scalars, size_t n, size_t count, uint32_t flags,
                               void *out_xy, uint8_t *out_inf) {
  return on_ctx(ctx, !srs || (n && count && !scalars) || (count && !out_xy), [&]() -> int {
    DISPATCH_CURVE(srs->curve, return msm_batch_impl<C>(ctx, srs, scalars, n, count, flags, out_xy, out_inf));
  });
}

// ---- HyraxPC (hyrax.cuh) -------------------------------------------------------------------------------------------------
// an odd number of variables is InvalidNumberOfVariables (hyrax/mod.rs:220-224, :289-293, :432-436); nv > 52 cannot be addressed
static bool hyrax_nv_bad(uint32_t nv) { return (nv & 1) || nv > 52; }

extern "C" int pcgpu_hyrax_commit(pcgpu_ctx *ctx, const pcgpu_srs *ck, uint32_t nv, const void *evals, const void *randomness,
                                  uint32_t flags, void *out_row_coms_xy, uint8_t *out_row_coms_inf, pcgpu_hyrax **out) {
  const bool bad_args = !ck || !evals || !randomness || !out_row_coms_xy || hyrax_nv_bad(nv) || (flags & ~(uint32_t)PCGPU_DEVICE_PTRS);
  return create(ctx, bad_args, out, [&](pcgpu_hyrax *h) -> int {
    DISPATCH_CURVE(ck->curve, return hyrax_commit_impl<C>(ctx, ck, nv, evals, randomness, flags, out_row_coms_xy, out_row_coms_inf, h));
  });
}

extern "C" void pcgpu_hyrax_release(pcgpu_ctx *ctx, pcgpu_hyrax *state) { release_after_stream(ctx, state); }

extern "C" int pcgpu_hyrax_open(pcgpu_ctx *ctx, const pcgpu_srs *ck, const pcgpu_hyrax *const *states, size_t count, uint32_t nv,
                                const void *point, const void *blinds, uint32_t flags, void *out_coms_xy, uint8_t *out_coms_inf,
                                void *out_lt, void *out_eval) {
  bool bad_args = !ck || hyrax_nv_bad(nv) || (nv && !point) || (count && (!states || !blinds || !out_coms_xy || !out_lt)) ||
                  (flags & ~(uint32_t)PCGPU_DEVICE_PTRS);
  for (size_t p = 0; !bad_args && p < count; p++) bad_args = !states[p];
  return on_ctx(ctx, bad_args, [&]() -> int {
    DISPATCH_CURVE(ck->curve, return hyrax_open_impl<C>(ctx, ck, states, count, nv, point, blinds, flags, out_coms_xy, out_coms_inf,
                                                        out_lt, out_eval));
  });
}

extern "C" int pcgpu_hyrax_check(pcgpu_ctx *ctx, const pcgpu_srs *vk, uint32_t nv, size_t count, const void *row_coms_xy,
                                 const uint8_t *row_coms_inf, const void *point, const void *proof_xy, const uint8_t *proof_inf,
                                 const void *proof_scalars, const void *challenges, uint32_t flags, uint8_t *out_ok) {
  const bool bad_args = !vk || hyrax_nv_bad(nv) || (nv && !point) ||
                        (count && (!row_coms_xy || !proof_xy || !proof_scalars || !challenges || !out_ok)) ||
                        (flags & ~(uint32_t)PCGPU_DEVICE_PTRS);
  return on_ctx(ctx, bad_args, [&]() -> int {
    DISPATCH_CURVE(vk->curve, return hyrax_check_impl<C>(ctx, vk, nv, count, row_coms_xy, row_coms_inf, point, proof_xy, proof_inf,
                                                         proof_scalars, challenges, flags, out_ok));
  });
}

extern "C" int pcgpu_ipa_begin(pcgpu_ctx *ctx, int curve, const void *comm_key_xy, size_t n, const void *coeffs, size_t n_coeffs,
                               const void *point, uint32_t flags, pcgpu_ipa **out) {
  const bool bad_args = !comm_key_xy || !point || n == 0 || (n & (n - 1)) || n_coeffs > n || (n_coeffs && !coeffs);
  return create(ctx, bad_args, out, [&](pcgpu_ipa *st) -> int {
    if (ctx->ipa_active) return PCGPU_E_BADARG;   // one halving loop at a time per context: the state lives in its IPA arena
    int rc = [&]() -> int { DISPATCH_CURVE(curve, return ipa_begin_impl<C>(ctx, comm_key_xy, n, coeffs, n_coeffs, point, flags, st)); }();
    if (rc == PCGPU_OK) { st->ctx = ctx; ctx->ipa_active = true; }
    return rc;
  });
}

// the IPA calls after begin run only on the context that began the open (pcgpu_ipa::ctx)
extern "C" int pcgpu_ipa_round_lr(pcgpu_ctx *ctx, pcgpu_ipa *st, const void *h_prime_xy, void *out_l_xy, uint8_t *out_l_inf,
                                  void *out_r_xy, uint8_t *out_r_inf) {
  return guarded([&]() -> int {
  if (!ctx || !st || st->ctx != ctx || !h_prime_xy || !out_l_xy || !out_r_xy) return PCGPU_E_BADARG;
  int src = ensure_siblings(ctx, 1);   // the two commitments of a round run on two streams
  if (src) return src;
  pcgpu_ctx *sib = ctx->siblings[0];
  std::lock_guard<std::mutex> lk(ctx->mu);
  std::lock_guard<std::mutex> lk2(sib->mu);
  SET_DEVICE(ctx);
  DISPATCH_CURVE(st->curve, return ipa_round_lr_impl<C>(ctx, sib, st, h_prime_xy, out_l_xy, out_l_inf, out_r_xy, out_r_inf));
  });
}

extern "C" int pcgpu_ipa_round_fold(pcgpu_ctx *ctx, pcgpu_ipa *st, const void *challenge, const void *challenge_inv) {
  return on_ctx(ctx, !st || st->ctx != ctx || !challenge || !challenge_inv, [&]() -> int {
    DISPATCH_CURVE(st->curve, return ipa_round_fold_impl<C>(ctx, st, challenge, challenge_inv));
  });
}

extern "C" size_t pcgpu_ipa_len(const pcgpu_ipa *st) { return st ? st->n : 0; }

extern "C" int pcgpu_ipa_finish(pcgpu_ctx *ctx, pcgpu_ipa *st, void *out_final_key_xy, void *out_c) {
  return on_ctx(ctx, !st || st->ctx != ctx, [&]() -> int {
    int rc = [&]() -> int { DISPATCH_CURVE(st->curve, return ipa_finish_impl<C>(ctx, st, out_final_key_xy, out_c)); }();
    ctx->ipa_active = false;   // the state's memory belongs to the context's IPA arena and is kept for the next open
    delete st;
    return rc;
  });
}

extern "C" int pcgpu_measure_imad_peak(pcgpu_ctx *ctx, double *ops_per_s) {
  return on_ctx(ctx, !ops_per_s, [&]() -> int {
    return measure_imad_peak_impl(ctx, ops_per_s);
  });
}

enum { PCGPU_BATCH_WAYS = 4 };

extern "C" int pcgpu_kzg_commit_batch(pcgpu_ctx *ctx, const pcgpu_srs *powers_of_g, const void *const *coeffs, const size_t *n,
                                      size_t count, uint32_t flags, void *out_xy, uint8_t *out_inf) {
  return guarded([&]() -> int {
  if (!ctx || !powers_of_g || (count && (!coeffs || !n || !out_xy))) return PCGPU_E_BADARG;
  const size_t ways = count < (size_t)PCGPU_BATCH_WAYS ? count : (size_t)PCGPU_BATCH_WAYS;
  if (ways > 1) {   // way 0 runs on ctx itself
    int rc = ensure_siblings(ctx, ways - 1);
    if (rc) return rc;
  }
  const size_t psz = affine_bytes(powers_of_g->curve);
  std::vector<int> rcs(ways, PCGPU_OK);
  auto work = [&](size_t w) {
    pcgpu_ctx *c = w == 0 ? ctx : ctx->siblings[w - 1];
    for (size_t i = w; i < count; i += ways) {
      int rc = pcgpu_kzg_commit(c, powers_of_g, coeffs[i], n[i], nullptr, nullptr, 0, flags, (char *)out_xy + i * psz,
                                out_inf ? out_inf + i : nullptr);
      if (rc) { rcs[w] = rc; return; }
    }
  };
  std::vector<std::thread> th;
  for (size_t w = 1; w < ways; w++) th.emplace_back(work, w);
  if (ways) work(0);
  for (auto &t : th) t.join();
  for (int rc : rcs) if (rc) return rc;
  return PCGPU_OK;
  });
}

extern "C" int pcgpu_ipa_check_final_key(pcgpu_ctx *ctx, const pcgpu_srs *comm_key, const void *challenges, uint32_t log_d,
                                         void *out_xy, uint8_t *out_inf) {
  return on_ctx(ctx, !comm_key || (log_d && !challenges) || !out_xy, [&]() -> int {
    DISPATCH_CURVE(comm_key->curve, return ipa_check_final_key_impl<C>(ctx, comm_key, challenges, log_d, out_xy, out_inf));
  });
}

extern "C" int pcgpu_ntt_split(uint32_t logn, uint32_t *m1, uint32_t *m2) {
  if (!m1 || !m2 || !ntt_supported(logn)) return PCGPU_E_BADARG;
  ntt_split(logn, m1, m2);
  return PCGPU_OK;
}

extern "C" int pcgpu_ntt_pass(pcgpu_ctx *ctx, int curve, uint32_t logn, uint32_t flags, int which, size_t lo, size_t count,
                              const void *in, size_t n_in, void *out) {
  return on_ctx(ctx, !out || (n_in && !in), [&]() -> int {
    DISPATCH_CURVE(curve, return ntt_pass_impl<C>(ctx, logn, flags, which, lo, count, in, n_in, out));
  });
}

extern "C" size_t pcgpu_g1_wire_size(int curve, uint32_t flags) {
  const bool comp = (flags & PCGPU_WIRE_COMPRESSED) != 0;
  switch (curve) {
    case PCGPU_BLS12_381: return wire_size<Bls12381>(comp);
    case PCGPU_BN254: return wire_size<Bn254>(comp);
    case PCGPU_PALLAS: return wire_size<Pallas>(comp);
    default: return 0;
  }
}

extern "C" int pcgpu_g1_serialize(pcgpu_ctx *ctx, int curve, const void *xy, const uint8_t *inf, size_t n, uint32_t flags,
                                  uint8_t *out_bytes) {
  return on_ctx(ctx, (n && (!xy || !out_bytes)), [&]() -> int {
    DISPATCH_CURVE(curve, return g1_serialize_impl<C>(ctx, xy, inf, n, flags, out_bytes));
  });
}

extern "C" int pcgpu_g1_deserialize(pcgpu_ctx *ctx, int curve, const uint8_t *bytes, size_t n, uint32_t flags, void *out_xy,
                                    uint8_t *out_inf, size_t *first_bad, int *reason) {
  return on_ctx(ctx, (n && (!bytes || !out_xy || !out_inf)), [&]() -> int {
    DISPATCH_CURVE(curve, return g1_deserialize_impl<C>(ctx, bytes, n, flags, out_xy, out_inf, first_bad, reason));
  });
}

extern "C" int pcgpu_fr_mul(pcgpu_ctx *ctx, int curve, const void *a, const void *b, void *out, size_t n, uint32_t flags) {
  return on_ctx(ctx, (n && (!a || !b || !out)), [&]() -> int {
    DISPATCH_CURVE(curve, return fr_mul_impl<C>(ctx, a, b, out, n, flags));
  });
}

// VariableBaseMSM::msm_bigint(bases, scalars) on bases that are not a registered key: the verifier-side combinations
// (hyrax/mod.rs:501-504 over row_coms; kzg10/mod.rs:357-373; marlin/mod.rs:109-148).  Composes the public entry points.
extern "C" int pcgpu_msm_bases(pcgpu_ctx *ctx, int curve, const void *bases_xy, const uint8_t *inf, const void *scalars, size_t n,
                               uint32_t flags, void *out_xy, uint8_t *out_inf) {
  return guarded([&]() -> int {
  if (!ctx || !out_xy || (n && (!bases_xy || !scalars)) || (flags & (PCGPU_DEVICE_PTRS | PCGPU_SRS_PRECOMPUTE | PCGPU_SRS_COMB)))
    return PCGPU_E_BADARG;
  pcgpu_srs *srs = nullptr;
  int rc = pcgpu_srs_register(ctx, curve, bases_xy, inf, n, 0, &srs);
  if (rc) return rc;
  rc = pcgpu_msm(ctx, srs, 0, scalars, n, flags, out_xy, out_inf);
  pcgpu_srs_release(ctx, srs);
  return rc;
  });
}

extern "C" int pcgpu_ntt_batch(pcgpu_ctx *ctx, int curve, const void *in, size_t n_in, size_t count, uint32_t logn, uint32_t flags,
                               void *out) {
  return on_ctx(ctx, (count && (!out || (n_in && !in))), [&]() -> int {
    DISPATCH_CURVE(curve, return ntt_batch_impl<C>(ctx, in, n_in, count, logn, flags, out));
  });
}

extern "C" int pcgpu_ntt_pass1_peer(pcgpu_ctx *ctx, int curve, uint32_t logn, uint32_t flags, size_t lo, size_t count, const void *in,
                                    size_t n_in, void *const *dst, uint32_t world) {
  return on_ctx(ctx, !dst || (n_in && !in), [&]() -> int {
    DISPATCH_CURVE(curve, return ntt_pass1_peer_impl<C>(ctx, logn, flags, lo, count, in, n_in, dst, world));
  });
}

// ---- multi-GPU over NVLink peer memory (peer.cuh) ---------------------------------------------------------------------
extern "C" size_t pcgpu_peer_window_bytes(void) { return (size_t)PEER_WINDOW_BYTES; }

extern "C" int pcgpu_peer_alloc(pcgpu_ctx *ctx, size_t bytes, void **out_ptr, uint8_t *handle) {
  return on_ctx(ctx, !out_ptr || !handle || bytes == 0, [&]() -> int {
    void *p = nullptr;
    int rc = rt::dev_malloc(&p, bytes);
    if (rc) return rc;
    memset(handle, 0, PCGPU_IPC_HANDLE_BYTES);
#ifndef PCGPU_EMUL
    if (cudaMemset(p, 0, bytes) != cudaSuccess) { rt::dev_free(p); return PCGPU_E_CUDA; }
    cudaIpcMemHandle_t h;
    static_assert(sizeof(h) <= PCGPU_IPC_HANDLE_BYTES, "IPC handle larger than the ABI's handle");
    if (cudaIpcGetMemHandle(&h, p) != cudaSuccess) { rt::dev_free(p); return PCGPU_E_CUDA; }
    memcpy(handle, &h, sizeof h);
#else
    memset(p, 0, bytes);
    memcpy(handle, &p, sizeof p);   // emulation: every "rank" lives in this process
#endif
    *out_ptr = p;
    return PCGPU_OK;
  });
}

extern "C" int pcgpu_peer_open(pcgpu_ctx *ctx, const uint8_t *handle, void **out_ptr) {
  return on_ctx(ctx, !handle || !out_ptr, [&]() -> int {
#ifndef PCGPU_EMUL
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, sizeof h);
    void *p = nullptr;
    if (cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); return PCGPU_E_CUDA; }
    *out_ptr = p;
#else
    memcpy(out_ptr, handle, sizeof(void *));
#endif
    return PCGPU_OK;
  });
}

extern "C" int pcgpu_peer_close(pcgpu_ctx *ctx, void *mapped) {
  return on_ctx(ctx, !mapped, [&]() -> int {
#ifndef PCGPU_EMUL
    cudaStreamSynchronize(ctx->stream);
    if (cudaIpcCloseMemHandle(mapped) != cudaSuccess) return PCGPU_E_CUDA;
#endif
    return PCGPU_OK;
  });
}

extern "C" int pcgpu_peer_free(pcgpu_ctx *ctx, void *ptr) {
  return on_ctx(ctx, !ptr, [&]() -> int {
#ifndef PCGPU_EMUL
    cudaStreamSynchronize(ctx->stream);
#endif
    rt::dev_free(ptr);
    return PCGPU_OK;
  });
}

static int peer_args_ok(void *const *win, uint32_t rank, uint32_t world) {
  if (!win || world == 0 || world > (uint32_t)PEER_MAX_WORLD || rank >= world) return 0;
  for (uint32_t d = 0; d < world; d++) if (!win[d]) return 0;
  return 1;
}

extern "C" int pcgpu_peer_signal(pcgpu_ctx *ctx, void *const *win, uint32_t rank, uint32_t world, uint32_t channel, uint64_t epoch) {
  return on_ctx(ctx, !peer_args_ok(win, rank, world) || channel >= 8, [&]() -> int {
    PeerSignalBody b;
    memset(&b, 0, sizeof b);
    for (uint32_t d = 0; d < world; d++) b.win[d] = (char *)win[d];
    b.rank = rank; b.world = world; b.flag_off = (uint32_t)PEER_FLAG_OFFSET + 256u * channel; b.epoch = epoch;
    int rc = rt::launch<32>(b, world, ctx->stream);
    if (rc) return rc;
    return rt::stream_sync(ctx->stream);
  });
}

extern "C" int pcgpu_peer_wait(pcgpu_ctx *ctx, void *local_win, uint32_t world, uint32_t channel, uint64_t epoch) {
  return on_ctx(ctx, !local_win || world == 0 || world > (uint32_t)PEER_MAX_WORLD || channel >= 8, [&]() -> int {
    rt::stream_t st = ctx->stream;
    uint32_t *d_timeout = &ctx->d_words->peer_timeout;
    int rc;
    if ((rc = rt::dev_memset(d_timeout, 0, 4, st))) return rc;
    if ((rc = rt::launch<32>(PeerWaitBody{(const char *)local_win, world, (uint32_t)PEER_FLAG_OFFSET + 256u * channel, epoch, PEER_WAIT_CYCLES, d_timeout}, world, st))) return rc;
    uint32_t t = 0;
    if ((rc = rt::copy_d2h(&t, d_timeout, 4, st))) return rc;
    if ((rc = rt::stream_sync(st))) return rc;
    return t ? PCGPU_E_PEER : PCGPU_OK;
  });
}

extern "C" int pcgpu_msm_peer(pcgpu_ctx *ctx, const pcgpu_srs *srs, size_t base_offset, const void *scalars, size_t n, uint32_t flags,
                              void *const *win, uint32_t rank, uint32_t world, uint64_t epoch, void *out_xy, uint8_t *out_inf) {
  return on_ctx(ctx, !srs || (n && !scalars) || !out_xy || !peer_args_ok(win, rank, world) || epoch == 0, [&]() -> int {
    DISPATCH_CURVE(srs->curve, return msm_peer_impl<C>(ctx, srs, base_offset, scalars, n, flags, win, rank, world, epoch, out_xy, out_inf));
  });
}

// ---- linear-code commitments (hash.cuh) ---------------------------------------------------------------------------------
extern "C" int pcgpu_lincode_hash_columns(pcgpu_ctx *ctx, int curve, const void *ext_mat, size_t n_rows, size_t n_cols, int hash,
                                          uint32_t flags, uint8_t *out_leaves) {
  return on_ctx(ctx, (n_cols && !out_leaves) || (n_rows && n_cols && !ext_mat), [&]() -> int {
    DISPATCH_CURVE(curve, return lincode_hash_columns_impl<C>(ctx, ext_mat, n_rows, n_cols, hash, flags, out_leaves));
  });
}

extern "C" int pcgpu_merkle_tree(pcgpu_ctx *ctx, const uint8_t *leaves, size_t n_leaves, uint32_t flags, uint8_t *out_nodes,
                                 uint8_t *out_root) {
  return on_ctx(ctx, !leaves, [&]() -> int {
    return merkle_tree_impl(ctx, leaves, n_leaves, flags, out_nodes, out_root);
  });
}

extern "C" int pcgpu_lincode_commit(pcgpu_ctx *ctx, int curve, const void *mat, size_t n_rows, size_t n_cols, uint32_t log_ext_cols,
                                    int hash, uint32_t flags, void *out_ext_mat, uint8_t *out_leaves, uint8_t *out_nodes,
                                    uint8_t *out_root) {
  return on_ctx(ctx, (n_rows && n_cols && !mat), [&]() -> int {
    DISPATCH_CURVE(curve, return lincode_commit_impl<C>(ctx, mat, n_rows, n_cols, log_ext_cols, hash, flags, out_ext_mat, out_leaves,
                                                        out_nodes, out_root));
  });
}

// ---- Brakedown (sprs.cuh) -----------------------------------------------------------------------------------------------
extern "C" int pcgpu_brakedown_register(pcgpu_ctx *ctx, int curve, size_t m, size_t m_ext, size_t levels, const uint64_t *a_dims,
                                        const uint64_t *b_dims, const uint64_t *const *ind_ptr, const uint64_t *const *col_ind,
                                        const void *const *val, uint32_t flags, pcgpu_brakedown **out) {
  (void)flags;
  return create(ctx, false, out, [&](pcgpu_brakedown *bd) -> int {
    DISPATCH_CURVE(curve, return brakedown_register_impl<C>(ctx, m, m_ext, levels, a_dims, b_dims, ind_ptr, col_ind, val, bd));
  });
}

extern "C" void pcgpu_brakedown_release(pcgpu_ctx *ctx, pcgpu_brakedown *code) { release_after_stream(ctx, code); }

extern "C" int pcgpu_brakedown_encode(pcgpu_ctx *ctx, const pcgpu_brakedown *code, const void *mat, size_t n_rows, size_t n_cols,
                                      uint32_t flags, void *out_ext) {
  return on_ctx(ctx, !code || !out_ext || (n_rows && n_cols && !mat), [&]() -> int {
    DISPATCH_CURVE(code->curve, return brakedown_commit_impl<C>(ctx, code, mat, n_rows, n_cols, -1, flags, out_ext, nullptr, nullptr, nullptr));
  });
}

extern "C" int pcgpu_brakedown_commit(pcgpu_ctx *ctx, const pcgpu_brakedown *code, const void *mat, size_t n_rows, size_t n_cols, int hash,
                                      uint32_t flags, void *out_ext, uint8_t *out_leaves, uint8_t *out_nodes, uint8_t *out_root) {
  return on_ctx(ctx, !code || hash < 0 || (n_rows && n_cols && !mat), [&]() -> int {
    DISPATCH_CURVE(code->curve, return brakedown_commit_impl<C>(ctx, code, mat, n_rows, n_cols, hash, flags, out_ext, out_leaves, out_nodes,
                                                                out_root));
  });
}

extern "C" int pcgpu_fr_sprs_row_mul(pcgpu_ctx *ctx, int curve, size_t n, size_t m, const uint64_t *ind_ptr, const uint64_t *col_ind,
                                     const void *val, const void *v, size_t count, uint32_t flags, void *out) {
  return on_ctx(ctx, !ind_ptr || (m && count && !out) || (n && count && !v), [&]() -> int {
    DISPATCH_CURVE(curve, return fr_sprs_row_mul_impl<C>(ctx, n, m, ind_ptr, col_ind, val, v, count, flags, out));
  });
}

// ---- fused KZG10 commit + open ------------------------------------------------------------------------------------------
static int ensure_siblings(pcgpu_ctx *ctx, size_t count) {
  std::lock_guard<std::mutex> lk(ctx->mu);
  while (ctx->siblings.size() < count) {
    pcgpu_ctx *s = nullptr;
    int rc = pcgpu_init(ctx->device, &s);
    if (rc) return rc;
    ctx->siblings.push_back(s);
  }
  return PCGPU_OK;
}

// one polynomial on the context pair (a, b); both mutexes are taken in a fixed order (a is never somebody's b)
static int commit_open_pair(pcgpu_ctx *a, pcgpu_ctx *b, const pcgpu_srs *pg, const void *coeffs, size_t n, const void *z, uint32_t flags,
                            void *out_c_xy, uint8_t *out_c_inf, void *out_w_xy, uint8_t *out_w_inf) {
  std::lock_guard<std::mutex> la(a->mu);
  std::lock_guard<std::mutex> lb(b->mu);
  SET_DEVICE(a);
  DISPATCH_CURVE(pg->curve, return kzg_commit_open_impl<C>(a, b, pg, coeffs, n, z, flags, out_c_xy, out_c_inf, out_w_xy, out_w_inf));
}

extern "C" int pcgpu_kzg_commit_open(pcgpu_ctx *ctx, const pcgpu_srs *powers_of_g, const void *coeffs, size_t n, const void *z,
                                     uint32_t flags, void *out_comm_xy, uint8_t *out_comm_inf, void *out_w_xy, uint8_t *out_w_inf) {
  return guarded([&]() -> int {
  if (!ctx || !powers_of_g || !z || (n && !coeffs) || !out_comm_xy || !out_w_xy) return PCGPU_E_BADARG;
  int rc = ensure_siblings(ctx, 1);
  if (rc) return rc;
  return commit_open_pair(ctx, ctx->siblings[0], powers_of_g, coeffs, n, z, flags, out_comm_xy, out_comm_inf, out_w_xy, out_w_inf);
  });
}

enum { PCGPU_COMMIT_OPEN_WAYS = 2, PCGPU_COMMIT_OPEN_MAX_WAYS = 4, PCGPU_BATCH_PAIR_TDIV = 2 };   // polynomials in flight (two MSM pipelines each); half-wave pair kernels in batch mode

extern "C" int pcgpu_kzg_commit_open_batch(pcgpu_ctx *ctx, const pcgpu_srs *powers_of_g, const void *const *coeffs, const size_t *n,
                                           size_t count, const void *z, uint32_t flags, void *out_comm_xy, uint8_t *out_comm_inf,
                                           void *out_w_xy, uint8_t *out_w_inf) {
  return guarded([&]() -> int {
  if (!ctx || !powers_of_g || !z || (count && (!coeffs || !n || !out_comm_xy || !out_w_xy))) return PCGPU_E_BADARG;
  size_t max_ways = PCGPU_COMMIT_OPEN_WAYS;
  if (const char *e = getenv("PCGPU_COMMIT_OPEN_WAYS")) { int v = atoi(e); if (v >= 1 && v <= PCGPU_COMMIT_OPEN_MAX_WAYS) max_ways = (size_t)v; }   // tuning knob
  const size_t ways = count < max_ways ? count : max_ways;
  if (ways == 0) return PCGPU_OK;
  int rc = ensure_siblings(ctx, 2 * ways - 1);   // way 0: (ctx, sib[0]); way w >= 1: (sib[2w-1], sib[2w])
  if (rc) return rc;
  const size_t psz = affine_bytes(powers_of_g->curve);
  int rcs[PCGPU_COMMIT_OPEN_MAX_WAYS] = {PCGPU_OK, PCGPU_OK, PCGPU_OK, PCGPU_OK};
  // throughput mode of the pair rounds while several pipelines are in flight (msm.cuh); PCGPU_BATCH_TDIV overrides
  uint32_t tdiv = ways >= 2 ? PCGPU_BATCH_PAIR_TDIV : 1;
  if (const char *e = getenv("PCGPU_BATCH_TDIV")) { int v = atoi(e); if (v >= 1 && v <= 8) tdiv = (uint32_t)v; }
  auto work = [&](size_t w) {
    pcgpu_ctx *a = w == 0 ? ctx : ctx->siblings[2 * w - 1], *b = ctx->siblings[w == 0 ? 0 : 2 * w];
    a->pair_tdiv = tdiv; b->pair_tdiv = tdiv;
    struct Restore { pcgpu_ctx *a, *b; ~Restore() { a->pair_tdiv = 1; b->pair_tdiv = 1; } } restore{a, b};
    for (size_t i = w; i < count; i += ways) {
      int r = commit_open_pair(a, b, powers_of_g, coeffs[i], n[i], (const char *)z, flags, (char *)out_comm_xy + i * psz,
                               out_comm_inf ? out_comm_inf + i : nullptr, (char *)out_w_xy + i * psz, out_w_inf ? out_w_inf + i : nullptr);
      if (r) { rcs[w] = r; return; }
    }
  };
  try {
    std::vector<std::thread> th;
    for (size_t w = 1; w < ways; w++) th.emplace_back(work, w);
    work(0);
    for (auto &t : th) t.join();
  } catch (...) { return PCGPU_E_OOM; }
  for (size_t w = 0; w < ways; w++) if (rcs[w]) return rcs[w];
  return PCGPU_OK;
  });
}

// ---- device buffers for callers that keep polynomials on the GPU across calls (PCGPU_DEVICE_PTRS arguments) ------------------
extern "C" int pcgpu_buf_alloc(pcgpu_ctx *ctx, size_t bytes, void **out) {
  return on_ctx(ctx, !out, [&]() -> int {
    void *p = nullptr;
    int rc = rt::dev_malloc(&p, bytes);
    if (rc) return rc;
    if ((rc = rt::dev_memset(p, 0, bytes ? bytes : 1, ctx->stream)) || (rc = rt::stream_sync(ctx->stream))) { rt::dev_free(p); return rc; }
    *out = p;
    return PCGPU_OK;
  });
}
extern "C" int pcgpu_buf_free(pcgpu_ctx *ctx, void *p) {
  return on_ctx(ctx, false, [&]() -> int {
    int rc = rt::stream_sync(ctx->stream);
    rt::dev_free(p);
    return rc;
  });
}
extern "C" int pcgpu_buf_write(pcgpu_ctx *ctx, void *dst, size_t dst_off, const void *src, size_t bytes) {
  return on_ctx(ctx, (bytes && (!dst || !src)), [&]() -> int {
    int rc = bytes ? rt::copy_h2d((char *)dst + dst_off, src, bytes, ctx->stream) : PCGPU_OK;
    return rc ? rc : rt::stream_sync(ctx->stream);
  });
}
extern "C" int pcgpu_buf_read(pcgpu_ctx *ctx, const void *src, size_t src_off, void *dst, size_t bytes) {
  return on_ctx(ctx, (bytes && (!dst || !src)), [&]() -> int {
    int rc = bytes ? rt::copy_d2h(dst, (const char *)src + src_off, bytes, ctx->stream) : PCGPU_OK;
    return rc ? rc : rt::stream_sync(ctx->stream);
  });
}
extern "C" int pcgpu_buf_zero(pcgpu_ctx *ctx, void *dst, size_t dst_off, size_t bytes) {
  return on_ctx(ctx, (bytes && !dst), [&]() -> int {
    int rc = bytes ? rt::dev_memset((char *)dst + dst_off, 0, bytes, ctx->stream) : PCGPU_OK;
    return rc ? rc : rt::stream_sync(ctx->stream);
  });
}

extern "C" int pcgpu_g1_sample_generators(pcgpu_ctx *ctx, int curve, const uint8_t *protocol_name, size_t name_len, uint64_t first_index,
                                          size_t n, uint32_t flags, void *out_xy) {
  return on_ctx(ctx, (name_len && !protocol_name) || (n && !out_xy), [&]() -> int {
    DISPATCH_CURVE(curve, return g1_sample_generators_impl<C>(ctx, protocol_name, name_len, first_index, n, flags, out_xy));
  });
}
