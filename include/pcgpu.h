/*
 * pcgpu.h -- C ABI of the H100-native polynomial-commitment compute engine.
 *
 * This is the drop-in boundary for the hot path of arkworks-rs/poly-commit (reference @ a05ec99;
 * all file:line citations below are relative to its root).  The reference has no FFI of
 * its own: the path sits behind Rust trait methods of un-vendored crates (ark-ec / ark-poly 0.5.0).
 * Each entry point therefore names the Rust call it replaces; INTEGRATION.md shows the Rust-side
 * `extern "C"` declarations and the patched call sites.
 *
 * Conventions (SURVEY.md section 8b)
 *   - Field elements: little-endian 64-bit limbs, least-significant first; 4 limbs for every Fr and for
 *     BN254/Pallas Fq, 6 limbs for BLS12-381 Fq (== ark-ff BigInt<N>([u64; N])).
 *   - "mont": Montgomery form with R = 2^(64*limbs) (the in-memory form of ark-ff Fp).
 *     "canonical": plain integer (what F::into_bigint returns).
 *   - Affine G1 point: x || y (2*limbs u64, Montgomery) plus a separate infinity byte (1 = identity;
 *     x, y are then written as zero).  Byte-identical to ark-ec's (x, y) so equality is a memcmp.
 *   - Every call is synchronous: on return the outputs are written.  The caller owns all host buffers;
 *     the library owns device memory behind the opaque handles.  Nothing unwinds across the ABI:
 *     0 = success, negative = error (pcgpu_strerror).
 *   - Thread safety: calls on one pcgpu_ctx are serialised by an internal mutex; use one context
 *     per host thread for concurrency (hyrax/mod.rs:233-242 calls msm from a Rayon par_iter).
 *   - There is no CPU fallback: every entry point fails with PCGPU_E_CUDA when no sm_90 device
 *     is usable.
 */
#ifndef PCGPU_H
#define PCGPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct pcgpu_ctx pcgpu_ctx;
typedef struct pcgpu_srs pcgpu_srs;

/* curve ids mirror the type parameter E / G of the reference's schemes */
enum { PCGPU_BLS12_381 = 0, PCGPU_BN254 = 1, PCGPU_PALLAS = 2 };
/* G2 group ids (E::G2 of the pairing curves): 0x100 + the curve id, out of the range of curve ids.  Accepted where a key's
 * group is named -- pcgpu_srs_register, pcgpu_msm_bases, pcgpu_g2_fixed_base_mul -- and by pcgpu_msm through the key; every
 * entry point that takes a scalar-field or G1 curve returns PCGPU_E_BADARG for them.  A G2 affine point is
 * x.c0 || x.c1 || y.c0 || y.c1, each `limbs` u64 Montgomery (Fq2 = Fq[u] / (u^2 + 1)), plus the separate infinity byte. */
enum { PCGPU_BLS12_381_G2 = 0x100, PCGPU_BN254_G2 = 0x101 };

enum {
  PCGPU_OK = 0,
  PCGPU_E_CUDA = -1,   /* CUDA runtime / launch failure, or no usable device */
  PCGPU_E_OOM = -2,    /* device allocation failed */
  PCGPU_E_BADARG = -3, /* null pointer, unknown curve id, ... */
  PCGPU_E_LEN = -4,    /* base_offset + n exceeds the registered bases (msm() returns Err(len) in ark-ec) */
  PCGPU_E_RANGE = -5,  /* a canonical scalar is >= r: not a reduced field element (into_bigint never produces one) */
  PCGPU_E_DEGREE = -6, /* Error::TooManyCoefficients, kzg10/mod.rs:392-402 */
  PCGPU_E_HIDING = -7, /* Error::HidingBoundToolarge, kzg10/mod.rs:404-422 */
  PCGPU_E_INVALID = -8, /* SerializationError::{InvalidData, UnexpectedFlags}: a wire-format element failed to decode / validate */
  PCGPU_E_PEER = -9     /* multi-GPU exchange: a peer did not signal within the wait budget, or its record is malformed */
};

/* flags */
enum {
  PCGPU_SCALARS_MONT = 1u,   /* scalars are Montgomery Fr; F::into_bigint is fused into the digit pass */
  PCGPU_DEVICE_PTRS = 2u,    /* bulk array arguments are device pointers (results stay host pointers) */
  PCGPU_SRS_PRECOMPUTE = 4u, /* srs_register: also store 2^(c*k)-multiples of the bases (window folding) */
  PCGPU_NTT_INVERSE = 8u,    /* pcgpu_ntt: ifft instead of fft */
  PCGPU_SRS_COMB = 16u,      /* srs_register: build fixed-base comb tables for pcgpu_msm_batch (shared-base batches) */
  PCGPU_WIRE_COMPRESSED = 32u,   /* g1_serialize / g1_deserialize: Compress::Yes (x + flag bits) instead of Compress::No */
  PCGPU_WIRE_NO_VALIDATE = 64u   /* g1_deserialize: Validate::No (skip the on-curve and subgroup checks) */
};

/* ---- context ---------------------------------------------------------------------------------- */
int pcgpu_init(int device, pcgpu_ctx **out);
void pcgpu_destroy(pcgpu_ctx *ctx);
const char *pcgpu_strerror(int code);
/* Run on the caller's CUDA stream (cudaStream_t passed as void*); NULL restores the context's own stream. */
int pcgpu_set_stream(pcgpu_ctx *ctx, void *cuda_stream);
/* Per-stage device timings (CUDA events on the launching stream).  stage: 0 digits/count, 1 scan,
 * 2 scatter, 3 tasks, 4 bucket accumulate (XYZZ), 5 bucket reduce, 6 final (host tail, wall clock), 7 fr division,
 * 8 fr axpy, 9 ntt, 10 comb batch, 11 affine pair rounds (all), 12 affine pair round 0 kernel alone, 13 peer push + wait,
 * 14 column hashes + Merkle tree, 15 Brakedown encoding, 16 MultilinearPC open fold chain, 17 pairing Miller loops + final
 * exponentiations (prepared or not), 18 G2 line preparation, 19 Hyrax transpose, tensors, row product and inner products.
 * enable=1 starts recording; get returns accumulated milliseconds and launch count since enable. */
int pcgpu_profile_enable(pcgpu_ctx *ctx, int enable);
int pcgpu_profile_get(pcgpu_ctx *ctx, int stage, double *ms, uint64_t *count);

/* ---- SRS / committer key ---------------------------------------------------------------------- */
/* The creators -- pcgpu_srs_register, pcgpu_mlpc_register, pcgpu_brakedown_register, pcgpu_ipa_begin, pcgpu_g2_prepare,
 * pcgpu_hyrax_commit -- set *out to
 * NULL whenever out is non-NULL, whatever they return, and store the new handle in it only on PCGPU_OK. */
/* Upload n affine bases once (kzg10 Powers::powers_of_g, data_structures.rs:124-129; ipa CommitterKey::comm_key;
 * hyrax com_key).  inf may be NULL (no identity points).  `curve` may be a G2 group id: the key then holds raw G2 bases
 * (PCGPU_SRS_PRECOMPUTE and PCGPU_SRS_COMB return PCGPU_E_BADARG) and pcgpu_msm over it is
 * <E::G2 as VariableBaseMSM>::msm_bigint, run without batched-affine rounds. */
int pcgpu_srs_register(pcgpu_ctx *ctx, int curve, const void *bases_xy, const uint8_t *inf, size_t n, uint32_t flags,
                       pcgpu_srs **out);
void pcgpu_srs_release(pcgpu_ctx *ctx, pcgpu_srs *srs);
size_t pcgpu_srs_len(const pcgpu_srs *srs);
int pcgpu_srs_curve(const pcgpu_srs *srs);

/* ---- MSM -------------------------------------------------------------------------------------- */
/* <G as VariableBaseMSM>::msm_bigint(&bases[base_offset..], scalars)   kzg10/mod.rs:175-178, :199-203, :255-258,
 * :270-273; ipa_pc/mod.rs:64; hyrax/mod.rs:92, :501.  Sums the first n pairs; n == 0 returns the identity
 * (kzg10/mod.rs:197-203 on the non-hiding path).  base_offset models `&powers_of_g[num_leading_zeros..]`.
 * scalars: n x 4 u64, canonical unless PCGPU_SCALARS_MONT.  out_xy: affine Montgomery x||y; *out_inf: 1 if identity. */
int pcgpu_msm(pcgpu_ctx *ctx, const pcgpu_srs *srs, size_t base_offset, const void *scalars, size_t n, uint32_t flags,
              void *out_xy, uint8_t *out_inf);
/* Same, result left projective (XYZZ: X, Y, ZZ, ZZZ each `limbs` u64, Montgomery; ZZ == 0 is the identity) -- the
 * per-GPU partial of an index-range-sharded MSM before the point-sum (SURVEY.md section 8e, partitioning B). */
int pcgpu_msm_partial(pcgpu_ctx *ctx, const pcgpu_srs *srs, size_t base_offset, const void *scalars, size_t n,
                      uint32_t flags, void *out_xyzz);
/* Point-sum of `count` XYZZ partials (host memory) -> affine.  The "NCCL point-sum": ranks all-gather their
 * partials as bytes and each adds them locally (NCCL has no reduction operator for curve points). */
int pcgpu_g1_sum_xyzz(pcgpu_ctx *ctx, int curve, const void *xyzz, size_t count, void *out_xy, uint8_t *out_inf);

/* `count` MSMs of length n over the SAME bases (the first n of `srs`): out[r] = sum_i scalars[r*n + i] * bases[i].
 * HyraxPC::commit row loop, hyrax/mod.rs:233-242 (dim Pedersen commitments over one com_key; append h as base n and the
 * row randomness as scalar n to get `pedersen_commit(row) + h * r` in the same pass).  With PCGPU_SRS_COMB tables the
 * batch is a fixed-base comb (no buckets); otherwise the rows run through pcgpu_msm one by one.
 * out_xy: count affine points; out_inf: count bytes. */
int pcgpu_msm_batch(pcgpu_ctx *ctx, const pcgpu_srs *srs, const void *scalars, size_t n, size_t count, uint32_t flags,
                    void *out_xy, uint8_t *out_inf);

/* <G as VariableBaseMSM>::msm_bigint(bases, scalars) on bases that are NOT a registered key -- the verifier-side
 * combinations: HyraxPC::check's t_prime over row_coms (hyrax/mod.rs:501-504), KZG10::batch_check's combination loop
 * (kzg10/mod.rs:357-373), Marlin::accumulate_commitments_and_values (marlin/mod.rs:109-148).  Host pointers only; the bases
 * are uploaded, used once and dropped.  flags: PCGPU_SCALARS_MONT. */
int pcgpu_msm_bases(pcgpu_ctx *ctx, int curve, const void *bases_xy, const uint8_t *inf, const void *scalars, size_t n,
                    uint32_t flags, void *out_xy, uint8_t *out_inf);

/* g.batch_mul(scalars): out[i] = scalars[i] * base -- KZG10::setup, kzg10/mod.rs:76, :82-86 (used to build synthetic
 * SRSs on the device).  base_xy: one affine point (host).  scalars: n canonical.  out_xy: n affine points, x||y only
 * (an identity result is written as x = y = 0).  With PCGPU_DEVICE_PTRS scalars and out_xy are device pointers. */
int pcgpu_g1_fixed_base_mul(pcgpu_ctx *ctx, int curve, const void *base_xy, const void *scalars, size_t n, uint32_t flags,
                            void *out_xy);
/* The same in G2: h.batch_mul(scalars), MultilinearPC::setup (multilinear_pc/mod.rs:62).  group: PCGPU_BLS12_381_G2 or
 * PCGPU_BN254_G2; base_xy and out_xy are G2 affine points. */
int pcgpu_g2_fixed_base_mul(pcgpu_ctx *ctx, int group, const void *base_xy, const void *scalars, size_t n, uint32_t flags,
                            void *out_xy);

/* InnerProductArgPC::sample_generators (ipa_pc/mod.rs:302-325) and HyraxPC::setup's generator loop (hyrax/mod.rs:143-163):
 * out[t] = the point obtained from Blake2s-256(protocol_name || (first_index + t) as u64 LE [|| j as u64 LE, j = 0, 1, ... while
 * G::from_random_bytes returns None]) -- "PC-DL-2020" for the IPA (ipa_pc/mod.rs:50), "Hyrax protocol" for Hyrax
 * (hyrax/mod.rs:26).  mul_by_cofactor_to_group is the identity on the cofactor-1 curves (BN254, Pallas); for BLS12-381 the
 * caller clears the cofactor.  n affine points x||y (Montgomery); an identity result (infinity flag on x = 0) is written as
 * zeros.  name_len <= 40.  With PCGPU_DEVICE_PTRS out_xy is a device pointer. */
int pcgpu_g1_sample_generators(pcgpu_ctx *ctx, int curve, const uint8_t *protocol_name, size_t name_len, uint64_t first_index, size_t n,
                               uint32_t flags, void *out_xy);

/* ---- G1 wire formats (SURVEY.md section 8f rank 1) ------------------------------------------------
 * The bytes CanonicalSerialize / CanonicalDeserialize produce for the G1Affine elements of kzg10::Powers
 * (kzg10/data_structures.rs:142-177), UniversalParams.powers_of_g (:57-112), Commitment (:315-328) and Proof.w (:479-495).
 * The encodings come from un-vendored crates (ark-serialize / ark-ec 0.5.0; ark-bls12-381 0.5.0's ZCash form) and are
 * restated from their published behaviour -- see poly-commit_b200/csrc/wire.cuh for the byte layouts.
 * pcgpu_g1_wire_size: bytes per point (BLS12-381 48 / 96, BN254 32 / 64, Pallas 33 / 65), 0 for an unknown curve.
 * pcgpu_g1_serialize: n affine points (Montgomery x||y + infinity bytes, inf may be NULL) -> n * wire_size bytes.
 * pcgpu_g1_deserialize: the inverse; decompression (one square root in Fq per point) and, unless PCGPU_WIRE_NO_VALIDATE,
 *   Valid::check (on curve, prime-order subgroup) run on the device.  On PCGPU_E_INVALID *first_bad (may be NULL) receives
 *   the index of the first offending element and *reason 1 = unexpected flags, 2 = coordinate >= p, 3 = not on the curve
 *   (no square root), 4 = not in the subgroup; the outputs of offending elements are zeroed.
 * With PCGPU_DEVICE_PTRS the point / byte / inf arrays are device pointers. */
size_t pcgpu_g1_wire_size(int curve, uint32_t flags);
int pcgpu_g1_serialize(pcgpu_ctx *ctx, int curve, const void *xy, const uint8_t *inf, size_t n, uint32_t flags, uint8_t *out_bytes);
int pcgpu_g1_deserialize(pcgpu_ctx *ctx, int curve, const uint8_t *bytes, size_t n, uint32_t flags, void *out_xy, uint8_t *out_inf,
                         size_t *first_bad, int *reason);

/* ---- Fr vector work around the MSM (all elements Montgomery) ----------------------------------- */
/* F::into_bigint over a slice -- convert_to_bigints, kzg10/mod.rs:463-470 */
int pcgpu_fr_from_mont(pcgpu_ctx *ctx, int curve, const void *in, void *out, size_t n, uint32_t flags);
/* out[i] = a[i] * b[i] -- the randomizer * point / randomizer * value products of the verifier-side combinations,
 * kzg10/mod.rs:360-367 */
int pcgpu_fr_mul(pcgpu_ctx *ctx, int curve, const void *a, const void *b, void *out, size_t n, uint32_t flags);
/* y += c * x -- DensePolynomial AddAssign<(F, &P)>, marlin_pc/mod.rs:286; ipa_pc/mod.rs:691-697.  c: host, 1 element */
int pcgpu_fr_axpy(pcgpu_ctx *ctx, int curve, void *y, const void *c, const void *x, size_t n, uint32_t flags);
/* q = p / (X - z), rem = p(z) -- compute_witness_polynomial, kzg10/mod.rs:217-240.  p: n coefficients, q: n-1,
 * z and rem: host, 1 element each (rem may be NULL) */
int pcgpu_fr_div_linear(pcgpu_ctx *ctx, int curve, const void *p, size_t n, const void *z, void *q, void *rem,
                        uint32_t flags);
/* <a, b> -- utils.rs:150-155.  out: host, 1 element */
int pcgpu_fr_inner_product(pcgpu_ctx *ctx, int curve, const void *a, const void *b, size_t n, void *out, uint32_t flags);
/* out = v * M, M rows x cols row-major -- Matrix::row_mul, utils.rs:127-146.  When the columns alone cannot fill the device the
 * rows are cut into spans whose partial sums a second pass adds (the same row product as pcgpu_hyrax_open's). */
int pcgpu_fr_row_mul(pcgpu_ctx *ctx, int curve, const void *v, const void *m, size_t rows, size_t cols, void *out,
                     uint32_t flags);

/* ---- NTT ---------------------------------------------------------------------------------------- */
/* EvaluationDomain::fft(coeffs) on the radix-2 domain of size 2^logn -- linear_codes/utils.rs:119-126 (reed_solomon):
 * the n_in <= 2^logn input elements are zero-padded, out[j] = p(w^j) in natural order with
 * w = root_of_unity^(2^(two_adicity - logn)).  PCGPU_NTT_INVERSE computes ifft (coefficients from evaluations,
 * includes the 1/N factor).  1 <= logn <= 22.  out: 2^logn elements. */
int pcgpu_ntt(pcgpu_ctx *ctx, int curve, const void *in, size_t n_in, uint32_t logn, uint32_t flags, void *out);

/* `count` independent transforms: row r = in[r * n_in .. (r + 1) * n_in) zero-padded to 2^logn, out row stride 2^logn --
 * the row-wise Reed-Solomon encoding of LinearEncode::compute_matrices (linear_codes/mod.rs:118-138: every row of the
 * coefficient matrix through reed_solomon, linear_codes/utils.rs:112-127).  Rows up to 2^11 are one launch for the whole
 * matrix.  Same flags as pcgpu_ntt. */
int pcgpu_ntt_batch(pcgpu_ctx *ctx, int curve, const void *in, size_t n_in, size_t count, uint32_t logn, uint32_t flags, void *out);

/* Multi-GPU building block (SURVEY.md section 8e, "NTT shards by the four-step row/column split"): N = N1 * N2 with
 * N1 = 2^m1, N2 = 2^m2 from pcgpu_ntt_split (m2 = 0 means the transform is a single block pass and does not shard).
 * All pointers are DEVICE pointers.
 *   which = 1: columns n2 in [lo, lo+count) of the zero-padded input `in` (n_in elements, natural order)
 *              -> out[k1 * count + (n2 - lo)]   (N1 x count, step-2 twiddles applied)
 *   which = 2: rows k1 in [lo, lo+count) given as in[(k1 - lo) * N2 + n2] -> out[k2 * count + (k1 - lo)] = X[k1 + N1 k2]
 * Between the two passes the ranks exchange blocks with an all-to-all (poly_commit_b200.sharded.ShardedNtt). */
int pcgpu_ntt_split(uint32_t logn, uint32_t *m1, uint32_t *m2);
int pcgpu_ntt_pass(pcgpu_ctx *ctx, int curve, uint32_t logn, uint32_t flags, int which, size_t lo, size_t count,
                   const void *in, size_t n_in, void *out);

/* Pass 1 with the all-to-all fused into its stores: element k1 of column n2 is written straight into the row buffer of the
 * rank that owns row k1, dst[k1 / rows][(k1 % rows) * N2 + n2] with rows = N1 / world.  dst[0 .. world) are device pointers
 * valid on THIS device: the local row buffer and peer-mapped ones (cudaDeviceEnablePeerAccess / cudaIpcOpenMemHandle); each
 * holds rows * N2 elements.  After a barrier every rank runs pcgpu_ntt_pass(which = 2, lo = rank * rows, count = rows) on its
 * own buffer (pcgpu_peer_signal / pcgpu_peer_wait below are that barrier when the ranks are separate processes). */
int pcgpu_ntt_pass1_peer(pcgpu_ctx *ctx, int curve, uint32_t logn, uint32_t flags, size_t lo, size_t count, const void *in, size_t n_in,
                         void *const *dst, uint32_t world);

/* ---- linear-code commitments: column hashes + Merkle tree (SURVEY.md section 8f rank 4) ---------------------------------
 * LinearCodePCS::commit steps 2-3, linear_codes/mod.rs:253-275, for the hashers the reference's tests and benches
 * instantiate (linear_codes/{ligero,multilinear_ligero,brakedown}/tests.rs; bench-templates/src/lib.rs):
 *   column hash   FieldToBytesColHasher<F, D> (linear_codes/utils.rs:208-236): D(u64 LE length || n_rows canonical 32-byte
 *                 LE field elements), D = BLAKE2s-256 (PCGPU_HASH_BLAKE2S) or SHA-256 (PCGPU_HASH_SHA256)
 *   Merkle tree   Leaf = Vec<u8> with LeafIdentityHasher, TwoToOneHash = ark-crypto-primitives sha256 (SHA-256(left || right)),
 *                 ByteDigestConverter at the leaf level (each leaf digest is prefixed with its u64 length), leaves padded to
 *                 a power of two with empty leaves (create_merkle_tree, linear_codes/mod.rs:507-523)
 * pcgpu_lincode_hash_columns: ext_mat is n_rows x n_cols Montgomery Fr, row-major (Matrix<F>, utils.rs:49-53); out_leaves
 *   receives n_cols x 32 bytes.  The matrix is read in place (one thread per column, rows coalesced across the warp).
 * pcgpu_merkle_tree: n_leaves >= 2 digests of 32 bytes -> the P - 1 inner nodes (P = next power of two) in heap order
 *   (node 0 = root, children of i are 2i+1, 2i+2 -- MerkleTree::non_leaf_nodes) and the 32-byte root (host pointer).
 * pcgpu_lincode_commit: the whole commit of one polynomial matrix without leaving the device: every row of `mat`
 *   (n_rows x n_cols) through reed_solomon to 2^log_ext_cols evaluations (compute_matrices, linear_codes/mod.rs:118-138),
 *   column hashes, tree.  out_ext_mat (n_rows x 2^log_ext_cols), out_leaves, out_nodes may be NULL; out_root: host.
 * With PCGPU_DEVICE_PTRS the matrix / leaves / nodes arguments are device pointers. */
enum { PCGPU_HASH_BLAKE2S = 0, PCGPU_HASH_SHA256 = 1 };
int pcgpu_lincode_hash_columns(pcgpu_ctx *ctx, int curve, const void *ext_mat, size_t n_rows, size_t n_cols, int hash, uint32_t flags,
                               uint8_t *out_leaves);
int pcgpu_merkle_tree(pcgpu_ctx *ctx, const uint8_t *leaves, size_t n_leaves, uint32_t flags, uint8_t *out_nodes, uint8_t *out_root);
int pcgpu_lincode_commit(pcgpu_ctx *ctx, int curve, const void *mat, size_t n_rows, size_t n_cols, uint32_t log_ext_cols, int hash,
                         uint32_t flags, void *out_ext_mat, uint8_t *out_leaves, uint8_t *out_nodes, uint8_t *out_root);

/* ---- Brakedown (MultilinearBrakedown, linear_codes/brakedown.rs + multilinear_brakedown/mod.rs) ------------------------
 * pcgpu_brakedown_register: the code of a BrakedownPCParams (brakedown.rs:146-203), uploaded once: m message columns,
 *   m_ext codeword columns, `levels` L, a_dims / b_dims as L (rows, cols, nonzeros per row) triples each, and 2L CSC matrices
 *   A_0..A_{L-1}, B_0..B_{L-1} exactly as SprsMat stores them (linear_codes/utils.rs:20-107): ind_ptr[cols + 1] and
 *   col_ind[ind_ptr[cols]] u64, val[ind_ptr[cols]] Montgomery Fr.  The matrices come from the caller's RNG (make_mat,
 *   brakedown.rs:305-333), so they are data here, like an SRS.  Checked on the host: PCGPU_E_BADARG when a_dims[0].0 != m,
 *   a_dims[i].1 != a_dims[i+1].0, b_dims[i].0 != end[i] - start[i], m_ext != codeword_len (brakedown.rs:292-299; with L = 0,
 *   m_ext < m), the Reed-Solomon output is shorter than its input, an ind_ptr does not start at 0, is not monotone or exceeds
 *   rows * nonzeros, or a col_ind >= rows; PCGPU_E_RANGE when a value is not a reduced field element.  At most 16 levels.
 * pcgpu_brakedown_encode: MultilinearBrakedown::encode (multilinear_brakedown/mod.rs:56-84) of every row of `mat`
 *   (n_rows x n_cols, row-major) -> out_ext (n_rows x m_ext, row-major, compute_matrices' ext_mat).  n_cols != m:
 *   PCGPU_E_LEN (Error::EncodingError).
 * pcgpu_brakedown_commit: encode + column hashes + Merkle tree without leaving the device, like pcgpu_lincode_commit (the tree
 *   pads m_ext leaves to a power of two with empty leaves); out_ext, out_leaves (m_ext x 32) and out_nodes may be NULL.
 * pcgpu_fr_sprs_row_mul: SprsMat::row_mul (utils.rs:41-52) of an n x m CSC matrix on `count` vectors (count x n, row-major)
 *   -> out (count x m).  The matrix arrays are host pointers (checked as above, without a nonzero bound).
 * With PCGPU_DEVICE_PTRS the matrix / vector / output arguments (not the CSC arrays) are device pointers.  Profile stage 15 is
 * the encoding; the hashes and the tree are stage 14. */
typedef struct pcgpu_brakedown pcgpu_brakedown;
int pcgpu_brakedown_register(pcgpu_ctx *ctx, int curve, size_t m, size_t m_ext, size_t levels, const uint64_t *a_dims,
                             const uint64_t *b_dims, const uint64_t *const *ind_ptr, const uint64_t *const *col_ind,
                             const void *const *val, uint32_t flags, pcgpu_brakedown **out);
void pcgpu_brakedown_release(pcgpu_ctx *ctx, pcgpu_brakedown *code);
int pcgpu_brakedown_encode(pcgpu_ctx *ctx, const pcgpu_brakedown *code, const void *mat, size_t n_rows, size_t n_cols, uint32_t flags,
                           void *out_ext);
int pcgpu_brakedown_commit(pcgpu_ctx *ctx, const pcgpu_brakedown *code, const void *mat, size_t n_rows, size_t n_cols, int hash,
                           uint32_t flags, void *out_ext, uint8_t *out_leaves, uint8_t *out_nodes, uint8_t *out_root);
int pcgpu_fr_sprs_row_mul(pcgpu_ctx *ctx, int curve, size_t n, size_t m, const uint64_t *ind_ptr, const uint64_t *col_ind,
                          const void *val, const void *v, size_t count, uint32_t flags, void *out);

/* ---- multi-GPU over NVLink peer memory (SURVEY.md section 8e) -------------------------------------------------------
 * One process per GPU.  Every rank allocates ONE window (pcgpu_peer_window_bytes() bytes, zero-filled) with pcgpu_peer_alloc,
 * the ranks exchange the 64-byte handles out of band (torch.distributed all_gather in poly_commit_b200.sharded.PeerGroup;
 * MPI / a socket in a Rust host) and map each other's windows with pcgpu_peer_open (cudaIpcOpenMemHandle; NVLink P2P).
 * win[0 .. world) below are the window pointers valid in THIS process: win[rank] is the local allocation, the others are
 * the mapped peers.  Epochs are caller-chosen, strictly increasing per channel (flags are never reset).
 *
 * pcgpu_msm_peer: "MSM shards by scalar/base pair across the GPUs with a final point-sum over NVLink" (BASELINE.json
 *   north_star; the reference computes the same sum in one msm_bigint call, kzg10/mod.rs:175-178): every rank calls it with
 *   ITS slice of the scalars and an SRS holding ITS slice of the bases; the last kernel of the rank's Pippenger pipeline
 *   stores the rank's bit-plane sums (~3 KB) into slot [rank] of every peer's window and raises a flag, a bounded spin on
 *   the local window's flags follows on the same stream, and one device-to-host copy returns all records: every rank
 *   obtains the full sum, affine, with no collective call.  flags: PCGPU_SCALARS_MONT, PCGPU_DEVICE_PTRS (scalars).
 * pcgpu_peer_signal / pcgpu_peer_wait: raise flag [rank] of `channel` (0..7; channel 0 is used by pcgpu_msm_peer) in every
 *   window / wait (bounded, PCGPU_E_PEER on expiry) until every flag of the local window reached `epoch` -- the barrier
 *   between pcgpu_ntt_pass1_peer and pass 2 of the sharded NTT. */
#define PCGPU_IPC_HANDLE_BYTES 64
size_t pcgpu_peer_window_bytes(void);
int pcgpu_peer_alloc(pcgpu_ctx *ctx, size_t bytes, void **out_ptr, uint8_t *handle /* PCGPU_IPC_HANDLE_BYTES */);
int pcgpu_peer_open(pcgpu_ctx *ctx, const uint8_t *handle, void **out_ptr);
int pcgpu_peer_close(pcgpu_ctx *ctx, void *mapped_ptr);
int pcgpu_peer_free(pcgpu_ctx *ctx, void *ptr);
int pcgpu_peer_signal(pcgpu_ctx *ctx, void *const *win, uint32_t rank, uint32_t world, uint32_t channel, uint64_t epoch);
int pcgpu_peer_wait(pcgpu_ctx *ctx, void *local_win, uint32_t world, uint32_t channel, uint64_t epoch);
int pcgpu_msm_peer(pcgpu_ctx *ctx, const pcgpu_srs *srs, size_t base_offset, const void *scalars, size_t n, uint32_t flags,
                   void *const *win, uint32_t rank, uint32_t world, uint64_t epoch, void *out_xy, uint8_t *out_inf);

/* ---- InnerProductArgPC::open halving loop, device-resident (ipa_pc/mod.rs:636-711) ------------------------- */
typedef struct pcgpu_ipa pcgpu_ipa;
/* Upload the committer key (n = d+1 affine points, n a power of two) and the combined polynomial's coefficients
 * (n_coeffs <= n Montgomery Fr, zero-padded :636-641); build z = [1, point, point^2, ...] on the device (:643-648).
 * One open at a time per context: PCGPU_E_BADARG while another open begun on ctx is not finished.  The state belongs to
 * ctx: pcgpu_ipa_round_lr, pcgpu_ipa_round_fold and pcgpu_ipa_finish return PCGPU_E_BADARG for any other context and
 * leave the state as it was (a rejected finish does not release it). */
int pcgpu_ipa_begin(pcgpu_ctx *ctx, int curve, const void *comm_key_xy, size_t n, const void *coeffs, size_t n_coeffs,
                    const void *point, uint32_t flags, pcgpu_ipa **out);
/* One round, first half (:671-677): l = cm_commit(key_l, coeffs_r) + h' * <coeffs_r, z_l>,
 * r = cm_commit(key_r, coeffs_l) + h' * <coeffs_l, z_r>, normalised.  h_prime_xy: affine h' (host). */
int pcgpu_ipa_round_lr(pcgpu_ctx *ctx, pcgpu_ipa *st, const void *h_prime_xy, void *out_l_xy, uint8_t *out_l_inf,
                       void *out_r_xy, uint8_t *out_r_inf);
/* One round, second half (:691-708): fold coeffs, z and the key with the round challenge (Montgomery Fr, and its
 * inverse), then halve n. */
int pcgpu_ipa_round_fold(pcgpu_ctx *ctx, pcgpu_ipa *st, const void *challenge, const void *challenge_inv);
/* Current size (1 when the loop is over). */
size_t pcgpu_ipa_len(const pcgpu_ipa *st);
/* final_comm_key = comm_key[0], c = coeffs[0] (:713-720); releases the state. */
int pcgpu_ipa_finish(pcgpu_ctx *ctx, pcgpu_ipa *st, void *out_final_key_xy, void *out_c);

/* The linear-time step of InnerProductArgPC::check (ipa_pc/mod.rs:760-766): check_poly.compute_coeffs()
 * (data_structures.rs:204-220; coeffs[idx] = product of challenges[i] over the set bits of idx, challenges[0] on the top
 * bit) followed by cm_commit(comm_key, coeffs).  challenges: log_d Montgomery Fr (host); comm_key: >= 2^log_d bases.
 * The caller compares the result with proof.final_comm_key. */
int pcgpu_ipa_check_final_key(pcgpu_ctx *ctx, const pcgpu_srs *comm_key, const void *challenges, uint32_t log_d,
                              void *out_xy, uint8_t *out_inf);

/* ---- MultilinearPC (XZZPD19, multilinear_pc/mod.rs) prover -----------------------------------------------------------
 * pcgpu_mlpc_register: the G2 half of a CommitterKey (after trim, :91-111).  curve: PCGPU_BLS12_381 or PCGPU_BN254.  Level i
 *   = 0 .. nv-1 is powers_of_h[i], 2^(nv-i) G2 affine points, with inf[i] its infinity bytes (inf or inf[i] may be NULL).  The
 *   key stores the pair-folded bases H'_i[b] = H_i[2b] + H_i[2b+1], one device G2 addition per pair, so that an open runs
 *   2^nv - 1 G2 terms; this holds for any key, honestly generated or not.  With PCGPU_DEVICE_PTRS the level arrays are
 *   device pointers.  1 <= nv <= 25.
 * pcgpu_mlpc_open: MultilinearPC::open (:131-168).  evals: the 2^nv Montgomery Fr values of the polynomial in
 *   to_evaluations() order (PCGPU_DEVICE_PTRS: a device pointer); point: nv Montgomery Fr (host).  The fold chain
 *   q_i[b] = r[2b+1] - r[2b], r'[b] = r[2b] (1 - point[i]) + r[2b+1] point[i] runs on the device (profile stage 16), then
 *   proof i = sum_b q_i[b] H'_i[b].  out_proofs_xy: nv G2 affine points, out_proofs_inf: nv bytes (may be NULL),
 *   out_value (may be NULL): the last r, which is p(point), Montgomery Fr.  n != 2^nv: PCGPU_E_LEN ("Invalid size of
 *   polynomial", :136).
 * The commitment (:114-128) is pcgpu_msm with PCGPU_SCALARS_MONT over a G1 key of powers_of_g[0]. */
typedef struct pcgpu_mlpc pcgpu_mlpc;
int pcgpu_mlpc_register(pcgpu_ctx *ctx, int curve, uint32_t nv, const void *const *powers_of_h, const uint8_t *const *inf,
                        uint32_t flags, pcgpu_mlpc **out);
void pcgpu_mlpc_release(pcgpu_ctx *ctx, pcgpu_mlpc *key);
int pcgpu_mlpc_open(pcgpu_ctx *ctx, const pcgpu_mlpc *key, const void *evals, size_t n, const void *point, uint32_t flags,
                    void *out_proofs_xy, uint8_t *out_proofs_inf, void *out_value);

/* ---- HyraxPC (hyrax/mod.rs) -----------------------------------------------------------------------------------------------
 * dim = 2^(nv / 2).  Every Fr is Montgomery.  The key (ck / vk) is com_key || h registered with PCGPU_SRS_COMB, dim + 1 bases.
 * The sponge and the RNG stay with the caller: randomness is an input in the order the reference draws it, challenges in the
 * order its sponge squeezes them, so the same streams give the reference's proofs byte for byte.
 * Errors: an odd nv (InvalidNumberOfVariables), a key without comb tables, a key or state of another curve, unknown flags:
 * PCGPU_E_BADARG; a key that does not hold dim + 1 bases (pedersen_commit's assert_eq) or a state whose nv differs from the
 * point's (MismatchedNumVars): PCGPU_E_LEN; an input Fr not below r: PCGPU_E_RANGE.  nv = 0 (dim = 1, l = r = [1]) is valid.
 * Flags: PCGPU_DEVICE_PTRS makes the arguments each call names device pointers; every other argument is a host pointer.
 * Profile stage 19 (transpose, tensors, row product, inner products); the comb rows are stage 10, the small MSMs stage 4.
 *
 * pcgpu_hyrax_commit: HyraxPC::commit of one polynomial (:213-252).  evals: 2^nv elements in to_evaluations() order;
 *   randomness: dim elements, r_i of row i.  The device transposes evals into the dim x (dim + 1) block [T | r]
 *   (flat_to_matrix_column_major, utils.rs:13-21) and commits to every row over the key: out_row_coms_xy / _inf receive dim
 *   points (inf may be NULL).  The block stays on the device in *out, the HyraxCommitmentState.  PCGPU_DEVICE_PTRS: evals and
 *   randomness.
 * pcgpu_hyrax_release: frees a state once the context's stream is idle.
 * pcgpu_hyrax_open: everything HyraxPC::open (:273-406) computes before the challenge, for `count` states at one point
 *   (point: nv elements).  blinds: per polynomial r_eval || d (dim) || r_d || r_b, the reference's draw order (:360, :367-368,
 *   :373, :377).  With l, r the tensors of the reversed, split point (:299-307), [lt | r_lt] = l^T [T | r], eval = <lt, r>,
 *   b = <r, d>, and com_eval = [eval, 0.., r_eval], com_d = [d | r_d], com_b = [b, 0.., r_b] as comb rows over the key.
 *   out_coms_xy / _inf: 3 * count points, per polynomial com_eval, com_d, com_b (the sponge's absorb order; inf may be NULL);
 *   out_lt: per polynomial lt || r_lt (dim + 1 elements); out_eval: count elements or NULL.  The caller squeezes c and finishes
 *   with pcgpu_fr_axpy: z = d + c lt; then z_d = c r_lt + r_d and z_b = c r_eval + r_b.  PCGPU_DEVICE_PTRS: blinds and out_lt.
 * pcgpu_hyrax_check: HyraxPC::check (:418-511) of `count` proofs at one point.  row_coms: count x dim points (inf may be NULL);
 *   proof_xy / proof_inf: count x 3 points com_eval, com_d, com_b (inf may be NULL); proof_scalars: count x (dim + 2) elements
 *   z || z_d || z_b; challenges: count elements.  out_ok[j] = 1 exactly when both of the reference's equations hold for proof j,
 *   each side compared as affine bytes with its infinity flag: (14) com_key[0] <r, z> + h z_b == c com_eval + com_b and
 *   (13) pedersen(z) + h z_d == c t_prime + com_d, t_prime = msm(row_coms, l).  The reference's answer is the AND of out_ok.
 *   Returns PCGPU_OK whether or not the proofs verify.  PCGPU_DEVICE_PTRS: row_coms_xy, row_coms_inf and proof_scalars. */
typedef struct pcgpu_hyrax pcgpu_hyrax;
int pcgpu_hyrax_commit(pcgpu_ctx *ctx, const pcgpu_srs *ck, uint32_t nv, const void *evals, const void *randomness, uint32_t flags,
                       void *out_row_coms_xy, uint8_t *out_row_coms_inf, pcgpu_hyrax **out);
void pcgpu_hyrax_release(pcgpu_ctx *ctx, pcgpu_hyrax *state);
int pcgpu_hyrax_open(pcgpu_ctx *ctx, const pcgpu_srs *ck, const pcgpu_hyrax *const *states, size_t count, uint32_t nv,
                     const void *point, const void *blinds, uint32_t flags, void *out_coms_xy, uint8_t *out_coms_inf, void *out_lt,
                     void *out_eval);
int pcgpu_hyrax_check(pcgpu_ctx *ctx, const pcgpu_srs *vk, uint32_t nv, size_t count, const void *row_coms_xy,
                      const uint8_t *row_coms_inf, const void *point, const void *proof_xy, const uint8_t *proof_inf,
                      const void *proof_scalars, const void *challenges, uint32_t flags, uint8_t *out_ok);

/* ---- pairing (verifiers) ----------------------------------------------------------------------------------------------
 * E::multi_pairing(a, b) for `count` independent equations of k pairs each: equation j is
 * prod_{i<k} e(P[j*k+i], Q[j*k+i]) (kzg10/mod.rs:326-330, :382-387; multilinear_pc/mod.rs:179-199; sonic_pc/mod.rs:128), the
 * optimal-ate pairing with the exact final exponentiation (p^12 - 1) / r.  curve: PCGPU_BLS12_381 or PCGPU_BN254 (any other
 * id, G2 ids included: PCGPU_E_BADARG).
 *   g1_xy: count * k G1 affine points (x || y); g2_xy: count * k G2 affine points (x.c0 x.c1 y.c0 y.c1); g1_inf / g2_inf: their
 *   identity bytes, either may be NULL.  A pair with an identity on either side contributes 1.  With PCGPU_DEVICE_PTRS the
 *   four input arrays are device pointers; the outputs are host arrays.
 *   out_gt: count Fq12 elements, 12 Fq coefficients each in ark's order (c0.c0.c0, c0.c0.c1, c0.c1.c0 ... c1.c2.c1), each
 *   `limbs` u64 Montgomery (tower Fq6 = Fq2[v]/(v^3 - xi), Fq12 = Fq6[w]/(w^2 - v), xi = 1 + u on BLS12-381, 9 + u on
 *   BN254); out_is_one: count bytes, 1 where the equation's product is one.  Either output may be NULL, not both.
 *   k == 0 gives the identity (ark's empty multi_pairing); k > PCGPU_PAIRING_MAX_K: PCGPU_E_BADARG; count == 0 is a no-op.
 * Points are NOT validated (on the curve, in the subgroup), as G1Prepared::from / G2Prepared::from do not validate either:
 * pass points decoded with validation.  Profile stage 17.  One equation is a serial chain in one thread; the device pays off
 * with many equations per call. */
#define PCGPU_PAIRING_MAX_K 64
int pcgpu_multi_pairing(pcgpu_ctx *ctx, int curve, const void *g1_xy, const uint8_t *g1_inf, const void *g2_xy,
                        const uint8_t *g2_inf, size_t k, size_t count, uint32_t flags, void *out_gt, uint8_t *out_is_one);

/* Prepared G2 points (ark's G2Prepared): the Miller loop's line coefficients of n fixed G2 points, computed once and kept on
 * the device, so pairings against them skip the twist arithmetic -- a verifier key's h, beta_h and degree-bound powers.
 *   pcgpu_g2_prepare: curve PCGPU_BLS12_381 or PCGPU_BN254 (any other id, G2 ids included: PCGPU_E_BADARG); g2_xy: n G2
 *   affine points (x.c0 x.c1 y.c0 y.c1), g2_inf: their identity bytes or NULL (an identity, or the all-zero encoding, makes
 *   its pairs contribute 1); with PCGPU_DEVICE_PTRS both are device pointers.  Points are NOT validated, as in
 *   G2Prepared::from.  About 19 KB of lines per point (68 lines on BLS12-381, 100 on BN254).  *out is cleared whenever out is non-null.
 *   Profile stage 18.
 *   pcgpu_multi_pairing_prepared: pcgpu_multi_pairing with equation j = prod_{i<k} e(P[j*k+i], Q[q_index[j*k+i]]) over the
 *   handle's points.  g1_xy / g1_inf as in pcgpu_multi_pairing (device pointers with PCGPU_DEVICE_PTRS); q_index: k * count
 *   indices, a host array in every mode, checked before anything runs (an index >= n: PCGPU_E_BADARG).  A handle prepared on
 *   another curve: PCGPU_E_BADARG.  Outputs, k == 0, count == 0 and PCGPU_PAIRING_MAX_K as in pcgpu_multi_pairing; profile
 *   stage 17. */
typedef struct pcgpu_g2_prepared pcgpu_g2_prepared;
int pcgpu_g2_prepare(pcgpu_ctx *ctx, int curve, const void *g2_xy, const uint8_t *g2_inf, size_t n, uint32_t flags,
                     pcgpu_g2_prepared **out);
void pcgpu_g2_prepared_release(pcgpu_ctx *ctx, pcgpu_g2_prepared *q);
int pcgpu_multi_pairing_prepared(pcgpu_ctx *ctx, int curve, const void *g1_xy, const uint8_t *g1_inf, const pcgpu_g2_prepared *q,
                                 const uint32_t *q_index, size_t k, size_t count, uint32_t flags, void *out_gt,
                                 uint8_t *out_is_one);

/* ---- KZG10 fused prover calls ------------------------------------------------------------------ */
/* KZG10::commit -- kzg10/mod.rs:157-210.  coeffs: n Montgomery Fr (low degree first; trailing zeros allowed and
 * ignored like DensePolynomial's truncation).  Hiding: pass gamma (powers_of_gamma_g) and n_blind > 0 blinding
 * coefficients (the reference samples them from its RNG, :182-195; here they are an input so results are
 * reproducible); gamma may be NULL when n_blind == 0.  Errors: PCGPU_E_DEGREE, PCGPU_E_HIDING. */
int pcgpu_kzg_commit(pcgpu_ctx *ctx, const pcgpu_srs *powers_of_g, const void *coeffs, size_t n,
                     const pcgpu_srs *powers_of_gamma_g, const void *blind, size_t n_blind, uint32_t flags,
                     void *out_xy, uint8_t *out_inf);
/* MarlinKZG10::commit's per-polynomial loop (marlin_pc/mod.rs:192-241) in one call: `count` independent non-hiding
 * KZG10 commitments over the same powers.  coeffs[i] points at n[i] Montgomery Fr coefficients; out_xy receives count
 * affine points, out_inf count flags.  Polynomials are processed `PCGPU_BATCH_WAYS` (4) at a time on sibling
 * contexts (own stream + workspace each) so that the latency-bound stages of one MSM overlap the multiply-bound stages
 * of another -- what the reference's serial loop leaves on the table.  BASELINE.json cfg5 = 64 such polynomials spread
 * over 8 GPUs (poly_commit_b200.sharded.poly_assignment). */
int pcgpu_kzg_commit_batch(pcgpu_ctx *ctx, const pcgpu_srs *powers_of_g, const void *const *coeffs, const size_t *n,
                           size_t count, uint32_t flags, void *out_xy, uint8_t *out_inf);
/* KZG10::open -- kzg10/mod.rs:287-310 (compute_witness_polynomial :217-240 then open_with_witness_polynomial
 * :243-284): witness = p / (X - z) on the device, then the MSM over the witness.  out_random_v (may be NULL)
 * receives blind(z) when n_blind > 0 (:264). */
int pcgpu_kzg_open(pcgpu_ctx *ctx, const pcgpu_srs *powers_of_g, const void *coeffs, size_t n, const void *z,
                   const pcgpu_srs *powers_of_gamma_g, const void *blind, size_t n_blind, uint32_t flags,
                   void *out_w_xy, uint8_t *out_w_inf, void *out_random_v);

/* KZG10::commit followed by KZG10::open of the same polynomial at z -- what a Marlin prover does per polynomial
 * (MarlinKZG10::commit, marlin_pc/mod.rs:192-241, then ::open, :245-336) -- as ONE call: the coefficients are uploaded once,
 * the commitment MSM (kzg10/mod.rs:175-178) and the witness division + MSM (:222-226, :255-258) run concurrently on two
 * streams of the same device.  Non-hiding path (hiding_bound = None, the benchmark protocol of bench-templates/src/lib.rs:79);
 * with blinding polynomials call pcgpu_kzg_commit and pcgpu_kzg_open.  flags: PCGPU_DEVICE_PTRS (coeffs).
 * pcgpu_kzg_commit_open_batch: `count` polynomials opened at the same point z (the query set of one Marlin opening), two
 * polynomials in flight; coeffs[i] / n[i] as in pcgpu_kzg_commit_batch, outputs are `count` points / flags each. */
int pcgpu_kzg_commit_open(pcgpu_ctx *ctx, const pcgpu_srs *powers_of_g, const void *coeffs, size_t n, const void *z, uint32_t flags,
                          void *out_comm_xy, uint8_t *out_comm_inf, void *out_w_xy, uint8_t *out_w_inf);
int pcgpu_kzg_commit_open_batch(pcgpu_ctx *ctx, const pcgpu_srs *powers_of_g, const void *const *coeffs, const size_t *n, size_t count,
                                const void *z, uint32_t flags, void *out_comm_xy, uint8_t *out_comm_inf, void *out_w_xy,
                                uint8_t *out_w_inf);

/* ---- device buffers ------------------------------------------------------------------------------------------------------
 * For callers that keep polynomials on the GPU across calls: the accumulators of MarlinKZG10::open (p, r, shifted_w,
 * shifted_r: `p += (challenge_j, polynomial)`, marlin_pc/mod.rs:286-307) live in such buffers, so every polynomial crosses
 * PCIe once and the combined polynomial never does.  The pointers are plain device pointers: pass them to any entry point
 * together with PCGPU_DEVICE_PTRS (offsets are byte arithmetic on the pointer).  alloc zero-fills. */
int pcgpu_buf_alloc(pcgpu_ctx *ctx, size_t bytes, void **out);
int pcgpu_buf_free(pcgpu_ctx *ctx, void *buf);
int pcgpu_buf_write(pcgpu_ctx *ctx, void *dst, size_t dst_offset, const void *src_host, size_t bytes);
int pcgpu_buf_read(pcgpu_ctx *ctx, const void *src, size_t src_offset, void *dst_host, size_t bytes);
int pcgpu_buf_zero(pcgpu_ctx *ctx, void *dst, size_t dst_offset, size_t bytes);

/* ---- diagnostics -------------------------------------------------------------------------------- */
/* Device self-test of the field layer: n pseudo-random pairs per field (Fq and Fr of `curve`), production
 * multiplier (carry-chained mad.lo/mad.hi schedule) against the plain 64-bit-accumulate multiplier compiled into
 * the same kernel, plus a*a^-1 == 1 on a few elements.  *mismatches receives the number of disagreeing results. */
/* Measures the chip's sustained 32x32+64 -> 64-bit integer multiply-add rate (IMAD.WIDE.U32, the instruction every field
 * multiplication is made of) with a register-resident dependent-chain kernel at full occupancy; *ops_per_s receives
 * multiply-adds per second.  bench.py divides the MSM kernels' multiply counts by it (the compute roofline that actually
 * binds them; the HBM roofline north_star asks for is reported next to it). */
int pcgpu_measure_imad_peak(pcgpu_ctx *ctx, double *ops_per_s);
/* Kernels launched by this library in the calling process so far (bench.py's gpu_launches). */
uint64_t pcgpu_launch_count(void);
int pcgpu_selftest_field(pcgpu_ctx *ctx, int curve, uint64_t seed, size_t n, uint64_t *mismatches);
/* The path and geometry the context's most recent MSM took, each value taken from the MSM's plan.  Writes
 * min(len, PCGPU_GEOM_FIELDS) words: out[PCGPU_GEOM_PATH] is PCGPU_MSM_PATH_NONE (n = 0, or no MSM yet), _SMALL (one-launch
 * kernel; out[PCGPU_GEOM_SPLIT] = blocks per window: 1, 3 or 6) or _BUCKETS (the bucket pipeline: window bits c, windows W,
 * table groups G (1 = raw bases), batched-affine rounds R, the pair-round kernel's threads T and its divisor tdiv, the one
 * resident wave of that kernel the round count was chosen against, entries = n * W, and the number of buckets reduced by
 * the heavy-bucket kernel, or UINT64_MAX where the pipeline's tail did not report it) or _COMB (pcgpu_msm_batch over
 * PCGPU_SRS_COMB tables: n = the row length, c = the comb window bits, W windows, split = the segment length each row is
 * cut into, entries = count * segments, the number of accumulate tasks).  A pcgpu_msm_batch without comb tables runs its
 * rows through pcgpu_msm, so it reports the last row's MSM.  Unused fields are 0. */
enum {
  PCGPU_GEOM_PATH = 0, PCGPU_GEOM_SPLIT = 1, PCGPU_GEOM_N = 2, PCGPU_GEOM_C = 3, PCGPU_GEOM_W = 4, PCGPU_GEOM_G = 5,
  PCGPU_GEOM_R = 6, PCGPU_GEOM_T = 7, PCGPU_GEOM_TDIV = 8, PCGPU_GEOM_WAVE = 9, PCGPU_GEOM_ENTRIES = 10,
  PCGPU_GEOM_HEAVY = 11, PCGPU_GEOM_FIELDS = 12
};
enum { PCGPU_MSM_PATH_NONE = 0, PCGPU_MSM_PATH_SMALL = 1, PCGPU_MSM_PATH_BUCKETS = 2, PCGPU_MSM_PATH_COMB = 3 };
int pcgpu_msm_last_geometry(pcgpu_ctx *ctx, uint64_t *out, size_t len);
/* One field primitive applied elementwise on the device (the same code the kernels use), for testing the field layer
 * against plain integers: which = 0 the base field Fq of `curve`, 1 its scalar field Fr, 2 its quadratic extension Fq2
 * (pairing curves only; elements c0 || c1; ops 0, 2, 3, 4, 5 (through the norm) and 9 (a^2)), 3 the pairing's Fq12 (pairing
 * curves only; elements in pcgpu_multi_pairing's GT layout; ops 0, 2, 3, 4, 5, 9, 10 and 11).  a, b, out: host arrays of n
 * elements, little-endian 32-bit limbs (Fq of BLS12-381: 12 limbs, every other field 8), Montgomery form.  op:
 *   0 mont_mul(a, b)   1 mont_mul_ref(a, b) (plain 64-bit accumulate)   2 a + b   3 a - b   4 -a   5 a^-1 (Fermat)
 *   6 mont_mul2(a, b, b, -a) (= 0)   7 mont_mul2(a, b, a + b, b - a)   8 a^-1 (binary GCD)   9 mont_sqr(a)
 *   10 a^p (Frobenius, Fq12 only)   11 a^((p^12 - 1) / r) (the final exponentiation, Fq12 only)
 * Ops 6 and 7 fall back to two products on a field without mont_mul2; inverses of 0 are 0. */
int pcgpu_diag_field_op(pcgpu_ctx *ctx, int curve, int which, int op, const void *a, const void *b, void *out, size_t n);

#ifdef __cplusplus
}
#endif
#endif /* PCGPU_H */
