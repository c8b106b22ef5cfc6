// TEST HARNESS ONLY: exposes individual device functions (compiled for the host with emulated
// carry flags) so tests can compare the production limb schedule against the 64-bit reference
// multiplier and the Python big-integer oracle.
#include <stddef.h>
#include <vector>
#include "../../poly-commit_b200/csrc/field_ops.cuh"
using namespace pcgpu;

template <class P>
static const uint32_t *pow2_table() {
  static std::vector<uint32_t> t;
  if (t.empty()) { t.resize(pow2_table_bytes<P>() / 4); Pow2TableBody<P>{t.data()}(0); }
  return t.data();
}

// the op switch is FieldOpBody (csrc/field_ops.cuh), the body pcgpu_diag_field_op launches on the device
template <class P>
static void mul_many(const uint32_t *a, const uint32_t *b, uint32_t *out, size_t n, int which) {
  const FieldOpBody<P> body{a, b, out, pow2_table<P>(), which};
  for (size_t i = 0; i < n; i++) body(i);
}

// field: 0 bls Fq, 1 bls Fr, 2 bn Fq, 3 bn Fr, 4 pallas Fq, 5 pallas Fr
extern "C" int hostcheck_field_op(int field, int which, const uint32_t *a, const uint32_t *b, uint32_t *out, size_t n) {
  switch (field) {
    case 0: mul_many<Bls12381Fq>(a, b, out, n, which); break;
    case 1: mul_many<Bls12381Fr>(a, b, out, n, which); break;
    case 2: mul_many<Bn254Fq>(a, b, out, n, which); break;
    case 3: mul_many<Bn254Fr>(a, b, out, n, which); break;
    case 4: mul_many<PallasFq>(a, b, out, n, which); break;
    case 5: mul_many<PallasFr>(a, b, out, n, which); break;
    default: return -1;
  }
  return 0;
}

// GLV split of one canonical scalar (host_glv.hpp): curve 1 = BN254, 2 = Pallas.  out: k1[5], k2[5], neg1, neg2, nbits, ok, jsf_len, u1_nz[5], u1_sg[5], u2_nz[5], u2_sg[5]
#include "../../poly-commit_b200/csrc/host_glv.hpp"
extern "C" int hostcheck_glv(int curve, const uint64_t *k, uint32_t *out) {
  host::GlvSplit g;
  if (curve == 1) g = host::glv_decompose<Bn254>(k);
  else if (curve == 2) g = host::glv_decompose<Pallas>(k);
  else return -1;
  for (int i = 0; i < 5; i++) { out[i] = g.k1[i]; out[5 + i] = g.k2[i]; }
  out[10] = g.neg1; out[11] = g.neg2; out[12] = g.nbits; out[13] = g.ok ? 1 : 0;
  out[14] = g.jsf_len;   // joint sparse form of (|k1|, |k2|): non-zero / sign masks of the two digit strings
  for (int i = 0; i < 5; i++) { out[15 + i] = g.u1_nz[i]; out[20 + i] = g.u1_sg[i]; out[25 + i] = g.u2_nz[i]; out[30 + i] = g.u2_sg[i]; }
  return 0;
}

// host_ec.hpp's 64-bit Montgomery product (the MSM tail's arithmetic): out[i] = a[i] * b[i] / R, n elements of N64 limbs.
// field ids as in hostcheck_field_op.
template <class P>
static void host_mul_many(const uint64_t *a, const uint64_t *b, uint64_t *out, size_t n) {
  constexpr int N = host::HFp<P>::N;
  for (size_t i = 0; i < n; i++) {
    host::HFp<P> x, y;
    memcpy(x.l, a + i * N, sizeof x.l); memcpy(y.l, b + i * N, sizeof y.l);
    host::HFp<P> r = host::mul<P>(x, y);
    memcpy(out + i * N, r.l, sizeof r.l);
  }
}
extern "C" int hostcheck_hostfield_mul(int field, const uint64_t *a, const uint64_t *b, uint64_t *out, size_t n) {
  switch (field) {
    case 0: host_mul_many<Bls12381Fq>(a, b, out, n); return 0;
    case 1: host_mul_many<Bls12381Fr>(a, b, out, n); return 0;
    case 2: host_mul_many<Bn254Fq>(a, b, out, n); return 0;
    case 3: host_mul_many<Bn254Fr>(a, b, out, n); return 0;
    case 4: host_mul_many<PallasFq>(a, b, out, n); return 0;
    case 5: host_mul_many<PallasFr>(a, b, out, n); return 0;
    default: return -1;
  }
}
