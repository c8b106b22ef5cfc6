/* Test oracle: MultilinearBrakedown::encode (poly-commit multilinear_brakedown/mod.rs:56-84) restated literally in portable C
 * over all rows of a matrix (OpenMP over rows), so that full-size device encodes can be checked in seconds.  Independent of
 * the library: 64-bit-limb CIOS Montgomery arithmetic with __int128, the modulus passed in at run time.  Elements are
 * Montgomery form, 4 little-endian u64 limbs, modulus < 2^255.  `deep_first` runs the B levels deepest first instead of the
 * reference's ascending order (used only to show that a test can tell the two apart). */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef unsigned __int128 u128;
typedef struct { uint64_t l[4]; } fe;

static int geq(const uint64_t *a, const uint64_t *p) {
  for (int i = 3; i >= 0; i--) if (a[i] != p[i]) return a[i] > p[i];
  return 1;
}
static void sub_p(uint64_t *a, const uint64_t *p) {
  uint64_t br = 0;
  for (int i = 0; i < 4; i++) { u128 d = (u128)a[i] - p[i] - br; a[i] = (uint64_t)d; br = (uint64_t)(d >> 64) & 1; }
}
static fe f_add(fe a, fe b, const uint64_t *p) {
  fe r; uint64_t c = 0;
  for (int i = 0; i < 4; i++) { u128 s = (u128)a.l[i] + b.l[i] + c; r.l[i] = (uint64_t)s; c = (uint64_t)(s >> 64); }
  if (geq(r.l, p)) sub_p(r.l, p);
  return r;
}
static fe f_mul(fe a, fe b, const uint64_t *p, uint64_t n0) {
  uint64_t t[6] = {0, 0, 0, 0, 0, 0};
  for (int i = 0; i < 4; i++) {
    uint64_t c = 0;
    for (int j = 0; j < 4; j++) { u128 s = (u128)a.l[j] * b.l[i] + t[j] + c; t[j] = (uint64_t)s; c = (uint64_t)(s >> 64); }
    u128 s = (u128)t[4] + c; t[4] = (uint64_t)s; t[5] = (uint64_t)(s >> 64);
    uint64_t q = t[0] * n0;
    s = (u128)q * p[0] + t[0]; c = (uint64_t)(s >> 64);
    for (int j = 1; j < 4; j++) { s = (u128)q * p[j] + t[j] + c; t[j - 1] = (uint64_t)s; c = (uint64_t)(s >> 64); }
    s = (u128)t[4] + c; t[3] = (uint64_t)s; t[4] = t[5] + (uint64_t)(s >> 64);
  }
  fe r; memcpy(r.l, t, 32);
  if (t[4] || geq(r.l, p)) sub_p(r.l, p);
  return r;
}

/* SprsMat::row_mul (utils.rs:41-52) */
static void row_mul(const fe *v, uint64_t m, const uint64_t *ind_ptr, const uint64_t *col_ind, const fe *val, fe *out,
                    const uint64_t *p, uint64_t n0) {
  for (uint64_t j = 0; j < m; j++) {
    fe acc = {{0, 0, 0, 0}};
    for (uint64_t k = ind_ptr[j]; k < ind_ptr[j + 1]; k++) acc = f_add(acc, f_mul(v[col_ind[k]], val[k], p, n0), p);
    out[j] = acc;
  }
}

void bdo_sprs_row_mul(const uint64_t *p, uint64_t n, uint64_t m, const uint64_t *ind_ptr, const uint64_t *col_ind, const uint64_t *val,
                      const uint64_t *v, uint64_t count, uint64_t *out) {
  uint64_t n0 = 1;
  for (int i = 0; i < 6; i++) n0 *= 2 - p[0] * n0;
  n0 = (uint64_t)0 - n0;
  for (uint64_t c = 0; c < count; c++)
    row_mul((const fe *)v + c * n, m, ind_ptr, col_ind, (const fe *)val, (fe *)out + c * m, p, n0);
}

/* a_dims / b_dims: L (rows, cols, d) triples; ind_ptr / col_ind / val: 2L matrices A_0..A_{L-1}, B_0..B_{L-1}; one_mont = R mod p */
void bdo_encode(const uint64_t *p, const uint64_t *one_mont, uint64_t m, uint64_t m_ext, uint64_t L, const uint64_t *a_dims,
                const uint64_t *b_dims, const uint64_t *const *ind_ptr, const uint64_t *const *col_ind, const uint64_t *const *val,
                const uint64_t *mat, uint64_t n_rows, uint64_t *out, int deep_first) {
  uint64_t n0 = 1;
  for (int i = 0; i < 6; i++) n0 *= 2 - p[0] * n0;
  n0 = (uint64_t)0 - n0;
  uint64_t *start = (uint64_t *)calloc(L + 1, 8), *end = (uint64_t *)calloc(L + 1, 8);
  uint64_t acc = 0, e = m_ext;
  for (uint64_t i = 0; i < L; i++) { acc += a_dims[3 * i]; start[i] = acc; e -= b_dims[3 * i + 1]; end[i] = e; }
  const uint64_t rss = L ? start[L - 1] : 0;
  const uint64_t rsie = rss + (L ? a_dims[3 * (L - 1) + 1] : m);
  const uint64_t rsoe = L ? end[L - 1] : m_ext;
  fe one; memcpy(one.l, one_mont, 32);
#pragma omp parallel for schedule(dynamic, 1)
  for (uint64_t r = 0; r < n_rows; r++) {
    fe *cw = (fe *)out + r * m_ext;
    memset(cw, 0, m_ext * sizeof(fe));
    memcpy(cw, (const fe *)mat + r * m, m * sizeof(fe));
    uint64_t len = m;
    for (uint64_t i = 0; i < L; i++) {         /* cw.append(A_i.row_mul(cw[s - a_dims[i].0 .. s])) */
      row_mul(cw + start[i] - a_dims[3 * i], a_dims[3 * i + 1], ind_ptr[i], col_ind[i], (const fe *)val[i], cw + len, p, n0);
      len += a_dims[3 * i + 1];
    }
    /* naive_reed_solomon(cw, rss, rsie, rsoe) (mod.rs:111-122) */
    fe *res = (fe *)calloc(rsoe - rss + 1, sizeof(fe));
    fe x = one;
    for (uint64_t t = 0; t < rsoe - rss; t++) {
      for (uint64_t j = rsie; j-- > rss;) { res[t] = f_mul(res[t], x, p, n0); res[t] = f_add(res[t], cw[j], p); }
      x = f_add(x, one, p);
    }
    memcpy(cw + rss, res, (rsoe - rss) * sizeof(fe));
    free(res);
    for (uint64_t q = 0; q < L; q++) {          /* cw[e..e + b_dims[i].1] = B_i.row_mul(cw[s..e]), i ascending */
      const uint64_t i = deep_first ? L - 1 - q : q;
      fe *o = (fe *)malloc((b_dims[3 * i + 1] + 1) * sizeof(fe));
      row_mul(cw + start[i], b_dims[3 * i + 1], ind_ptr[L + i], col_ind[L + i], (const fe *)val[L + i], o, p, n0);
      memcpy(cw + end[i], o, b_dims[3 * i + 1] * sizeof(fe));
      free(o);
    }
  }
  free(start); free(end);
}
