// Batched-affine pairwise reduction rounds for the bucket accumulation.
//
// An affine addition costs 1 inversion + 2M + 1S; with Montgomery's trick over a batch of K independent
// additions the inversion is shared: 3 multiplications per element plus ONE inversion per batch, i.e.
// ~6.2 modular multiplications per addition instead of the 9.5 of the XYZZ mixed addition -- provided the
// shared inversion is cheap.  It is: fp_inv_gcd runs on the ALU pipe, which idles while the integer-multiply
// pipe saturates, so across warps the two overlap.
//
// Independent additions come from pairing neighbours inside every bucket: round r turns the cnt_b points of
// bucket b into ceil(cnt_b / 2) points (an odd one out is copied).  Thread t of a round owns the output slots
// t, t+T, t+2T, ... (coalesced); pass 1 walks them accumulating the running product of the denominators
// (x2 - x1) and storing the prefix products, pass 2 walks back turning the single inverse into every 1/(x2 - x1)
// and emitting the sums.  Exceptional pairs (P = Q, P = -Q, identity operands) get denominator 2y / 1 and are
// resolved in pass 2.  After R rounds the remaining points (a few per bucket) go through the XYZZ task kernel.
#pragma once
#include "msm.cuh"

namespace pcgpu {

enum : uint32_t { PAIR_SINGLE = 0x80000000u, PAIR_EXC = 0x40000000u, PAIR_NONE = 0xffffffffu };

struct PairCountBody {   // cnt_out[b] = ceil(cnt_in[b] / 2)
  const uint32_t *off_in; uint32_t *cnt_out;
  PCGPU_KERNEL_DEV void operator()(size_t b) const { cnt_out[b] = (off_in[b + 1] - off_in[b] + 1) / 2; }
};

struct PairPlanBody {    // src[o] = index of the first operand of output slot o (| PAIR_SINGLE when it has no partner)
  const uint32_t *off_in; const uint32_t *off_out; uint32_t TB; uint32_t *src;
  PCGPU_KERNEL_DEV void operator()(size_t o) const {
    if (o >= off_out[TB]) return;
    uint32_t lo = 0, hi = TB;   // last b with off_out[b] <= o
    while (hi - lo > 1) { uint32_t mid = (lo + hi) / 2; if (off_out[mid] <= (uint32_t)o) lo = mid; else hi = mid; }
    uint32_t b = lo, j = (uint32_t)o - off_out[b], cnt = off_in[b + 1] - off_in[b];
    uint32_t first = off_in[b] + 2 * j;
    src[o] = first | ((2 * j + 1 >= cnt) ? PAIR_SINGLE : 0u);
  }
};

// read-only (non-coherent) loads: the operands of a pair round are never written by it, which lets the compiler hoist
// the gathers of several iterations above the prefix stores
PCGPU_DEV u32x4 ldg4(const u32x4 *p) {
#ifdef __CUDA_ARCH__
  uint4 v = __ldg(reinterpret_cast<const uint4 *>(p));
  u32x4 r; r.x = v.x; r.y = v.y; r.z = v.z; r.w = v.w; return r;
#else
  return *p;
#endif
}
PCGPU_DEV uint32_t ldg_plain(const uint32_t *p) { return *p; }   // coherent load (data written earlier by the same thread)
PCGPU_DEV uint32_t ldg1(const uint32_t *p) {
#ifdef __CUDA_ARCH__
  return __ldg(p);
#else
  return *p;
#endif
}
template <class Q>
PCGPU_DEV Fp<Q> load_fq(const uint32_t *p) {
  constexpr int N = Q::N;
  const u32x4 *q = reinterpret_cast<const u32x4 *>(p);
  Fp<Q> r;
#pragma unroll
  for (int j = 0; j < N / 4; j++) { u32x4 v = ldg4(q + j); r.l[4 * j] = v.x; r.l[4 * j + 1] = v.y; r.l[4 * j + 2] = v.z; r.l[4 * j + 3] = v.w; }
  return r;
}
template <class Q>
PCGPU_DEV void store_fq(uint32_t *p, const Fp<Q> &a) {
  constexpr int N = Q::N;
  u32x4 *q = reinterpret_cast<u32x4 *>(p);
#pragma unroll
  for (int j = 0; j < N / 4; j++) { u32x4 v; v.x = a.l[4 * j]; v.y = a.l[4 * j + 1]; v.z = a.l[4 * j + 2]; v.w = a.l[4 * j + 3]; q[j] = v; }
}

// pair classification: which formula pass 2 uses, and the field element whose inverse it needs
enum : uint32_t { PK_ADD = 0, PK_DBL = 1, PK_TAKE_P = 2, PK_TAKE_Q = 3, PK_INF = 4 };
template <class C>
PCGPU_DEV uint32_t pair_classify(const Affine<C> &P, const Affine<C> &Qp, bool single, Fp<typename C::Fq> &d) {
  using Q = typename C::Fq;
  d = Fp<Q>::one();
  if (single) return PK_TAKE_P;
  if (P.is_inf()) return Qp.is_inf() ? PK_INF : PK_TAKE_Q;
  if (Qp.is_inf()) return PK_TAKE_P;
  if (P.x == Qp.x) {
    if (P.y == Qp.y && !P.y.is_zero()) { d = fp_dbl<Q>(P.y); return PK_DBL; }
    return PK_INF;
  }
  d = fp_sub<Q>(Qp.x, P.x);
  return PK_ADD;
}

template <class C, bool FROM_TABLES>
struct MsmAffinePairBody {
  const uint32_t *tables; MsmGeom g; const uint32_t *entries;  // round 0: operands are (table group, base, sign) entries
  const Affine<C> *pts_in;                                      // later rounds: operands are affine points
  uint32_t *src; const uint32_t *off_out;                       // plan; total outputs = off_out[g.TB] (pass 1 may set PAIR_EXC)
  uint32_t T;                                                   // threads in this launch
  uint32_t *prefix;                                             // per (iteration, thread): prefix product; round 0 also x1 and d
  const uint32_t *pow2;                                         // fp_inv_gcd table
  Affine<C> *pts_out;

  // Slot descriptor: round 0 -> (entry of P, entry of Q or PAIR_NONE); later rounds -> (index of P, PAIR_NONE if single).
  // Descriptors are fetched ONE iteration ahead so that the only load latency exposed per iteration is the point gather.
  struct Slot { uint32_t a, b; };
  PCGPU_DEV Slot fetch_slot(uint32_t o) const {
    uint32_t sv = ldg1(src + o);
    uint32_t i0 = sv & ~(PAIR_SINGLE | PAIR_EXC);
    bool single = (sv & PAIR_SINGLE) != 0;
    Slot s;
    if (FROM_TABLES) { s.a = ldg1(entries + i0); s.b = single ? PAIR_NONE : ldg1(entries + i0 + 1); }
    else { s.a = i0; s.b = single ? PAIR_NONE : 0u; }
    return s;
  }
  PCGPU_DEV const uint32_t *slot_rec(uint32_t v) const {   // record of a round-0 entry
    uint32_t grp = (v & ~ENTRY_SIGN) >> ENTRY_GROUP_SHIFT;
    return table_record<C>(tables, (size_t)grp * g.table_stride + g.base_off + (v & ENTRY_IDX_MASK), g);
  }
  PCGPU_DEV Fp<typename C::Fq> slot_x(const Slot &s, int which) const {
    using Q = typename C::Fq;
    if (FROM_TABLES) return load_fq<Q>(slot_rec(which ? s.b : s.a));
    return load_fq<Q>(reinterpret_cast<const uint32_t *>(pts_in + s.a + which));
  }
  PCGPU_DEV Affine<C> slot_point(const Slot &s, int which) const {
    using Q = typename C::Fq;
    if (FROM_TABLES) {
      uint32_t v = which ? s.b : s.a;
      const uint32_t *rec = slot_rec(v);
      Affine<C> a; a.x = load_fq<Q>(rec); a.y = load_fq<Q>(rec + g.y_words);
      if (!a.is_inf()) a.y = fp_cneg<Q>(a.y, (v & ENTRY_SIGN) != 0);
      return a;
    }
    return load_affine<C>(pts_in + s.a + which);
  }
  PCGPU_DEV Fp<typename C::Fq> slot_denominator(const Slot &s) const {
    using Q = typename C::Fq;
    if (s.b == PAIR_NONE) return Fp<Q>::one();
    Fp<Q> x1 = slot_x(s, 0), x2 = slot_x(s, 1);
    if (x1 != x2 && !x1.is_zero() && !x2.is_zero()) return fp_sub<Q>(x2, x1);
    Affine<C> P = slot_point(s, 0), Qp = slot_point(s, 1);   // exceptional pair: rare
    Fp<Q> d;
    pair_classify<C>(P, Qp, false, d);
    return d;
  }

  PCGPU_KERNEL_DEV void operator()(size_t t) const {
    using Q = typename C::Fq;
    constexpr int N = Q::N;
    if (t >= T) return;
    const uint32_t total = off_out[g.TB];
    uint32_t *xbuf = prefix + (size_t)T * N * ((total + T - 1) / T);   // round 0 only: x1 per slot, then d per slot
    uint32_t *dbuf = xbuf + (size_t)T * N * ((total + T - 1) / T);
    // ---- pass 1: running product of the denominators, prefix products to memory ----
    const uint32_t kmax = (uint32_t)t < total ? (total - (uint32_t)t + T - 1) / T : 0u;   // slots k*T + t < total
    Fp<Q> acc = Fp<Q>::one();
    {
      Slot nxt; nxt.a = 0; nxt.b = PAIR_NONE;
      if (kmax) nxt = fetch_slot((uint32_t)t);
      for (uint32_t k = 0; k < kmax; k++) {
        Slot cur = nxt;
        if (k + 1 < kmax) nxt = fetch_slot((k + 1) * T + (uint32_t)t);   // descriptor of the next slot: in flight during this one
        Fp<Q> d;
        if (FROM_TABLES) {
          // Round 0 gathers every base twice (x here, y in pass 2).  x1 and the denominator are written out next to the
          // prefix product (coalesced), so pass 2 re-reads them sequentially and gathers ONLY the y halves of the records:
          // the random traffic of the round halves (random 64/128-byte HBM accesses run at ~1/4 of the streaming rate).
          Fp<Q> x1 = slot_x(cur, 0);
          bool exc = false;
          if (cur.b == PAIR_NONE) d = Fp<Q>::one();
          else {
            Fp<Q> x2 = slot_x(cur, 1);
            if (x1 != x2 && !x1.is_zero() && !x2.is_zero()) d = fp_sub<Q>(x2, x1);
            else { Affine<C> P = slot_point(cur, 0), Qp = slot_point(cur, 1); pair_classify<C>(P, Qp, false, d); exc = true; }
          }
          if (exc) src[k * T + (uint32_t)t] |= PAIR_EXC;
          store_fq<Q>(xbuf + ((size_t)k * T + t) * N, x1);
          store_fq<Q>(dbuf + ((size_t)k * T + t) * N, d);
        } else {
          d = slot_denominator(cur);
        }
        store_fq<Q>(prefix + ((size_t)k * T + t) * N, acc);
        acc = fp_mul<Q>(acc, d);
      }
    }
    Fp<Q> inv = fp_inv_gcd<Q>(acc, pow2);
    // ---- pass 2: walk back, one inverse per pair, emit the sums ----
    Slot nxt2; nxt2.a = 0; nxt2.b = PAIR_NONE;
    if (kmax) nxt2 = fetch_slot((kmax - 1) * T + (uint32_t)t);
    for (uint32_t k2 = kmax; k2-- > 0;) {
      const uint32_t k = k2;
      uint32_t o = k * T + (uint32_t)t;
      Slot cur = nxt2;
      const bool exc = FROM_TABLES && (ldg_plain(src + o) & PAIR_EXC) != 0;
      if (k > 0) nxt2 = fetch_slot(o - T);
      bool single = cur.b == PAIR_NONE;
      if (FROM_TABLES && !exc) {
        // fast path: x1, d from pass 1 (sequential), y halves gathered
        Fp<Q> x1 = load_fq<Q>(xbuf + ((size_t)k * T + t) * N), d = load_fq<Q>(dbuf + ((size_t)k * T + t) * N);
        Fp<Q> y1 = fp_cneg<Q>(load_fq<Q>(slot_rec(cur.a) + g.y_words), (cur.a & ENTRY_SIGN) != 0);
        Fp<Q> dinv = fp_mul<Q>(inv, load_fq<Q>(prefix + ((size_t)k * T + t) * N));
        inv = fp_mul<Q>(inv, d);
        Affine<C> R;
        if (single) { R.x = x1; R.y = y1; if (x1.is_zero() && y1.is_zero()) R = Affine<C>::inf(); }
        else {
          Fp<Q> y2 = fp_cneg<Q>(load_fq<Q>(slot_rec(cur.b) + g.y_words), (cur.b & ENTRY_SIGN) != 0);
          Fp<Q> lam = fp_mul<Q>(fp_sub<Q>(y2, y1), dinv);
          Fp<Q> x2 = fp_add<Q>(x1, d);
          Fp<Q> x3 = fp_sub<Q>(fp_sub<Q>(fp_sqr<Q>(lam), x1), x2);
          R.x = x3;
          R.y = fp_sub<Q>(fp_mul<Q>(lam, fp_sub<Q>(x1, x3)), y1);
        }
        Affine<C> *dst0 = pts_out + o;
        store_fq<Q>(reinterpret_cast<uint32_t *>(dst0), R.x);
        store_fq<Q>(reinterpret_cast<uint32_t *>(dst0) + N, R.y);
        continue;
      }
      Affine<C> P = slot_point(cur, 0), Qp = single ? Affine<C>::inf() : slot_point(cur, 1);
      Fp<Q> d;
      uint32_t kind = pair_classify<C>(P, Qp, single, d);
      Fp<Q> dinv = fp_mul<Q>(inv, load_fq<Q>(prefix + ((size_t)k * T + t) * N));
      inv = fp_mul<Q>(inv, d);
      Affine<C> R;
      if (kind == PK_ADD || kind == PK_DBL) {
        Fp<Q> num = kind == PK_ADD ? fp_sub<Q>(Qp.y, P.y) : fp_mul3<Q>(fp_sqr<Q>(P.x));
        Fp<Q> lam = fp_mul<Q>(num, dinv);
        Fp<Q> x3 = fp_sub<Q>(fp_sub<Q>(fp_sqr<Q>(lam), P.x), kind == PK_ADD ? Qp.x : P.x);
        R.x = x3;
        R.y = fp_sub<Q>(fp_mul<Q>(lam, fp_sub<Q>(P.x, x3)), P.y);
      } else if (kind == PK_TAKE_P) R = P;
      else if (kind == PK_TAKE_Q) R = Qp;
      else R = Affine<C>::inf();
      Affine<C> *dst = pts_out + o;
      store_fq<Q>(reinterpret_cast<uint32_t *>(dst), R.x);
      store_fq<Q>(reinterpret_cast<uint32_t *>(dst) + N, R.y);
    }
  }
};

}  // namespace pcgpu
