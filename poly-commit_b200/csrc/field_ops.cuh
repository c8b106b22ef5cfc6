// One field primitive applied to element i of two operand arrays.  pcgpu_diag_field_op runs this body on the device and the
// host-emulation harness (tests/host_emul) runs the same body on the host, so the field layer is checked against plain
// integers through identical code on both.  Op numbers: include/pcgpu.h, pcgpu_diag_field_op.
#pragma once
#include "ec.cuh"
#include "rt.cuh"

namespace pcgpu {

// pow2: the fp_inv_gcd table of P (Pow2TableBody<P>); only op 8 reads it
template <class P>
PCGPU_DEV Fp<P> field_op(int op, const Fp<P> &x, const Fp<P> &y, const uint32_t *pow2) {
  switch (op) {
    case 0: return mont_mul<P>(x, y);
    case 1: return mont_mul_ref<P>(x, y);
    case 2: return fp_add<P>(x, y);
    case 3: return fp_sub<P>(x, y);
    case 4: return fp_neg<P>(x);
    case 5: return fp_inv<P>(x);
    case 6:   // x*y + y*(-x) = 0
      if constexpr (mont_mul2_supported<P>()) return mont_mul2<P>(x, y, y, fp_neg<P>(x));
      else return Fp<P>::zero();
    case 7:   // x*y + (x+y)(y-x): a sum of two products, one reduction
      if constexpr (mont_mul2_supported<P>()) return mont_mul2<P>(x, y, fp_add<P>(x, y), fp_sub<P>(y, x));
      else return fp_add<P>(mont_mul<P>(x, y), mont_mul<P>(fp_add<P>(x, y), fp_sub<P>(y, x)));
    case 8: return fp_inv_gcd<P>(x, pow2);
    case 9: return mont_sqr<P>(x);
    default: return Fp<P>::zero();
  }
}

template <class P>
struct FieldOpBody {
  const uint32_t *a, *b; uint32_t *out; const uint32_t *pow2; int op;
  PCGPU_KERNEL_DEV void operator()(size_t i) const {
    Fp<P> x, y;
#pragma unroll
    for (int j = 0; j < P::N; j++) { x.l[j] = a[i * P::N + j]; y.l[j] = b[i * P::N + j]; }
    const Fp<P> r = field_op<P>(op, x, y, pow2);
#pragma unroll
    for (int j = 0; j < P::N; j++) out[i * P::N + j] = r.l[j];
  }
};

}  // namespace pcgpu
