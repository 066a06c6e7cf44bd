// Element-wise test operations on the pairing towers (include/gmsm.h GMSM_TOWER_OP_*), one element per thread: each op calls the
// tower.cuh / pairing_kernels.cuh function it names, so tests reach the Fp6 / Fp12 operations, the sparse line products and the
// G2 line steps on operands the Miller loop and the final exponentiation never produce.  Run on the GPU by gmsm_test_tower_op
// (pairing.cu) and on the CPU by the kernel emulation (tests/emu/emu_pairing.cpp).  Not used by any production path.
#pragma once
#include "pairing_kernels.cuh"

namespace gmsm {

// Operand and output widths in Fp2 units (0: no operand; *wo = 0: an op this curve does not have).  E6 = 3, E12 = 6, a line or a
// G2Proj point = 3, a G2 affine point = 2, a G1 affine point = 1 (x, y share the layout of one Fp2), the product of two lines = 5.
template <class P>
GMSM_HD void tower_op_sizes(int op, int* wa, int* wb, int* wo) {
  *wa = *wb = *wo = 0;
  switch (op) {
    case 0: *wa = 3; *wb = 3; *wo = 3; break;                  // E6_MUL
    case 1: *wa = 3; *wo = 3; break;                           // E6_INV
    case 2: case 4: *wa = 3; *wb = 2; *wo = 3; break;          // E6_MUL_BY_01, E6_MUL_BY_12
    case 3: *wa = 3; *wb = 1; *wo = 3; break;                  // E6_MUL_BY_1
    case 5: *wa = 6; *wb = 6; *wo = 6; break;                  // E12_MUL
    case 6: case 7: case 8: case 9: case 10: case 11: case 12: case 13: case 14: case 15: case 23:
      *wa = 6; *wo = 6; break;                                 // one E12 in, one out
    case 16:                                                   // E12_EXPT_HALF: bls12-381 only
      if (!is_dtwist<P>()) { *wa = 6; *wo = 6; }
      break;
    case 17: *wa = 6; *wb = 3; *wo = 6; break;                 // E12_MUL_BY_LINE
    case 18: *wa = 3; *wb = 3; *wo = 5; break;                 // LINE_BY_LINE
    case 19: *wa = 6; *wb = 5; *wo = 6; break;                 // E12_MUL_BY_TWO_LINES
    case 20: *wa = 3; *wo = 6; break;                          // DOUBLE_STEP
    case 21: case 22: *wa = 3; *wb = 2; *wo = 6; break;        // ADD_MIXED_STEP, LINE_COMPUTE
    case 24: *wa = 1; *wb = 2; *wo = 6; break;                 // MILLER_LOOP_ONE
    default: break;
  }
}

template <class P>
GMSM_HD void tower_op_one(int op, const Fp2<P>* a, const Fp2<P>* b, Fp2<P>* o) {
  using E2 = Fp2<P>;
  using E6 = Fp6<P>;
  using E12 = Fp12<P>;
  auto e6 = [](const E2* p) { return E6{p[0], p[1], p[2]}; };
  auto e12 = [&](const E2* p) { return E12{e6(p), e6(p + 3)}; };
  auto put6 = [&](const E6& x) { o[0] = x.b0; o[1] = x.b1; o[2] = x.b2; };
  auto put12 = [&](const E12& x) {
    o[0] = x.c0.b0; o[1] = x.c0.b1; o[2] = x.c0.b2; o[3] = x.c1.b0; o[4] = x.c1.b1; o[5] = x.c1.b2;
  };
  auto point_line = [&](const G2Proj<P>& p, const Line<P>& l) {
    o[0] = p.x; o[1] = p.y; o[2] = p.z; o[3] = l.r0; o[4] = l.r1; o[5] = l.r2;
  };
  switch (op) {
    case 0: put6(e6_mul(e6(a), e6(b))); break;
    case 1: put6(e6_inv(e6(a))); break;
    case 2: put6(e6_mul_by_01(e6(a), b[0], b[1])); break;
    case 3: put6(e6_mul_by_1(e6(a), b[0])); break;
    case 4: put6(e6_mul_by_12(e6(a), b[0], b[1])); break;
    case 5: put12(e12_mul(e12(a), e12(b))); break;
    case 6: put12(e12_sqr(e12(a))); break;
    case 7: put12(e12_inv(e12(a))); break;
    case 8: put12(e12_conj(e12(a))); break;
    case 9: put12(e12_frob<1>(e12(a))); break;
    case 10: put12(e12_frob<2>(e12(a))); break;
    case 11: put12(e12_frob<3>(e12(a))); break;
    case 12: put12(e12_cyclo_sqr(e12(a))); break;
    case 13: put12(e12_cyclo_sqr_compressed(e12(a))); break;
    case 14: put12(e12_decompress_karabina(e12(a))); break;
    case 15: put12(e12_expt(e12(a))); break;
    case 16: put12(e12_expt_half(e12(a))); break;
    case 17: put12(mul_line(e12(a), Line<P>{b[0], b[1], b[2]})); break;   // mul_by_034 (bn254) / mul_by_014 (bls12-381)
    case 18: {                                                                   // mul_034_by_034 / mul_014_by_014
      E2 z[5];
      if constexpr (is_dtwist<P>()) e2_mul_034_by_034(a[0], a[1], a[2], b[0], b[1], b[2], z);
      else e2_mul_014_by_014(a[0], a[1], a[2], b[0], b[1], b[2], z);
      for (int i = 0; i < 5; i++) o[i] = z[i];
    } break;
    case 19: {                                                                   // mul_by_01234 / mul_by_01245
      const E2 x[5] = {b[0], b[1], b[2], b[3], b[4]};
      if constexpr (is_dtwist<P>()) put12(e12_mul_by_01234(e12(a), x));
      else put12(e12_mul_by_01245(e12(a), x));
    } break;
    case 20: {
      G2Proj<P> p{a[0], a[1], a[2]};
      const Line<P> l = double_step(p);
      point_line(p, l);
    } break;
    case 21: {
      G2Proj<P> p{a[0], a[1], a[2]};
      const Line<P> l = add_mixed_step(p, Affine<E2>{b[0], b[1]});
      point_line(p, l);
    } break;
    case 22: {
      const G2Proj<P> p{a[0], a[1], a[2]};
      point_line(p, line_compute(p, Affine<E2>{b[0], b[1]}));
    } break;
    case 23: {
      const E12 z = e12(a);
      put12(final_exp(&z, 1u));
    } break;
    case 24: put12(miller_loop_one(Affine<Fp<P>>{a[0].a0, a[0].a1}, Affine<E2>{b[0], b[1]})); break;
    default: break;
  }
}

// out[i] = op(a[i], b[i]) for i < n, operands and results at their tower_op_sizes strides
template <class P>
__global__ void __launch_bounds__(PAIRING_THREADS) k_tower_op(int op, const Fp2<P>* __restrict__ a, const Fp2<P>* __restrict__ b,
                                                              Fp2<P>* __restrict__ out, uint32_t n) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int wa, wb, wo;
  tower_op_sizes<P>(op, &wa, &wb, &wo);
  tower_op_one<P>(op, a + (size_t)i * wa, b + (size_t)i * wb, out + (size_t)i * wo);
}

}  // namespace gmsm
