// explicit instantiation of the engine for bw6761_g1 (next-row N4, ecc/bw6-761/multiexp.go:32)
// 12-word Fp = 24 32-bit limbs per coordinate (an extended-Jacobian accumulator alone is 96 registers), 6-word scalars
// (fr.Bits = 377).  G1 and G2 of this curve are both defined over Fp, so they share every kernel shape.  Out-of-line
// multiplier / squaring / fused two-product routines: 1152 IMAD.WIDE per product do not fit inlined ten times.
#define GMSM_MUL_NOINLINE 1
#define GMSM_ACC_NOPREFETCH 1
#ifndef GMSM_SQR_DEDICATED
#define GMSM_SQR_DEDICATED 1
#endif
#ifndef GMSM_DOT2
#define GMSM_DOT2 1
#endif
#include "engine_impl.cuh"
namespace gmsm {
GMSM_INSTANTIATE_PAIRING_G1(bw6761_g1, vt_bw6761_g1)
}
