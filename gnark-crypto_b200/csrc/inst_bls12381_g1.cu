// explicit instantiation of the engine for bls12381_g1
// out-of-line field multiplier: faster for the 12-limb and Fp2 groups (instruction-cache bound when inlined),
// slower for bn254 G1 -- see field.cuh
#define GMSM_MUL_NOINLINE 1
// Per-group build choices, each chosen by an A/B timing of the MultiExp:
//  * dedicated squaring + fused two-product y-coordinate (field.cuh): fewer IMAD.WIDE per mixed addition
//  * bn254 G1 only: no software prefetch of the next point (the gather latency is covered by the other warps), which frees its
//    16 registers: 128 registers, 4 blocks / SM, no spills (for the 12-limb G1 groups the prefetch stays)
#ifndef GMSM_SQR_DEDICATED
#define GMSM_SQR_DEDICATED 1
#endif
#ifndef GMSM_DOT2
#define GMSM_DOT2 1
#endif
#include "engine_impl.cuh"
namespace gmsm {
GMSM_INSTANTIATE_PAIRING_G1(bls12381_g1, vt_bls12381_g1)
}
