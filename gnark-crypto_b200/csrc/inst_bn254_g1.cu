// explicit instantiation of the engine for bn254_g1
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
#ifndef GMSM_ACC_NOPREFETCH
#define GMSM_ACC_NOPREFETCH 1
#endif
#ifndef GMSM_ACC_MINBLOCKS_SMALL
#define GMSM_ACC_MINBLOCKS_SMALL 4
#endif
#include "engine_impl.cuh"
namespace gmsm {
GMSM_INSTANTIATE_PAIRING_G1(bn254_g1, vt_bn254_g1)
}
