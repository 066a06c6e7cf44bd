// explicit instantiation of the engine for bls24317_g1 (next-row N4, ecc/bls24-317/multiexp.go:32): 5-word Fp = 10 32-bit limbs, 4-word scalars.
// Between the 8-limb (inlined multiplier) and 12-limb (out-of-line) groups; built like the 12-limb G1 groups, but at 3 blocks per SM:
// k_accumulate needs 190 registers unconstrained (2 blocks); capped at 168 it spills a little and runs 12 warps per SM, which
// is faster (the 12-limb groups, 232 registers, gain nothing from the cap)
#define GMSM_MUL_NOINLINE 1
#ifndef GMSM_ACC_MINBLOCKS_BIG
#define GMSM_ACC_MINBLOCKS_BIG 3
#endif
#ifndef GMSM_SQR_DEDICATED
#define GMSM_SQR_DEDICATED 1
#endif
#ifndef GMSM_DOT2
#define GMSM_DOT2 1
#endif
#include "engine_impl.cuh"
namespace gmsm {
GMSM_INSTANTIATE_PAIRING_G1(bls24317_g1, vt_bls24317_g1)
}
