// explicit instantiation of the engine for bw6633_g1 (next-row N4, ecc/bw6-633/multiexp.go:32): 10-word Fp = 20 32-bit limbs per coordinate, both groups
// of the curve over Fp, 5-word scalars (fr.Bits = 315: 40-byte fr.Element, loaded in 8-byte granules).  Built like bw6-761.
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
GMSM_INSTANTIATE_PAIRING_G1(bw6633_g1, vt_bw6633_g1)
}
