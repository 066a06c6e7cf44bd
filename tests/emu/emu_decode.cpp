// TEST INFRASTRUCTURE ONLY -- the G1 decoding kernel (gnark-crypto_b200/csrc/decode_kernels.cuh, the header decode.cu
// includes) on the CPU, launched as decode.cu's gmsm_g1_decode_device launches it: the per-curve constants from the same
// host helper, one thread per point, the first error folded with a 64-bit atomicMin (defined here: the stand-in runtime
// header has only the 32-bit atomics the MSM kernels use).
#include <cuda_runtime.h>   // the stand-in of tests/emu

#include <algorithm>
#include <cstring>

// the 64-bit atomicMin k_g1_decode folds the first error with (sequential, so a plain read-modify-write); declared before the
// kernel's header so that its non-dependent call binds to it
static inline unsigned long long atomicMin(unsigned long long* p, unsigned long long v) {
  const unsigned long long o = *p;
  *p = std::min(o, v);
  return o;
}

#include "decode_kernels.cuh"

// curve: a G1 id of gmsm_curve_t; bytes: n points (raw: 2 * fp.Bytes each, else fp.Bytes); out: n affine points (Go layout);
// *first_error = (index << 8 | code) of the first bad point, all-ones if none.  Returns 0, or 1 for a curve without a decoder.
extern "C" int emu_g1_decode_run(int curve, const uint8_t* bytes, uint32_t n, int raw, int check_on_curve, uint32_t* out,
                                 unsigned long long* first_error) {
  *first_error = ~0ull;
  const int rc = gmsm::with_g1_decode_consts(curve, [&](const auto& kc) {
    using K = std::decay_t<decltype(kc)>;
    using F = decltype(K::b);
    auto* pts = reinterpret_cast<gmsm::Affine<F>*>(out);
    const unsigned blocks = (n + 127) / 128;
    if (n) emu_launch(gmsm::k_g1_decode<typename F::Params>, dim3(blocks), 128u, bytes, n, raw, check_on_curve, kc, pts, first_error);
    return 0;
  });
  return rc < 0 ? 1 : 0;
}
