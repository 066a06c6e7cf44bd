// TEST INFRASTRUCTURE ONLY -- the G2 decoding and point encoding kernels (gnark-crypto_b200/csrc/marshal_kernels.cuh, the header
// decode.cu includes) on the CPU, launched as decode.cu's gmsm_g2_decode_device and gmsm_points_encode_device launch them: the
// per-group constants from the same host helpers, one thread per point, the first error folded with a 64-bit atomicMin
// (defined here: the stand-in runtime header has only the 32-bit atomics the MSM kernels use).  The encoder stages a block's
// output in shared memory between a barrier, so it runs under the cooperative launcher.
#include <cuda_runtime.h>   // the stand-in of tests/emu

#include <algorithm>
#include <cstring>
#include <type_traits>

static inline unsigned long long atomicMin(unsigned long long* p, unsigned long long v) {
  const unsigned long long o = *p;
  *p = std::min(o, v);
  return o;
}

#include "marshal_kernels.cuh"

namespace {
template <class P>
void launch_decode(const gmsm::DecodeConsts<P>& kc, const uint8_t* bytes, uint32_t n, int raw, int check, uint32_t* out,
                   unsigned long long* err) {
  emu_launch(gmsm::k_g1_decode<P>, dim3((n + 127) / 128), 128u, bytes, n, raw, check, kc, reinterpret_cast<gmsm::Affine<gmsm::Fp<P>>*>(out), err);
}
template <class P>
void launch_decode(const gmsm::G2DecodeConsts<P>& kc, const uint8_t* bytes, uint32_t n, int raw, int check, uint32_t* out,
                   unsigned long long* err) {
  emu_launch(gmsm::k_g2_decode<P>, dim3((n + 127) / 128), 128u, bytes, n, raw, check, kc, reinterpret_cast<gmsm::Affine<gmsm::Fp2<P>>*>(out), err);
}
}  // namespace

// curve: a G2 id of gmsm_curve_t; bytes: n points (raw: 2 coordinates each, else 1); out: n affine points (Go layout);
// *first_error = (index << 8 | code) of the first bad point, all-ones if none.  Returns 0, or 1 for a group without a decoder.
extern "C" int emu_g2_decode_run(int curve, const uint8_t* bytes, uint32_t n, int raw, int check_on_curve, uint32_t* out,
                                 unsigned long long* first_error) {
  *first_error = ~0ull;
  const int rc = gmsm::with_g2_decode_consts(curve, [&](const auto& kc) {
    if (n) launch_decode(kc, bytes, n, raw, check_on_curve, out, first_error);
    return 0;
  });
  return rc < 0 ? 1 : 0;
}

// curve: a G1 or G2 id of a pairing curve; points: n affine points (Go layout); out: n encoded points.  Returns 0, or 1 for a
// group without an encoder.
extern "C" int emu_points_encode_run(int curve, const uint32_t* points, uint32_t n, int raw, uint32_t* out) {
  const int rc = gmsm::with_encode_group(curve, [&](auto g) {
    using G = decltype(g);
    using P = typename G::Params;
    using C = std::conditional_t<G::degree == 1, gmsm::Fp<P>, gmsm::Fp2<P>>;
    const auto* pts = reinterpret_cast<const gmsm::Affine<C>*>(points);
    const dim3 grid((n + gmsm::ENC_THREADS - 1) / gmsm::ENC_THREADS);
    if (n && raw) emu_launch_coop(gmsm::k_points_encode<P, G::degree, 1>, grid, (unsigned)gmsm::ENC_THREADS, pts, n, out);
    if (n && !raw) emu_launch_coop(gmsm::k_points_encode<P, G::degree, 0>, grid, (unsigned)gmsm::ENC_THREADS, pts, n, out);
    return 0;
  });
  return rc < 0 ? 1 : 0;
}
