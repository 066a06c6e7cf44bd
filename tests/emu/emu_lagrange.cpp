// TEST INFRASTRUCTURE ONLY -- the kzg.ToLagrangeG1 kernels (gnark-crypto_b200/csrc/lagrange_kernels.cuh) on the CPU for one G1
// group per object (-DEMU_GROUP = the group's gmsm_curve_t id), launched by the library's schedule (lagrange_schedule, as
// engine_impl.cuh's run_to_lagrange): stage 0 from the affine input, the other stages on the workspace, then the finish kernel.
// The domain inverses w^-1 and 1/n come from the caller (the library takes them from fft.cu).  tests/test_emu_lagrange_cpu.py.
#include <cstring>
#include <vector>

#include "lagrange_kernels.cuh"

using namespace gmsm;

#ifndef EMU_GROUP
#error "compile with -DEMU_GROUP=<gmsm_curve_t id of a pairing G1 group>"
#endif
#if EMU_GROUP == 0
using EmuG = bn254_g1;
#elif EMU_GROUP == 2
using EmuG = bls12381_g1;
#elif EMU_GROUP == 4
using EmuG = bls12377_g1;
#elif EMU_GROUP == 7
using EmuG = bw6761_g1;
#elif EMU_GROUP == 9
using EmuG = bls24315_g1;
#elif EMU_GROUP == 10
using EmuG = bls24317_g1;
#elif EMU_GROUP == 11
using EmuG = bw6633_g1;
#else
#error "not a pairing G1 group"
#endif

namespace {
unsigned nblk(uint64_t n, unsigned t) { return (unsigned)((n + t - 1) / t); }
}  // namespace

#define EMU_CAT2(a, b) a##b
#define EMU_CAT(a, b) EMU_CAT2(a, b)
// out = ToLagrangeG1(points), n = 2^k points (reference layout); w_inv, n_inv: Montgomery fr limbs.  out may equal points.
// Returns 0, 1 for a bad n, 2 if the kernels wrote to the input.
extern "C" int EMU_CAT(emu_to_lagrange_, EMU_GROUP)(const void* points, uint64_t n, const void* w_inv, const void* n_inv, void* out) {
  using G = EmuG;
  using F = typename G::F;
  using Fr = typename G::Fr;
  using A = Affine<F>;
  if (n == 0 || (n & (n - 1)) || n > (1ull << LAG_MAX_LOG)) return 1;
  std::vector<A> in(n);
  std::memcpy(in.data(), points, n * sizeof(A));
  if (n == 1) {
    std::memcpy(out, in.data(), sizeof(A));
    return 0;
  }
  int logn = 0;
  while ((1ull << logn) < n) logn++;
  Fr wi, ni;
  std::memcpy(wi.l, w_inv, sizeof(Fr));
  std::memcpy(ni.l, n_inv, sizeof(Fr));
  const LagPowers<G> pw = lag_powers<G>(wi, logn);
  std::vector<XYZZ<F>> ws(n);
  std::vector<A> res(n);
  lagrange_schedule(
      n, logn,
      [&](int s, uint64_t threads) {
        if (s == 0)
          emu_launch(k_lag_stage<G, true>, dim3(nblk(threads, 128)), 128u, (const A*)in.data(), ws.data(), (uint32_t)threads, logn, s, pw);
        else
          emu_launch(k_lag_stage<G, false>, dim3(nblk(threads, 128)), 128u, (const A*)in.data(), ws.data(), (uint32_t)threads, logn, s, pw);
      },
      [&](uint64_t threads) {
        emu_launch(k_lag_finish<G>, dim3(nblk(threads, 128)), 128u, (const XYZZ<F>*)ws.data(), (uint32_t)n, logn, ni, res.data());
      });
  const int modified = std::memcmp(in.data(), points, n * sizeof(A)) != 0;
  std::memcpy(out, res.data(), n * sizeof(A));
  return modified ? 2 : 0;
}
