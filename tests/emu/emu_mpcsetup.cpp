// TEST INFRASTRUCTURE ONLY -- the mpcsetup kernel (gnark-crypto_b200/csrc/mpc_kernels.cuh: out[i] = [c r^(start + i)] points[i])
// on the CPU for one group per object (-DEMU_GROUP = the group's gmsm_curve_t id), launched by the library's schedule
// (scale_powers_args and scale_powers_schedule, as engine_impl.cuh's run_scale_powers).  tests/test_emu_mpcsetup_cpu.py.
#include <cstring>
#include <vector>

#include "mpc_kernels.cuh"

using namespace gmsm;

#ifndef EMU_GROUP
#error "compile with -DEMU_GROUP=0..12"
#endif
#if EMU_GROUP == 0
using EmuG = bn254_g1;
#elif EMU_GROUP == 1
using EmuG = bn254_g2;
#elif EMU_GROUP == 2
using EmuG = bls12381_g1;
#elif EMU_GROUP == 3
using EmuG = bls12381_g2;
#elif EMU_GROUP == 4
using EmuG = bls12377_g1;
#elif EMU_GROUP == 5
using EmuG = bls12377_g2;
#elif EMU_GROUP == 6
using EmuG = secp256k1_g1;
#elif EMU_GROUP == 7
using EmuG = bw6761_g1;
#elif EMU_GROUP == 8
using EmuG = bw6761_g2;
#elif EMU_GROUP == 9
using EmuG = bls24315_g1;
#elif EMU_GROUP == 10
using EmuG = bls24317_g1;
#elif EMU_GROUP == 11
using EmuG = bw6633_g1;
#else
using EmuG = bw6633_g2;
#endif

#define EMU_CAT2(a, b) a##b
#define EMU_CAT(a, b) EMU_CAT2(a, b)
// out[i] = [c r^(start + i)] points[i], i < n (reference layout, Montgomery fr limbs c, r).  Returns 0, or 2 if the kernel wrote to
// the input.
extern "C" int EMU_CAT(emu_scale_powers_, EMU_GROUP)(const void* points, uint64_t n, const void* c, const void* r, uint64_t start,
                                                      void* out) {
  using A = Affine<typename EmuG::F>;
  if (n == 0) return 0;
  std::vector<A> in(n), res(n);
  std::memcpy(in.data(), points, n * sizeof(A));
  const ScalePowers<EmuG> pw = scale_powers_args<EmuG>((const uint64_t*)c, (const uint64_t*)r, start);
  scale_powers_schedule(n, [&](uint64_t threads) {
    emu_launch(k_scale_powers<EmuG>, dim3((unsigned)((threads + 127) / 128)), 128u, (const A*)in.data(), (uint32_t)n, pw, res.data());
  });
  const int modified = std::memcmp(in.data(), points, n * sizeof(A)) != 0;
  std::memcpy(out, res.data(), n * sizeof(A));
  return modified ? 2 : 0;
}
