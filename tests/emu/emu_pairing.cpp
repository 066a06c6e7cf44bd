// TEST INFRASTRUCTURE ONLY -- the pairing kernels (gnark-crypto_b200/csrc/pairing_kernels.cuh: k_miller_loop, k_gt_reduce,
// k_gt_accumulate, k_final_exp) on the CPU, launched in the library's order (pairing_schedule, as pairing.cu's run_miller), for
// bn254 (EMU_CURVE = 0) and bls12-381 (1), and the tower test ops (tower_testops.cuh: k_tower_op).  tests/test_emu_pairing_cpu.py,
// tests/test_tower_stress_cpu.py.
#include <cstring>
#include <vector>

#include "pairing_kernels.cuh"
#include "tower_testops.cuh"

using namespace gmsm;

#ifndef EMU_CURVE
#error "compile with -DEMU_CURVE=0 (bn254) or 1 (bls12-381)"
#endif
#if EMU_CURVE == 0
using EmuP = bn254_fp;
#else
using EmuP = bls12381_fp;
#endif

#define EMU_CAT2(a, b) a##b
#define EMU_CAT(a, b) EMU_CAT2(a, b)

// out = MillerLoop(P, Q) over n >= 1 pairs (reference layout), in chunks of `chunk` pairs and `threads` threads per block, blocks in
// emu_block_order = block_order
extern "C" void EMU_CAT(emu_miller_loop_, EMU_CURVE)(const void* pts, const void* qs, uint64_t n, uint64_t chunk, unsigned threads,
                                                    unsigned block_order, void* out) {
  using G = Fp12<EmuP>;
  emu_block_order = block_order;
  std::vector<G> work(pairing_work_elems(n, chunk));
  const auto* P = reinterpret_cast<const Affine<Fp<EmuP>>*>(pts);
  const auto* Q = reinterpret_cast<const Affine<Fp2<EmuP>>*>(qs);
  pairing_schedule(
      n, chunk,
      [&](size_t off, size_t m, size_t dst) {
        emu_launch(k_miller_loop<EmuP>, dim3((unsigned)((m + threads - 1) / threads)), threads, P + off, Q + off, (uint32_t)m, work.data() + dst);
      },
      [&](size_t src, size_t m, size_t dst) {
        emu_launch(k_gt_reduce<EmuP>, dim3((unsigned)((m / 2 + threads) / threads)), threads, (const G*)work.data() + src, (uint32_t)m,
                   work.data() + dst);
      },
      [&](size_t src, bool first) {
        emu_launch(k_gt_accumulate<EmuP>, dim3(1), 1u, work.data() + pairing_acc_index(n, chunk), (const G*)work.data() + src, (int)first);
      });
  emu_block_order = 0;
  std::memcpy(out, work.data() + pairing_acc_index(n, chunk), sizeof(G));
}

// out[i] = op(a[i], b[i]) for i < n (tower_testops.cuh, widths of tower_op_sizes); returns 0, or 1 for an op the curve does not have
extern "C" int EMU_CAT(emu_tower_op_, EMU_CURVE)(int op, const void* a, const void* b, void* out, uint64_t n, unsigned threads) {
  int wa, wb, wo;
  tower_op_sizes<EmuP>(op, &wa, &wb, &wo);
  if (wo == 0) return 1;
  emu_launch(k_tower_op<EmuP>, dim3((unsigned)((n + threads - 1) / threads)), threads, op, reinterpret_cast<const Fp2<EmuP>*>(a),
             reinterpret_cast<const Fp2<EmuP>*>(b), reinterpret_cast<Fp2<EmuP>*>(out), (uint32_t)n);
  return 0;
}

// out = FinalExponentiation(z[0], z[1..k))
extern "C" void EMU_CAT(emu_final_exp_, EMU_CURVE)(const void* z, uint64_t k, void* out) {
  emu_launch(k_final_exp<EmuP>, dim3(1), 1u, reinterpret_cast<const Fp12<EmuP>*>(z), (uint32_t)k, reinterpret_cast<Fp12<EmuP>*>(out));
}
