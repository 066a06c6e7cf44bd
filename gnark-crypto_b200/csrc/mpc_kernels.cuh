// Device side of the point updates of a trusted-setup contribution (ecc/bn254/mpcsetup/mpcsetup.go; the mpcsetup packages of the
// other pairing curves are the same generated code): out[i] = [c r^(start + i)] points[i], the one form of
//   UpdateMonomialsG1 / G2 (mpcsetup.go:365-381)   c = r on A[1:]
//   the alpha tau^i / beta tau^i slices            c = alpha (or beta), r = tau
//   the slice loop of UpdateValues (:64-81)        r = 1
// Included by engine_impl.cuh (one instantiation per group, with its inst_*.cu field build choices) and by the CPU kernel
// emulation of tests/emu/ (tests/test_emu_mpcsetup_cpu.py); the launch schedule below is shared by both.
//
//   k_scale_powers  SCALE_M consecutive points per thread: the thread's first scalar c r^(start + first) from the powers r^(2^k)
//                   (one product per set bit of `first`), then one product by r per point; each point through lag_scalar_mul (the
//                   variable-base ladder of ToLagrangeG1), then the affine normal form of BatchJacobianToAffineG1 with one
//                   inversion per thread (Montgomery's trick over ZZZ, as k_lag_finish).  out may equal points: a thread reads
//                   its own points before it writes them, and no other thread touches them.
//
// The reference runs one ScalarMultiplication (GLV on G1 / G2) per point; here the scalar multiplication is a signed-window
// double-and-add, fr.Bits doublings per point, so the kernel is bound by the multiplier, not by memory traffic.  Field arithmetic
// is exact and every result fully reduced: the affine output is limb-identical to the reference's.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <cstring>

#include "lagrange_kernels.cuh"

namespace gmsm {

// window width of lag_scalar_mul here, chosen by an A/B timing of W = 3, 4, 5 (tools/time_mpcsetup.py --ab, DESIGN.md section 3):
// ToLagrangeG1's 4 for the groups with 8-limb coordinates (bn254 G1, secp256k1), 5 for every larger coordinate (bls12-381 G1 and
// bn254 G2 were 2-3 % faster at W = 5; bw6-633 and bw6-761 have 5 already).  GMSM_SCALE_W = w builds a variant with W = w for
// every group.
#ifndef GMSM_SCALE_W
#define GMSM_SCALE_W 0
#endif
template <class G>
inline constexpr int scale_w = GMSM_SCALE_W > 0 ? GMSM_SCALE_W : (G::F::N > 8 ? 5 : lag_w<G>);
static constexpr int SCALE_M = 8;          // points per thread (one inversion each)
static constexpr int SCALE_MAX_LOG = 32;   // n < 2^32 per launch: `first` has at most 32 bits

// c r^start and r^(2^k), k < 32, Montgomery form; passed by value
template <class G>
struct ScalePowers {
  typename G::Fr c;
  typename G::Fr r[SCALE_MAX_LOG];
};

template <class G>
__global__ void __launch_bounds__(128)
k_scale_powers(const Affine<typename G::F>* points, uint32_t n, ScalePowers<G> pw, Affine<typename G::F>* out) {
  using F = typename G::F;
  using Fr = typename G::Fr;
  const uint64_t first = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) * SCALE_M;
  if (first >= n) return;
  const int cnt = (n - first < (uint64_t)SCALE_M) ? (int)(n - first) : SCALE_M;
  Fr s = pw.c;   // c r^(start + first)
  for (int k = 0; k < SCALE_MAX_LOG; k++)
    if ((first >> k) & 1u) s = f_mul(s, pw.r[k]);
  XYZZ<F> pts[SCALE_M];
  F pref[SCALE_M];
  F prod = F::one();
  for (int i = 0; i < cnt; i++) {
    const XYZZ<F> p = lag_scalar_mul<G, scale_w<G>>(xyzz_from_affine(load_vec(points + first + i)), s);
    s = f_mul(s, pw.r[0]);
    pts[i] = p;
    pref[i] = prod;   // product of the ZZZ of the finite points before i
    if (!p.is_inf()) prod = f_mul(prod, p.zzz);
  }
  F inv = f_inv(prod);
  for (int i = cnt - 1; i >= 0; i--) {
    Affine<F> a = Affine<F>::inf();
    if (!pts[i].is_inf()) {
      const F i3 = f_mul(inv, pref[i]);   // 1 / ZZZ_i
      inv = f_mul(inv, pts[i].zzz);
      const F i2 = f_mul(f_sqr(pts[i].zz), f_sqr(i3));   // 1 / ZZ_i = ZZ_i^2 / ZZZ_i^2
      a.x = f_mul(pts[i].x, i2);
      a.y = f_mul(pts[i].y, i3);
    }
    store_vec(out + first + i, a);
  }
}

// ---- launch schedule (host), shared by engine_impl.cuh and the CPU emulation ----

// the kernel's scalars for out[i] = [c r^(start + i)] points[i]: c r^start (square-and-multiply over the bits of start) and
// r^(2^k), from reduced Montgomery limbs
template <class G>
ScalePowers<G> scale_powers_args(const uint64_t* c, const uint64_t* r, uint64_t start) {
  using Fr = typename G::Fr;
  ScalePowers<G> pw{};
  Fr rr;
  memcpy(pw.c.l, c, sizeof(Fr));
  memcpy(rr.l, r, sizeof(Fr));
  for (int k = 0; k < 64; k++) {   // rr = r^(2^k)
    if (k < SCALE_MAX_LOG) pw.r[k] = rr;
    if ((start >> k) & 1u) pw.c = f_mul(pw.c, rr);
    rr = f_sqr(rr);
  }
  return pw;
}

// 1 <= n < 2^32 points: one launch of ceil(n / SCALE_M) threads
template <class Launch>
void scale_powers_schedule(uint64_t n, Launch&& launch) {
  launch((n + SCALE_M - 1) / SCALE_M);
}

}  // namespace gmsm
