// Device side of kzg.ToLagrangeG1 (ecc/bn254/kzg/utils.go:25-64; the kzg packages of the other pairing curves are the same
// generated code): the canonical SRS [tau^i]G becomes its Lagrange form [L_i(tau)]G by an inverse FFT whose elements are G1
// points.  Included by engine_impl.cuh (one instantiation per pairing G1 group, with its inst_*.cu field build choices) and by
// the CPU kernel emulation of tests/emu/ (tests/test_emu_lagrange_cpu.py); the launch schedule below is shared by both.
//
//   k_lag_stage   one DIF butterfly per thread, one launch per stage s (difFFTG1, utils.go:119-172):
//                   a <- a + b,  b <- [w^(-j 2^s)](a - b)   (no multiplication for j = 0)
//                 stage 0 reads the affine input, every stage reads and writes a workspace of n extended-Jacobian points
//   k_lag_finish  out[i] = [1/n] ws[bitrev(i)] (bitReverse, utils.go:95-105, then the scaling loop), then the affine normal form
//                 of BatchJacobianToAffineG1: LAG_FIN_M points per thread, one inversion (Montgomery's trick over ZZZ)
//
// The twiddle w^(-j 2^s) is computed per thread from the powers w^(-2^k), k < log2 n, of the domain's inverse root (host side:
// fft.cu, the roots of fr.Generator).  Field arithmetic is exact and every result is fully reduced, so the affine output is
// limb-identical to the reference's whatever the coordinates and the order of the operations.
//
// Cost: a twiddle multiplication is fr.Bits doublings plus about fr.Bits / W additions (thousands of Fp products per point against
// a few hundred bytes moved), so the stages are bound by the multiplier, not by memory traffic.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "kernels.cuh"

namespace gmsm {

// window width W of the twiddle multiplication: signed digits of W bits (partitionScalars' recoding, DigitStream) against a
// per-thread table of [1..2^(W-1)]P.  Chosen per group by an A/B timing of W = 3, 4, 5 (DESIGN.md section 3): 4 for the scalar
// fields of at most 255 bits, 5 for the 315- and 377-bit ones of bw6-633 and bw6-761.  GMSM_LAG_W = w builds a variant with
// W = w for every group.
#ifndef GMSM_LAG_W
#define GMSM_LAG_W 0
#endif
template <class G>
inline constexpr int lag_w = GMSM_LAG_W > 0 ? GMSM_LAG_W : (G::FrParams::BITS > 300 ? 5 : 4);
static constexpr int LAG_FIN_M = 8;      // points per thread of k_lag_finish (one inversion each)

// w^(-2^k) for k < log2 n, Montgomery form; passed by value
template <class G>
struct LagPowers {
  typename G::Fr w[LAG_MAX_LOG];
};

// +-table[|d| - 1] for a non-zero digit code (code_bucket, kernels.cuh): the negative of (X, Y, ZZ, ZZZ) is (X, -Y, ZZ, ZZZ)
template <class F>
GMSM_D XYZZ<F> lag_entry(const XYZZ<F>* tab, uint32_t code) {
  XYZZ<F> t = tab[code_bucket(code)];
  if (code & 1u) t.y = f_neg(t.y);
  return t;
}

// [s]p for a Montgomery-form scalar s (ScalarMultiplication of the reference with s.BigInt).  Digits: DigitStream with c = W
// over fr.Bits / W + 1 windows, so the top window (at most W - 1 bits plus a carry) stays within the table as well.
// Horner from the top non-zero window: W Jacobian doublings (dbl-2009-l, 2M + 5S) and one extended-Jacobian addition of
// +-table entry per window (the Horner step of k_finalize); the addition takes the doubling and cancellation branches.
// W: ToLagrangeG1's lag_w unless a caller of another shape chooses its own (mpc_kernels.cuh).
template <class G, int W = lag_w<G>>
GMSM_D XYZZ<typename G::F> lag_scalar_mul(const XYZZ<typename G::F>& p, const typename G::Fr& s) {
  using F = typename G::F;
  constexpr int NWIN = G::FrParams::BITS / W + 1, NT = 1 << (W - 1);
  static_assert(W >= 2 && W <= 7, "the window codes are stored in bytes");
  if (p.is_inf() || s.is_zero()) return XYZZ<F>::inf();
  uint8_t codes[NWIN];
  {
    DigitStream<G> ds;
    ds.init(s, W, NWIN);
    for (int j = 0; j < NWIN; j++) codes[j] = (uint8_t)ds.next(j);
  }
  XYZZ<F> tab[NT];   // tab[k] = [k + 1]p
  tab[0] = p;
  for (int k = 1; k < NT; k++) {
    tab[k] = tab[k - 1];
    xyzz_add_cold(tab[k], p);
  }
  int j = NWIN - 1;
  while (j >= 0 && codes[j] == 0) j--;
  if (j < 0) return XYZZ<F>::inf();
  XYZZ<F> acc = lag_entry(tab, codes[j]);
  for (j--; j >= 0; j--) {
    Jac<F> dj = xyzz_to_jac(acc);
    for (int l = 0; l < W; l++) dj = jac_double_cold(dj);
    acc = jac_to_xyzz(dj);
    if (codes[j]) xyzz_add_cold(acc, lag_entry(tab, (uint32_t)codes[j]));
  }
  return acc;
}

// stage s of the DIF FFT on n = 2^logn points, one butterfly per thread (n / 2 threads): blocks of 2h points, h = n >> (s + 1);
// thread t takes j = t mod h of block t / h, i.e. points i0 = 2h (t / h) + j and i1 = i0 + h.  FIRST: read (affine) `in`, else ws.
template <class G, bool FIRST>
__global__ void __launch_bounds__(128)
k_lag_stage(const Affine<typename G::F>* __restrict__ in, XYZZ<typename G::F>* __restrict__ ws, uint32_t half_n, int logn, int s,
            LagPowers<G> pw) {
  using F = typename G::F;
  using Fr = typename G::Fr;
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= half_n) return;
  const int lh = logn - 1 - s;
  const uint32_t j = t & ((1u << lh) - 1u);
  const uint32_t i0 = ((t >> lh) << (lh + 1)) | j, i1 = i0 + (1u << lh);
  XYZZ<F> a, b;
  if constexpr (FIRST) {
    a = xyzz_from_affine(load_vec_ro(in + i0));
    b = xyzz_from_affine(load_vec_ro(in + i1));
  } else {
    a = load_vec(ws + i0);
    b = load_vec(ws + i1);
  }
  XYZZ<F> d = b;   // d = a - b
  d.y = f_neg(d.y);
  xyzz_add_cold(d, a);
  xyzz_add_cold(a, b);
  if (j != 0) {
    // w^(-j 2^s) = prod of w^(-2^k) over the set bits k of j 2^s (< n / 2)
    const uint32_t e = j << s;
    Fr w = Fr::one();
    for (int k = s; k < logn - 1; k++)
      if ((e >> k) & 1u) w = f_mul(w, pw.w[k]);
    d = lag_scalar_mul<G>(d, w);
  }
  store_vec(ws + i0, a);
  store_vec(ws + i1, d);
}

// out[i] = affine([n_inv] ws[bitrev(i)]) for LAG_FIN_M consecutive i per thread; infinity is (0, 0).  out may be the input of
// stage 0 (it is not read any more).  logn >= 1.
template <class G>
__global__ void __launch_bounds__(128)
k_lag_finish(const XYZZ<typename G::F>* __restrict__ ws, uint32_t n, int logn, typename G::Fr n_inv, Affine<typename G::F>* __restrict__ out) {
  using F = typename G::F;
  const uint64_t first = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) * LAG_FIN_M;
  if (first >= n) return;
  const int cnt = (n - first < (uint64_t)LAG_FIN_M) ? (int)(n - first) : LAG_FIN_M;
  XYZZ<F> pts[LAG_FIN_M];
  F pref[LAG_FIN_M];
  F prod = F::one();
  for (int i = 0; i < cnt; i++) {
    const uint64_t src = __brevll(first + i) >> (64 - logn);
    const XYZZ<F> p = lag_scalar_mul<G>(load_vec(ws + src), n_inv);
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

// w^(-2^k), k < logn, from the domain's inverse root w_inv = fr.Generator(n)^-1 (computeTwiddlesInv, utils.go:66-93)
template <class G>
LagPowers<G> lag_powers(typename G::Fr w_inv, int logn) {
  LagPowers<G> pw{};
  for (int k = 0; k < logn && k < LAG_MAX_LOG; k++) {
    pw.w[k] = w_inv;
    w_inv = f_sqr(w_inv);
  }
  return pw;
}

// n = 2^logn >= 2: stage(s, threads) for s = 0 .. logn - 1 (n / 2 butterflies each), then finish(threads).
template <class Stage, class Finish>
void lagrange_schedule(uint64_t n, int logn, Stage&& stage, Finish&& finish) {
  for (int s = 0; s < logn; s++) stage(s, n >> 1);
  finish((n + LAG_FIN_M - 1) / LAG_FIN_M);
}

}  // namespace gmsm
