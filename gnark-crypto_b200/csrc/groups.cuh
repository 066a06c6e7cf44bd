// The (curve, group) instantiations on the MultiExp path and their memory sizes: the four of the hot path, then next-row N4.
//   bn254 G1 / G2       ecc/bn254/g1.go:18-30, g2.go:19-31, fr = ecc/bn254/fr (254 bits)
//   bls12-381 G1 / G2   ecc/bls12-381/g1.go, g2.go, fr = ecc/bls12-381/fr (255 bits)
#pragma once
#include "curve.cuh"

namespace gmsm {

template <int ID_, class FP, class FR, bool G2>
struct GroupT;

template <int ID_, class FP, class FR>
struct GroupT<ID_, FP, FR, false> {
  static constexpr int ID = ID_;
  using F = Fp<FP>;
  using Fr = Fp<FR>;
  using FrParams = FR;
};
template <int ID_, class FP, class FR>
struct GroupT<ID_, FP, FR, true> {
  static constexpr int ID = ID_;
  using F = Fp2<FP>;
  using Fr = Fp<FR>;
  using FrParams = FR;
};

// ids are the C-ABI's gmsm_curve_t values (include/gmsm.h)
using bn254_g1 = GroupT<0, bn254_fp, bn254_fr, false>;
using bn254_g2 = GroupT<1, bn254_fp, bn254_fr, true>;
using bls12381_g1 = GroupT<2, bls12381_fp, bls12381_fr, false>;
using bls12381_g2 = GroupT<3, bls12381_fp, bls12381_fr, true>;
// next-row N4 (pure parametrisation): bls12-377 G1, ecc/bls12-377/g1.go, fr 253 bits
using bls12377_g1 = GroupT<4, bls12377_fp, bls12377_fr, false>;
using bls12377_g2 = GroupT<5, bls12377_fp, bls12377_fr, true>;   // Fp2 with u^2 = -5
// N4 remainder: secp256k1 (ecc/secp256k1/g1.go; fp and fr fill all 256 bits: Params::FULL, carry-aware field ops),
// bw6-761 G1 and G2 (ecc/bw6-761/g1.go, g2.go: BOTH over the 12-word Fp; fr = 6 words, 377 bits)
using secp256k1_g1 = GroupT<6, secp256k1_fp, secp256k1_fr, false>;
using bw6761_g1 = GroupT<7, bw6761_fp, bw6761_fr, false>;
using bw6761_g2 = GroupT<8, bw6761_fp, bw6761_fr, false>;
// bls24-315 / bls24-317 G1 (5-word Fp = 10 limbs; G2 of these curves is over Fp4: not on this path), bw6-633 G1 / G2 (10-word Fp,
// both groups over Fp; fr = 5 words, 315 bits: 40-byte scalars)
using bls24315_g1 = GroupT<9, bls24315_fp, bls24315_fr, false>;
using bls24317_g1 = GroupT<10, bls24317_fp, bls24317_fr, false>;
using bw6633_g1 = GroupT<11, bw6633_fp, bw6633_fr, false>;
using bw6633_g2 = GroupT<12, bw6633_fp, bw6633_fr, false>;

// word (u32) counts
template <class G> constexpr int coord_words() { return G::F::N; }
template <class G> constexpr int affine_words() { return 2 * G::F::N; }
template <class G> constexpr int xyzz_words() { return 4 * G::F::N; }
template <class G> constexpr int jac_words() { return 3 * G::F::N; }

// scan tiling (k_scan_* in kernels.cuh; the host sizes block_sums with it)
static constexpr int SCAN_THREADS = 256;
static constexpr int SCAN_ITEMS = 8;                              // per thread
static constexpr int SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;       // per block

// kzg.ToLagrangeG1 (lagrange_kernels.cuh) takes n <= 2^LAG_MAX_LOG points: butterfly and output indices fit in 32 bits
static constexpr int LAG_MAX_LOG = 31;

// ---- window plan (computeNbChunks / lastC, ecc/bn254/multiexp.go:681-693) ----
struct WindowPlan {
  int c;          // window width in bits
  int nwin;       // W = ceil(fr.Bits / c)
  int last_c;     // lastC(c)
  uint32_t nb;    // buckets of a regular window: 2^(c-1)
  uint32_t nb_last;   // buckets of the last window: 2^(last_c-1)
  uint32_t nb_total;  // (W-1)*nb + nb_last
};

inline WindowPlan make_plan(int fr_bits, int c) {
  WindowPlan p;
  p.c = c;
  p.nwin = (fr_bits + c - 1) / c;
  int avail = p.nwin * c - fr_bits;
  p.last_c = c + 1 - avail;
  p.nb = 1u << (c - 1);
  p.nb_last = 1u << (p.last_c - 1);
  p.nb_total = (uint32_t)(p.nwin - 1) * p.nb + p.nb_last;
  return p;
}

}  // namespace gmsm
