// Device side of the G2 point decoding and of the point encoding of the twelve pairing groups (next-row N2): the kernels of
// decode.cu and their helpers, in a header of their own so that the CPU kernel emulation of tests/emu/ can compile and run them
// too.  See decode.cu for the reference citations and the wire format.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <type_traits>

#include "decode_kernels.cuh"

namespace gmsm {

// per-field constants of the G2 decoder over Fp2 = Fp[u]/(u^2 - beta), computed once on the host (make_g2_decode_consts): the
// square-root constants of Fp, the twist's b' (Montgomery form), 1/beta and 1/2
template <class P>
struct G2DecodeConsts {
  DecodeConsts<P> fp;   // fp.b is unused
  Fp2<P> b;
  Fp<P> inv_beta;
  Fp<P> half;
};

// whether a is a square in Fp, with a root in r when it is
template <class P>
GMSM_HD bool fp_sqrt_checked(const Fp<P>& a, const DecodeConsts<P>& k, Fp<P>& r) {
  r = fp_sqrt_ts(a, k);
  return fp_sqr(r) == a;
}

// a square root of a in Fp2 by the complex method; returns false when there is none, decided by the norm a0^2 - beta a1^2 as
// E2.Legendre decides it (internal/fptower/e2.go).  Any root serves: the caller fixes the sign.
//   a1 = 0: a0 itself when it is a square, else c u with c^2 = a0 / beta (beta is a non-residue, so a0 / beta is a square);
//   a1 != 0: alpha = sqrt(norm); exactly one of (a0 +- alpha) / 2 is a square (their product is beta a1^2 / 4, a non-residue
//   times a square), call it delta != 0; the root is x0 + x1 u with x0 = sqrt(delta), x1 = a1 / (2 x0).
template <class P>
GMSM_HD bool fp2_sqrt(const Fp2<P>& a, const G2DecodeConsts<P>& k, Fp2<P>& r) {
  using F = Fp<P>;
  F s;
  if (a.a1.is_zero()) {
    if (fp_sqrt_checked(a.a0, k.fp, s)) {
      r = Fp2<P>{s, F::zero()};
    } else {
      fp_sqrt_checked(fp_mul(a.a0, k.inv_beta), k.fp, s);
      r = Fp2<P>{F::zero(), s};
    }
    return true;
  }
  F t = fp_sqr(a.a1);
  if (P::FP2_NONRES == -5) t = fp_mul_by5(t);
  F alpha;
  if (!fp_sqrt_checked(fp_add(fp_sqr(a.a0), t), k.fp, alpha)) return false;
  if (!fp_sqrt_checked(fp_mul(fp_add(a.a0, alpha), k.half), k.fp, s)) fp_sqrt_checked(fp_mul(fp_sub(a.a0, alpha), k.half), k.fp, s);
  r = Fp2<P>{s, fp_mul(a.a1, fp_inv(fp_dbl(s)))};
  return true;
}

// E2.LexicographicallyLargest: A1 decides, or A0 when A1 = 0
template <class P>
GMSM_D bool coord_largest(const Fp2<P>& y) {
  return y.a1.is_zero() ? lexicographically_largest(y.a0) : lexicographically_largest(y.a1);
}
template <class P>
GMSM_D bool coord_largest(const Fp<P>& y) {
  return lexicographically_largest(y);
}

// bytes -> G2Affine over Fp2, the twin of k_g1_decode: wire order X.A1 || X.A0 (|| Y.A1 || Y.A0), flags in the top byte of X.A1,
// the same homogeneous-stream rule, error codes and first-error folding
template <class P>
__global__ void __launch_bounds__(128)
k_g2_decode(const uint8_t* __restrict__ bytes, uint32_t n, int raw, int check_curve, G2DecodeConsts<P> kc, Affine<Fp2<P>>* __restrict__ out,
            unsigned long long* __restrict__ first_error) {
  using F = Fp<P>;
  using E = Fp2<P>;
  using W = WireFlags<P>;
  constexpr int NB = 4 * P::N;
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int len = raw ? 4 * NB : 2 * NB;
  const uint8_t* b = bytes + (size_t)i * len;
  const uint32_t m = b[0] & W::MASK;
  int err = DEC_OK;
  Affine<E> pt = Affine<E>::inf();
  const bool is_inf = raw ? (m == W::UNC_INF) : (m == W::INF);
  if (is_inf) {
    uint32_t any = b[0] & ~W::MASK & 0xFFu;
    for (int k = 1; k < len; k++) any |= b[k];
    if (any) err = DEC_BAD_INFINITY;
  } else if ((raw && m != W::UNC) || (!raw && m != W::SMALL && m != W::LARGE)) {
    err = DEC_BAD_FLAGS;
  } else {
    const F x1 = read_be<P>(b, ~W::MASK & 0xFFu);
    const F x0 = read_be<P>(b + NB, 0xFFu);
    if (!below_modulus(x1) || !below_modulus(x0)) err = DEC_BAD_ELEMENT;
    const E X{fp_to_mont(x0), fp_to_mont(x1)};
    const E rhs = f_add(f_mul(f_sqr(X), X), kc.b);           // X^3 + b'   (marshal.go:1175-1176)
    E Y = E::zero();
    if (raw) {
      const F y1 = read_be<P>(b + 2 * NB, 0xFFu);
      const F y0 = read_be<P>(b + 3 * NB, 0xFFu);
      if (!below_modulus(y1) || !below_modulus(y0)) err = DEC_BAD_ELEMENT;
      Y = E{fp_to_mont(y0), fp_to_mont(y1)};
      if (!err && check_curve && !(f_sqr(Y) == rhs) && !(X.is_zero() && Y.is_zero())) err = DEC_NOT_ON_CURVE;
    } else {
      if (!fp2_sqrt(rhs, kc, Y)) {
        if (!err) err = DEC_NO_SQRT;                              // E2.Legendre == -1, marshal.go:1177-1179
      } else if (coord_largest(Y) != (m == W::LARGE)) {
        Y = f_neg(Y);                                             // marshal.go:1182-1192
      }
    }
    pt.x = X;
    pt.y = Y;
  }
  if (err) {
    atomicMin(first_error, ((unsigned long long)i << 8) | (unsigned long long)err);
    pt = Affine<E>::inf();
  }
  store_vec(out + i, pt);
}

// ---- encoding: G1Affine / G2Affine Bytes and RawBytes ----
constexpr int ENC_THREADS = 128;

// a coordinate's base-field elements in wire order (A1 before A0)
template <class P>
GMSM_D void wire_elems(const Fp<P>& a, Fp<P>* e) { e[0] = a; }
template <class P>
GMSM_D void wire_elems(const Fp2<P>& a, Fp<P>* e) { e[0] = a.a1; e[1] = a.a0; }

GMSM_D uint32_t bswap32(uint32_t v) { return (v >> 24) | ((v >> 8) & 0xFF00u) | ((v << 8) & 0xFF0000u) | (v << 24); }

// One thread per point: the point's bytes are assembled in shared memory (a row per thread, padded to an odd number of words
// so that the rows of a warp fall in distinct banks), then the block's contiguous output is written by consecutive threads
// with consecutive 32-bit stores.  D = 1 (Fp) or 2 (Fp2) elements per coordinate; RAW: X || Y, else X with the flags.
template <class P, int D, int RAW>
__global__ void __launch_bounds__(ENC_THREADS)
k_points_encode(const Affine<std::conditional_t<D == 1, Fp<P>, Fp2<P>>>* __restrict__ pts, uint32_t n, uint32_t* __restrict__ out) {
  using W = WireFlags<P>;
  constexpr int N = P::N;
  constexpr int NE = (RAW ? 2 : 1) * D;                 // base-field elements per encoded point
  constexpr int PW = NE * N;                            // 32-bit words per encoded point
  constexpr int RS = PW | 1;                            // shared-memory row stride
  __shared__ uint32_t stage[ENC_THREADS * RS];
  const uint32_t first = blockIdx.x * ENC_THREADS;
  const uint32_t i = first + threadIdx.x;
  if (i < n) {
    const auto p = load_vec_ro(pts + i);
    uint32_t* row = stage + threadIdx.x * RS;
    if (p.is_inf()) {
      // Bytes: mCompressedInfinity; RawBytes: mUncompressedInfinity, or all zeroes on bn254 (marshal.go:801-846, :1051-1100)
      const uint32_t flag = RAW ? (W::THREE ? W::UNC_INF : W::UNC) : W::INF;
#pragma unroll
      for (int k = 0; k < PW; k++) row[k] = 0;
      row[0] = bswap32(flag << 24);
    } else {
      Fp<P> e[NE];
      wire_elems(p.x, e);
      if (RAW) wire_elems(p.y, e + D);
#pragma unroll
      for (int j = 0; j < NE; j++) {
        const Fp<P> c = fp_from_mont(e[j]);
#pragma unroll
        for (int k = 0; k < N; k++) row[j * N + k] = bswap32(c.l[N - 1 - k]);
      }
      if (!RAW) row[0] |= bswap32((coord_largest(p.y) ? W::LARGE : W::SMALL) << 24);
    }
  }
  __syncthreads();
  const uint32_t cnt = n - first < (uint32_t)ENC_THREADS ? n - first : (uint32_t)ENC_THREADS;
  uint32_t* dst = out + (size_t)first * PW;
  for (uint32_t t = threadIdx.x; t < cnt * PW; t += ENC_THREADS) dst[t] = stage[(t / PW) * RS + t % PW];
}

// ---- host helpers shared by decode.cu and the emulation ----
// host: the G2 decoder's constants for the twist y^2 = x^3 + b' over Fp2 (b' = b_num / (d0 + d1 u), or b_num (d0 + d1 u) when
// !divide)
template <class P>
G2DecodeConsts<P> make_g2_decode_consts(uint32_t b_num, uint32_t d0, uint32_t d1, bool divide) {
  using F = Fp<P>;
  auto small = [](uint32_t v) { F x = F::zero(); x.l[0] = v; return fp_to_mont(x); };
  G2DecodeConsts<P> k;
  k.fp = make_decode_consts<P>(1, false);
  const Fp2<P> d{small(d0), small(d1)};
  const Fp2<P> t = divide ? f_inv(d) : d;
  k.b = Fp2<P>{fp_mul(t.a0, small(b_num)), fp_mul(t.a1, small(b_num))};
  k.inv_beta = fp_inv(fp_neg(small((uint32_t)(-P::FP2_NONRES))));
  k.half = fp_inv(small(2));
  return k;
}

// the G2 group ids with a decoder
inline bool is_g2_decode_group(int curve) {
  return curve == GMSM_BN254_G2 || curve == GMSM_BLS12381_G2 || curve == GMSM_BLS12377_G2 || curve == GMSM_BW6761_G2 ||
         curve == GMSM_BW6633_G2;
}

// calls fn with the decoder constants of a G2 group id: G2DecodeConsts for the groups over Fp2, DecodeConsts (the G1 decoder's,
// with the twist's b) for the two bw6 groups over Fp; returns -1 for any other id.  bTwistCurveCoeff: bn254 3 / (9 + u),
// bls12-381 4 (1 + u), bls12-377 1 / u, bw6-761 4, bw6-633 8 (the curves' .go files).
template <class Fn>
int with_g2_decode_consts(int curve, Fn&& fn) {
  switch (curve) {
    case GMSM_BN254_G2: return fn(make_g2_decode_consts<bn254_fp>(3, 9, 1, true));
    case GMSM_BLS12381_G2: return fn(make_g2_decode_consts<bls12381_fp>(4, 1, 1, false));
    case GMSM_BLS12377_G2: return fn(make_g2_decode_consts<bls12377_fp>(1, 0, 1, true));
    case GMSM_BW6761_G2: return fn(make_decode_consts<bw6761_fp>(4, false));
    case GMSM_BW6633_G2: return fn(make_decode_consts<bw6633_fp>(8, false));
  }
  return -1;
}

template <class P, int D>
struct EncodeGroup {
  using Params = P;
  static constexpr int degree = D;
};

// calls fn(EncodeGroup<P, D>{}) for a G1 or G2 group of the seven pairing curves; returns -1 for any other id (secp256k1 too)
template <class Fn>
int with_encode_group(int curve, Fn&& fn) {
  switch (curve) {
    case GMSM_BN254_G1: return fn(EncodeGroup<bn254_fp, 1>{});
    case GMSM_BN254_G2: return fn(EncodeGroup<bn254_fp, 2>{});
    case GMSM_BLS12381_G1: return fn(EncodeGroup<bls12381_fp, 1>{});
    case GMSM_BLS12381_G2: return fn(EncodeGroup<bls12381_fp, 2>{});
    case GMSM_BLS12377_G1: return fn(EncodeGroup<bls12377_fp, 1>{});
    case GMSM_BLS12377_G2: return fn(EncodeGroup<bls12377_fp, 2>{});
    case GMSM_BW6761_G1: case GMSM_BW6761_G2: return fn(EncodeGroup<bw6761_fp, 1>{});
    case GMSM_BLS24315_G1: return fn(EncodeGroup<bls24315_fp, 1>{});
    case GMSM_BLS24317_G1: return fn(EncodeGroup<bls24317_fp, 1>{});
    case GMSM_BW6633_G1: case GMSM_BW6633_G2: return fn(EncodeGroup<bw6633_fp, 1>{});
  }
  return -1;
}

}  // namespace gmsm
