// Device side of the G1 point decoding (next-row N2): the kernel of decode.cu and its helpers, in a header of their own so
// that the CPU kernel emulation of tests/emu/ can compile and run them too; decode.cu includes this file verbatim.  See
// decode.cu for the reference citations and the wire format.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "../../include/gmsm.h"
#include "kernels.cuh"

namespace gmsm {

enum { DEC_OK = 0, DEC_BAD_INFINITY = 1, DEC_BAD_ELEMENT = 2, DEC_NO_SQRT = 3, DEC_NOT_ON_CURVE = 4, DEC_BAD_FLAGS = 5 };

template <class P>
struct WireFlags {
  static constexpr int SPARE = 32 * P::N - P::BITS;
  static constexpr bool THREE = SPARE >= 3;
  static constexpr uint32_t MASK = THREE ? (0b111u << 5) : (0b11u << 6);
  static constexpr uint32_t UNC = 0;
  static constexpr uint32_t UNC_INF = THREE ? (0b010u << 5) : 0xFFFFu;     // (none for bn254)
  static constexpr uint32_t SMALL = THREE ? (0b100u << 5) : (0b10u << 6);
  static constexpr uint32_t LARGE = THREE ? (0b101u << 5) : (0b11u << 6);
  static constexpr uint32_t INF = THREE ? (0b110u << 5) : (0b01u << 6);
};

// per-field constants of the decoder, computed once on the host (make_decode_consts): the curve's b (Montgomery form; it is
// q - 1 for bw6-761) and those of the square root.  q - 1 = 2^s * t with t odd; z_t = z^t for a quadratic non-residue z;
// e = (t - 1) / 2 as little-endian 32-bit limbs.
template <class P>
struct DecodeConsts {
  Fp<P> b;
  Fp<P> z_t;
  uint32_t e[P::N];
  int s;
};

// big-endian bytes -> little-endian 32-bit limbs (canonical integer), top byte masked with `keep`
template <class P>
GMSM_D Fp<P> read_be(const uint8_t* b, uint32_t keep) {
  constexpr int N = P::N;
  Fp<P> r;
#pragma unroll
  for (int k = 0; k < N; k++) {
    const uint8_t* q = b + 4 * (N - 1 - k);
    uint32_t v = ((uint32_t)q[0] << 24) | ((uint32_t)q[1] << 16) | ((uint32_t)q[2] << 8) | (uint32_t)q[3];
    if (k == N - 1) v &= (keep << 24) | 0x00FFFFFFu;
    r.l[k] = v;
  }
  return r;
}
template <class P>
GMSM_D bool below_modulus(const Fp<P>& a) {   // smallerThanModulus, fp/element.go:347-349
  for (int i = P::N - 1; i >= 0; i--) {
    if (a.l[i] < P::mod(i)) return true;
    if (a.l[i] > P::mod(i)) return false;
  }
  return false;
}
// canonical value > (q - 1) / 2  <=>  2 * value > q - 1  <=>  2 * value >= q + 1 ... evaluated as value >= (q + 1) / 2
template <class P>
GMSM_D bool lexicographically_largest(const Fp<P>& y_mont) {
  const Fp<P> y = fp_from_mont(y_mont);
  // h = (q + 1) / 2 (q odd): q >> 1, plus one
  uint32_t h[P::N];
#pragma unroll
  for (int i = 0; i < P::N; i++) h[i] = (P::mod(i) >> 1) | ((i + 1 < P::N ? P::mod(i + 1) : 0u) << 31);
  uint32_t carry = 1;
#pragma unroll
  for (int i = 0; i < P::N; i++) { const uint32_t s = h[i] + carry; carry = (s < carry) ? 1u : 0u; h[i] = s; }
  for (int i = P::N - 1; i >= 0; i--) {
    if (y.l[i] > h[i]) return true;
    if (y.l[i] < h[i]) return false;
  }
  return true;
}

// x^e for an exponent of P::N little-endian 32-bit limbs (left to right square-and-multiply)
template <class P>
GMSM_HD Fp<P> fp_pow_limbs(const Fp<P>& x, const uint32_t* e) {
  Fp<P> acc = Fp<P>::one();
  bool started = false;
  for (int i = 32 * P::N - 1; i >= 0; i--) {
    if (started) acc = fp_sqr(acc);
    if ((e[i >> 5] >> (i & 31)) & 1u) {
      acc = started ? fp_mul(acc, x) : x;
      started = true;
    }
  }
  return acc;
}

// Tonelli-Shanks: a root of a when a is a square; otherwise some value whose square is not a (the caller checks).  Any
// root serves, LexicographicallyLargest picks the sign afterwards.  For q = 3 mod 4 (s = 1) it is a^((q+1)/4), fp.Sqrt of
// fp/element.go:1142-1153; for q = 1 mod 4 (bls12-377: s = 46, bls24-315: s = 20, bw6-633: s = 2) the loop runs at most
// s - 1 rounds of at most s - 1 squarings each.
template <class P>
GMSM_HD Fp<P> fp_sqrt_ts(const Fp<P>& a, const DecodeConsts<P>& k) {
  using F = Fp<P>;
  if (a.is_zero()) return a;
  const F w = fp_pow_limbs(a, k.e);       // a^((t-1)/2)
  F r = fp_mul(a, w);                     // a^((t+1)/2)
  F b = fp_mul(r, w);                     // a^t: in the subgroup of order 2^s; r^2 = a * b
  F c = k.z_t;
  const F one = F::one();
  int m = k.s;
  while (!(b == one)) {
    int i = 0;                            // least i with b^(2^i) = 1
    F b2 = b;
    while (i < m && !(b2 == one)) { b2 = fp_sqr(b2); i++; }
    if (i >= m) break;                    // a is a non-residue
    F g = c;
    for (int j = 0; j < m - i - 1; j++) g = fp_sqr(g);
    r = fp_mul(r, g);
    c = fp_sqr(g);
    b = fp_mul(b, c);
    m = i;
  }
  return r;
}

// host: the constants of DecodeConsts for the curve y^2 = x^3 + b with b = b_small, or -b_small when b_negative
template <class P>
DecodeConsts<P> make_decode_consts(uint32_t b_small, bool b_negative) {
  using F = Fp<P>;
  constexpr int N = P::N;
  DecodeConsts<P> k;
  F b = F::zero();
  b.l[0] = b_small;
  b = fp_to_mont(b);
  k.b = b_negative ? fp_neg(b) : b;
  // t = (q - 1) >> s (q odd: subtracting 1 clears bit 0 without a borrow)
  uint32_t t[N];
  for (int i = 0; i < N; i++) t[i] = P::mod(i);
  t[0] -= 1;
  int s = 0;
  while ((t[0] & 1u) == 0) {
    for (int i = 0; i < N; i++) t[i] = (t[i] >> 1) | ((i + 1 < N ? t[i + 1] : 0u) << 31);
    s++;
  }
  k.s = s;
  for (int i = 0; i < N; i++) k.e[i] = (t[i] >> 1) | ((i + 1 < N ? t[i + 1] : 0u) << 31);   // (t - 1) / 2 = t >> 1 (t odd)
  // z: the smallest integer >= 2 with z^((q-1)/2) = -1 (Euler's criterion); (q - 1) / 2 = t * 2^(s-1)
  const F minus_one = fp_neg(F::one());
  for (uint32_t zi = 2;; zi++) {
    F z = F::zero();
    z.l[0] = zi;
    z = fp_to_mont(z);
    const F ze = fp_pow_limbs(z, k.e);
    const F zt = fp_mul(fp_sqr(ze), z);   // z^(2e + 1) = z^t
    F l = zt;
    for (int j = 0; j < s - 1; j++) l = fp_sqr(l);
    if (l == minus_one) { k.z_t = zt; break; }
  }
  return k;
}

template <class P>
__global__ void __launch_bounds__(128)
k_g1_decode(const uint8_t* __restrict__ bytes, uint32_t n, int raw, int check_curve, DecodeConsts<P> kc, Affine<Fp<P>>* __restrict__ out,
            unsigned long long* __restrict__ first_error) {
  using F = Fp<P>;
  using W = WireFlags<P>;
  constexpr int NB = 4 * P::N;
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint8_t* b = bytes + (size_t)i * (raw ? 2 * NB : NB);
  const uint32_t m = b[0] & W::MASK;
  int err = DEC_OK;
  Affine<F> pt = Affine<F>::inf();
  // a stream is homogeneous: raw = 1 holds uncompressed points, raw = 0 compressed ones.  A point is infinity only under its
  // own stream kind's flag, whose payload is exactly the point's stride (bn254 has no raw infinity flag: its raw infinity is
  // the all-zero point, which decodes to (0, 0) below); every other pattern is DEC_BAD_FLAGS.
  const bool is_inf = raw ? (m == W::UNC_INF) : (m == W::INF);
  if (is_inf) {
    const int len = raw ? 2 * NB : NB;
    uint32_t any = b[0] & ~W::MASK & 0xFFu;
    for (int k = 1; k < len; k++) any |= b[k];
    if (any) err = DEC_BAD_INFINITY;
  } else if ((raw && m != W::UNC) || (!raw && m != W::SMALL && m != W::LARGE)) {
    err = DEC_BAD_FLAGS;
  } else {
    const F xc = read_be<P>(b, ~W::MASK & 0xFFu);
    if (!below_modulus(xc)) err = DEC_BAD_ELEMENT;
    const F X = fp_to_mont(xc);
    const F rhs = fp_add(fp_mul(fp_sqr(X), X), kc.b);       // x^3 + b   (marshal.go:925-927)
    if (raw) {
      const F yc = read_be<P>(b + NB, 0xFFu);
      if (!below_modulus(yc)) err = DEC_BAD_ELEMENT;
      const F Y = fp_to_mont(yc);
      if (!err && check_curve && !(fp_sqr(Y) == rhs) && !(xc.is_zero() && yc.is_zero())) err = DEC_NOT_ON_CURVE;
      pt.x = X;
      pt.y = Y;
    } else {
      F Y = fp_sqrt_ts(rhs, kc);
      if (!err && !(fp_sqr(Y) == rhs)) err = DEC_NO_SQRT;       // fp.Sqrt returns nil, marshal.go:928-930
      const bool largest = lexicographically_largest(Y);
      if (largest != (m == W::LARGE)) Y = fp_neg(Y);            // marshal.go:932-942
      pt.x = X;
      pt.y = Y;
    }
  }
  if (err) {
    atomicMin(first_error, ((unsigned long long)i << 8) | (unsigned long long)err);
    pt = Affine<F>::inf();
  }
  store_vec(out + i, pt);
}

// calls fn(P-typed DecodeConsts) for a G1 group id (gmsm_curve_t); returns -1 for any other id.  y^2 = x^3 + b with b:
// bn254 3, bls12-381 4, bls12-377 1, bls24-315 1, bls24-317 4, bw6-633 4, bw6-761 -1 (the curves' .go files).
template <class Fn>
int with_g1_decode_consts(int curve, Fn&& fn) {
  switch (curve) {
    case GMSM_BN254_G1: return fn(make_decode_consts<bn254_fp>(3, false));
    case GMSM_BLS12381_G1: return fn(make_decode_consts<bls12381_fp>(4, false));
    case GMSM_BLS12377_G1: return fn(make_decode_consts<bls12377_fp>(1, false));
    case GMSM_BLS24315_G1: return fn(make_decode_consts<bls24315_fp>(1, false));
    case GMSM_BLS24317_G1: return fn(make_decode_consts<bls24317_fp>(4, false));
    case GMSM_BW6633_G1: return fn(make_decode_consts<bw6633_fp>(4, false));
    case GMSM_BW6761_G1: return fn(make_decode_consts<bw6761_fp>(1, true));
  }
  return -1;
}

}  // namespace gmsm
