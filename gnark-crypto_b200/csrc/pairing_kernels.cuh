// Multi-pair Miller loop, GT product tree and final exponentiation of bn254 and bls12-381 (pairing.cu).
//
// Replaces (reference): ecc/bn254/pairing.go (FinalExponentiation :52, MillerLoop :111, doubleStep, addMixedStep, lineCompute)
// and ecc/bls12-381/pairing.go (FinalExponentiation, MillerLoop :103-233, doubleStep, addMixedStep, tangentLine).
//
// The reference runs one loop over all pairs with shared squarings of the accumulator.  Squaring distributes over the product,
// so that accumulator equals the product of the per-pair Miller functions, and every field value is unique: k_miller_loop runs
// one pair per thread (the reference's projective line formulas, infinity skipped as the value 1) and k_gt_reduce multiplies the
// per-pair values pairwise into one, limb-identical to the reference whatever the split.  Device memory is bounded by running
// the pairs in chunks of PAIRING_CHUNK: each chunk is reduced to one value and multiplied into an accumulator
// (pairing_schedule).  k_final_exp multiplies k values and raises the product to the reference's exponent in one thread.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "curve.cuh"
#include "tower.cuh"

namespace gmsm {

template <class P>
struct G2Proj {
  Fp2<P> x, y, z;
};
template <class P>
struct Line {
  Fp2<P> r0, r1, r2;
};
template <class P>
constexpr bool is_dtwist() { return std::is_same<P, bn254_fp>::value; }

// g2Proj.doubleStep: the point doubles; the tangent line is (-H, 3 J, I) (bn254) or (I, 3 J, -H) (bls12-381)
template <class P>
GMSM_TOWER Line<P> double_step(G2Proj<P>& p) {
  const Fp2<P> A = e2_halve(f_mul(p.x, p.y));
  const Fp2<P> B = f_sqr(p.y);
  const Fp2<P> C = f_sqr(p.z);
  const Fp2<P> D = f_add(f_dbl(C), C);
  const Fp2<P> E = f_mul(D, btwist<P>());
  const Fp2<P> F = f_add(f_dbl(E), E);
  const Fp2<P> G = e2_halve(f_add(B, F));
  const Fp2<P> H = f_sub(f_sqr(f_add(p.y, p.z)), f_add(B, C));
  const Fp2<P> I = f_sub(E, B);
  const Fp2<P> J = f_sqr(p.x);
  const Fp2<P> EE = f_sqr(E);
  const Fp2<P> K = f_add(f_dbl(EE), EE);
  p.x = f_mul(f_sub(B, F), A);
  p.y = f_sub(f_sqr(G), K);
  p.z = f_mul(B, H);
  const Fp2<P> J3 = f_add(f_dbl(J), J);
  if constexpr (is_dtwist<P>()) return Line<P>{f_neg(H), J3, I};
  else return Line<P>{I, J3, f_neg(H)};
}
// tangentLine (bls12-381): the line of double_step without moving the point
template <class P>
GMSM_HD Line<P> tangent_line(const G2Proj<P>& p) {
  G2Proj<P> t = p;
  return double_step(t);
}
// lineCompute: the line through p and a, (L, -O, J) (bn254) or (J, -O, L) (bls12-381)
template <class P>
GMSM_HD Line<P> line_compute(const G2Proj<P>& p, const Affine<Fp2<P>>& a, Fp2<P>* O_out = nullptr, Fp2<P>* L_out = nullptr) {
  const Fp2<P> O = f_sub(p.y, f_mul(a.y, p.z));
  const Fp2<P> L = f_sub(p.x, f_mul(a.x, p.z));
  const Fp2<P> J = f_sub(f_mul(a.x, O), f_mul(L, a.y));
  if (O_out) *O_out = O;
  if (L_out) *L_out = L;
  if constexpr (is_dtwist<P>()) return Line<P>{L, f_neg(O), J};
  else return Line<P>{J, f_neg(O), L};
}
// addMixedStep: p += a and the line through them
template <class P>
GMSM_TOWER Line<P> add_mixed_step(G2Proj<P>& p, const Affine<Fp2<P>>& a) {
  Fp2<P> O, L;
  const Line<P> l = line_compute(p, a, &O, &L);
  const Fp2<P> C = f_sqr(O);
  const Fp2<P> D = f_sqr(L);
  const Fp2<P> E = f_mul(L, D);
  const Fp2<P> F = f_mul(p.z, C);
  const Fp2<P> G = f_mul(p.x, D);
  const Fp2<P> H = f_sub(f_add(E, F), f_dbl(G));
  const Fp2<P> t1 = f_mul(p.y, E);
  p.x = f_mul(L, H);
  p.y = f_sub(f_mul(f_sub(G, H), O), t1);
  p.z = f_mul(E, p.z);
  return l;
}
// the line evaluated at P: bn254 r0 *= P.y, r1 *= P.x; bls12-381 r1 *= P.x, r2 *= P.y
template <class P>
GMSM_HD Line<P> scale_line(Line<P> l, const Affine<Fp<P>>& q) {
  if constexpr (is_dtwist<P>()) {
    l.r0 = e2_by_fp(l.r0, q.y);
    l.r1 = e2_by_fp(l.r1, q.x);
  } else {
    l.r1 = e2_by_fp(l.r1, q.x);
    l.r2 = e2_by_fp(l.r2, q.y);
  }
  return l;
}
template <class P>
GMSM_TOWER Fp12<P> mul_line(const Fp12<P>& f, const Line<P>& l) {
  if constexpr (is_dtwist<P>()) return e12_mul_by_034(f, l.r0, l.r1, l.r2);
  else return e12_mul_by_014(f, l.r0, l.r1, l.r2);
}
template <class P>
GMSM_TOWER Fp12<P> mul_two_lines(const Fp12<P>& f, const Line<P>& a, const Line<P>& b) {
  Fp2<P> z[5];
  if constexpr (is_dtwist<P>()) {
    e2_mul_034_by_034(a.r0, a.r1, a.r2, b.r0, b.r1, b.r2, z);
    return e12_mul_by_01234(f, z);
  } else {
    e2_mul_014_by_014(a.r0, a.r1, a.r2, b.r0, b.r1, b.r2, z);
    return e12_mul_by_01245(f, z);
  }
}

// the Miller function of one pair (P, Q), neither at infinity; bls12-381's final conjugation included
template <class P>
GMSM_TOWER Fp12<P> miller_loop_one(const Affine<Fp<P>>& p, const Affine<Fp2<P>>& q) {
  using T = typename TowerOf<P>::T;
  G2Proj<P> r{q.x, q.y, Fp2<P>::one()};
  Fp12<P> f = Fp12<P>::one();
  if constexpr (is_dtwist<P>()) {
    const Affine<Fp2<P>> qn{q.x, f_neg(q.y)};
    f = mul_line(f, scale_line(double_step(r), p));
    f = e12_sqr(f);
    {
      const Line<P> l2 = scale_line(line_compute(r, qn), p);
      const Line<P> l1 = scale_line(add_mixed_step(r, q), p);
      f = mul_two_lines(f, l1, l2);
    }
    for (int i = T::LOOP_LEN - 4; i >= 0; i--) {
      f = e12_sqr(f);
      const Line<P> l1 = scale_line(double_step(r), p);
      const int d = T::loop(i);
      if (d == 0) {
        f = mul_line(f, l1);
      } else {
        const Line<P> l2 = scale_line(add_mixed_step(r, d == 1 ? q : qn), p);
        f = mul_two_lines(f, l1, l2);
      }
    }
    // Q1 = pi(Q), Q2 = -pi^2(Q)
    const Affine<Fp2<P>> q1{f_mul(e2_conj(q.x), frob_coeff<P>(1, 2)), f_mul(e2_conj(q.y), frob_coeff<P>(1, 3))};
    const Affine<Fp2<P>> q2{f_mul(q.x, frob_coeff<P>(2, 2)), f_neg(f_mul(q.y, frob_coeff<P>(2, 3)))};
    const Line<P> l2 = scale_line(add_mixed_step(r, q1), p);
    const Line<P> l1 = scale_line(line_compute(r, q2), p);
    return mul_two_lines(f, l1, l2);
  } else {
    {
      const Line<P> l1 = scale_line(double_step(r), p);
      const Line<P> l2 = scale_line(add_mixed_step(r, q), p);
      f = mul_two_lines(f, l2, l1);
    }
    for (int i = T::LOOP_LEN - 3; i >= 1; i--) {
      f = e12_sqr(f);
      const Line<P> l1 = scale_line(double_step(r), p);
      if (T::loop(i) == 0) {
        f = mul_line(f, l1);
      } else {
        const Line<P> l2 = scale_line(add_mixed_step(r, q), p);
        f = mul_two_lines(f, l2, l1);
      }
    }
    f = e12_sqr(f);
    f = mul_line(f, scale_line(tangent_line(r), p));
    return e12_conj(f);
  }
}

// FinalExponentiation of the product of z[0..k)
template <class P>
GMSM_TOWER Fp12<P> final_exp(const Fp12<P>* z, uint32_t k) {
  Fp12<P> result = z[0];
  for (uint32_t i = 1; i < k; i++) result = e12_mul(result, z[i]);
  // easy part: result^((p^6 - 1)(p^2 + 1))
  Fp12<P> t0 = e12_mul(e12_conj(result), e12_inv(result));
  result = e12_mul(e12_frob<2>(t0), t0);
  if (result.is_one()) return result;
  if constexpr (is_dtwist<P>()) {
    t0 = e12_cyclo_sqr(e12_conj(e12_expt(result)));
    Fp12<P> t1 = e12_mul(t0, e12_cyclo_sqr(t0));
    Fp12<P> t2 = e12_conj(e12_expt(t1));
    Fp12<P> t3 = e12_conj(t1);
    t1 = e12_mul(t2, t3);
    t3 = e12_cyclo_sqr(t2);
    const Fp12<P> t4 = e12_mul(t1, e12_expt(t3));
    t3 = e12_mul(t0, t4);
    t0 = e12_mul(result, e12_mul(t2, t4));
    t0 = e12_mul(e12_frob<1>(t3), t0);
    t0 = e12_mul(e12_frob<2>(t4), t0);
    t2 = e12_frob<3>(e12_mul(e12_conj(result), t3));
    return e12_mul(t2, t0);
  } else {
    t0 = e12_cyclo_sqr(result);
    Fp12<P> t1 = e12_mul(e12_expt_half(t0), e12_conj(result));
    Fp12<P> t2 = e12_expt(t1);
    t1 = e12_mul(e12_conj(t1), t2);
    t2 = e12_expt(t1);
    t1 = e12_mul(e12_frob<1>(t1), t2);
    result = e12_mul(result, t0);
    t0 = e12_expt(t1);
    t2 = e12_expt(t0);
    t0 = e12_frob<2>(t1);
    t1 = e12_mul(e12_mul(e12_conj(t1), t2), t0);
    return e12_mul(result, t1);
  }
}

constexpr unsigned PAIRING_THREADS = 64;
constexpr size_t PAIRING_CHUNK = (size_t)1 << 16;   // pairs per Miller-loop launch

// out[i] = MillerLoop(P[i], Q[i]) for one pair per thread; 1 when either point is infinity
template <class P>
__global__ void __launch_bounds__(PAIRING_THREADS) k_miller_loop(const Affine<Fp<P>>* __restrict__ pts, const Affine<Fp2<P>>* __restrict__ qs,
                                                                 uint32_t n, Fp12<P>* __restrict__ out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const Affine<Fp<P>> p = pts[i];
  const Affine<Fp2<P>> q = qs[i];
  out[i] = (p.is_inf() || q.is_inf()) ? Fp12<P>::one() : miller_loop_one(p, q);
}
// out[i] = in[2i] in[2i + 1] (in[2i] alone for the last of an odd n), i < ceil(n / 2)
template <class P>
__global__ void __launch_bounds__(PAIRING_THREADS) k_gt_reduce(const Fp12<P>* __restrict__ in, uint32_t n, Fp12<P>* __restrict__ out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (2 * i >= n) return;
  out[i] = (2 * i + 1 < n) ? e12_mul(in[2 * i], in[2 * i + 1]) : in[2 * i];
}
// *acc = x (first chunk) or *acc * x
template <class P>
__global__ void k_gt_accumulate(Fp12<P>* acc, const Fp12<P>* x, int first) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  *acc = first ? *x : e12_mul(*acc, *x);
}
template <class P>
__global__ void k_final_exp(const Fp12<P>* z, uint32_t k, Fp12<P>* out) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  *out = final_exp(z, k);
}

// GT elements of workspace for n pairs in chunks of `chunk`: the chunk's Miller values, the first reduction level, the accumulator
static inline size_t pairing_work_elems(size_t n, size_t chunk) {
  const size_t c = n < chunk ? n : chunk;
  return c + (c + 1) / 2 + 1;
}
// The launch order of the multi-pair Miller loop over n >= 1 pairs, the product left in work[acc]: miller(off, m, dst) runs pairs
// [off, off + m) into dst, reduce(src, m, dst) one tree level, accumulate(src, first) multiplies src into the accumulator.
// Indices are GT elements of the workspace (pairing_work_elems).
template <class Miller, class Reduce, class Accum>
static inline void pairing_schedule(size_t n, size_t chunk, Miller miller, Reduce reduce, Accum accumulate) {
  const size_t c = n < chunk ? n : chunk;
  const size_t a = 0, b = c;   // ping-pong buffers: c and ceil(c / 2) elements
  for (size_t off = 0; off < n; off += c) {
    size_t m = n - off < c ? n - off : c;
    miller(off, m, a);
    size_t src = a, dst = b;
    while (m > 1) {
      reduce(src, m, dst);
      m = (m + 1) / 2;
      const size_t t = src;
      src = dst;
      dst = t;
    }
    accumulate(src, off == 0);
  }
}
static inline size_t pairing_acc_index(size_t n, size_t chunk) { return pairing_work_elems(n, chunk) - 1; }

}  // namespace gmsm
