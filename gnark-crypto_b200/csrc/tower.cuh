// Pairing towers of bn254 and bls12-381: Fp6 = Fp2[v]/(v^3 - xi), Fp12 = Fp6[w]/(w^2 - v), xi = 9 + u (bn254) or 1 + u (bls12-381).
//
// Replaces (reference): ecc/<curve>/internal/fptower/e6.go (Mul, Square, Inverse, MulBy01, MulBy1, MulBy12, MulByE2,
// MulByNonResidue), e12.go (Mul, Square, Inverse, Conjugate, CyclotomicSquare, CyclotomicSquareCompressed, DecompressKarabina),
// frobenius.go (Frobenius, FrobeniusSquare, FrobeniusCube) and e12_pairing.go (Expt, ExptHalf, MulBy034 / Mul034By034 /
// MulBy01234 for bn254, MulBy014 / Mul014By014 / MulBy01245 for bls12-381).  Every product is a field value, so any correct
// formula gives the reference's limbs; the Frobenius maps use gamma[k][e] = xi^(e (p^k - 1) / 6) on the coefficient of w^e
// (field_consts.cuh, computed by tools/gen_consts.py).  Memory order: E12{C0, C1}, E6{B0, B1, B2}, E2{A0, A1}.  Builds for the host
// too (the CPU kernel emulation runs it).
#pragma once
#include <type_traits>

#include "fp2.cuh"

// The Fp6 / Fp12 operations are real calls, not inlined: the Miller loop and the final exponentiation inline to far more code than
// the compilers handle in reasonable time, and a call keeps one copy of each operation in the instruction cache.
#if defined(__CUDACC__)
#define GMSM_TOWER __host__ __device__ __noinline__
#else
#define GMSM_TOWER __attribute__((noinline))
#endif

namespace gmsm {

template <class P> struct TowerOf;
template <> struct TowerOf<bn254_fp> { using T = bn254_tower; };
template <> struct TowerOf<bls12381_fp> { using T = bls12381_tower; };

template <class P>
struct Fp6 {
  Fp2<P> b0, b1, b2;
};
template <class P>
struct Fp12 {
  Fp6<P> c0, c1;
  GMSM_HD static Fp12 one() { return Fp12{{Fp2<P>::one(), Fp2<P>::zero(), Fp2<P>::zero()}, {Fp2<P>::zero(), Fp2<P>::zero(), Fp2<P>::zero()}}; }
  GMSM_HD bool is_one() const {
    return c0.b0 == Fp2<P>::one() && c0.b1.is_zero() && c0.b2.is_zero() && c1.b0.is_zero() && c1.b1.is_zero() && c1.b2.is_zero();
  }
};

// ---- constants and small multiples ----
template <class P, class F>
GMSM_HD Fp<P> fp_table(F f, int base) {
  Fp<P> r;
#pragma unroll
  for (int i = 0; i < P::N; i++) r.l[i] = f(base + i);
  return r;
}
template <class P>
GMSM_HD Fp2<P> btwist() {
  using T = typename TowerOf<P>::T;
  return Fp2<P>{fp_table<P>(T::btwist, 0), fp_table<P>(T::btwist, P::N)};
}
template <class P>
GMSM_HD Fp2<P> frob_coeff(int k, int e) {   // gamma[k][e], 1 <= k <= 3, 1 <= e <= 5
  using T = typename TowerOf<P>::T;
  const int base = (((k - 1) * 5 + e - 1) * 2) * P::N;
  return Fp2<P>{fp_table<P>(T::frob, base), fp_table<P>(T::frob, base + P::N)};
}
template <int K, class P>
GMSM_HD Fp<P> fp_mul_int(const Fp<P>& a) {
  if constexpr (K == 1) return a;
  else if constexpr (K % 2 == 0) return fp_dbl(fp_mul_int<K / 2>(a));
  else return fp_add(fp_mul_int<K - 1>(a), a);
}
template <class P>
GMSM_HD Fp2<P> e2_halve(const Fp2<P>& a) {
  using T = typename TowerOf<P>::T;
  const Fp<P> h = fp_table<P>(T::half, 0);
  return Fp2<P>{fp_mul(a.a0, h), fp_mul(a.a1, h)};
}
template <class P>
GMSM_HD Fp2<P> e2_by_fp(const Fp2<P>& a, const Fp<P>& s) { return Fp2<P>{fp_mul(a.a0, s), fp_mul(a.a1, s)}; }
template <class P>
GMSM_HD Fp2<P> e2_conj(const Fp2<P>& a) { return Fp2<P>{a.a0, fp_neg(a.a1)}; }
// times xi = XI0 + u (u^2 = -1)
template <class P>
GMSM_HD Fp2<P> e2_nr(const Fp2<P>& a) {
  using T = typename TowerOf<P>::T;
  static_assert(T::XI1 == 1 && P::FP2_NONRES == -1, "xi = XI0 + u over u^2 = -1");
  return Fp2<P>{fp_sub(fp_mul_int<T::XI0>(a.a0), a.a1), fp_add(fp_mul_int<T::XI0>(a.a1), a.a0)};
}

// ---- Fp6 ----
template <class P> GMSM_HD Fp6<P> e6_add(const Fp6<P>& a, const Fp6<P>& b) { return Fp6<P>{f_add(a.b0, b.b0), f_add(a.b1, b.b1), f_add(a.b2, b.b2)}; }
template <class P> GMSM_HD Fp6<P> e6_sub(const Fp6<P>& a, const Fp6<P>& b) { return Fp6<P>{f_sub(a.b0, b.b0), f_sub(a.b1, b.b1), f_sub(a.b2, b.b2)}; }
template <class P> GMSM_HD Fp6<P> e6_neg(const Fp6<P>& a) { return Fp6<P>{f_neg(a.b0), f_neg(a.b1), f_neg(a.b2)}; }
template <class P> GMSM_HD Fp6<P> e6_dbl(const Fp6<P>& a) { return Fp6<P>{f_dbl(a.b0), f_dbl(a.b1), f_dbl(a.b2)}; }
template <class P> GMSM_HD Fp6<P> e6_nr(const Fp6<P>& a) { return Fp6<P>{e2_nr(a.b2), a.b0, a.b1}; }   // times v
template <class P> GMSM_HD Fp6<P> e6_by_e2(const Fp6<P>& a, const Fp2<P>& c) { return Fp6<P>{f_mul(a.b0, c), f_mul(a.b1, c), f_mul(a.b2, c)}; }

// Karatsuba, 6 Fp2 products
template <class P>
GMSM_TOWER Fp6<P> e6_mul(const Fp6<P>& a, const Fp6<P>& b) {
  const Fp2<P> v0 = f_mul(a.b0, b.b0), v1 = f_mul(a.b1, b.b1), v2 = f_mul(a.b2, b.b2);
  Fp6<P> z;
  z.b0 = f_add(v0, e2_nr(f_sub(f_sub(f_mul(f_add(a.b1, a.b2), f_add(b.b1, b.b2)), v1), v2)));
  z.b1 = f_add(f_sub(f_sub(f_mul(f_add(a.b0, a.b1), f_add(b.b0, b.b1)), v0), v1), e2_nr(v2));
  z.b2 = f_add(f_sub(f_sub(f_mul(f_add(a.b0, a.b2), f_add(b.b0, b.b2)), v0), v2), v1);
  return z;
}
// a * (c0 + c1 v)
template <class P>
GMSM_TOWER Fp6<P> e6_mul_by_01(const Fp6<P>& a, const Fp2<P>& c0, const Fp2<P>& c1) {
  const Fp2<P> t0 = f_mul(a.b0, c0), t1 = f_mul(a.b1, c1);
  Fp6<P> z;
  z.b0 = f_add(t0, e2_nr(f_mul(a.b2, c1)));
  z.b1 = f_sub(f_sub(f_mul(f_add(a.b0, a.b1), f_add(c0, c1)), t0), t1);
  z.b2 = f_add(f_mul(a.b2, c0), t1);
  return z;
}
// a * (c1 v)
template <class P>
GMSM_HD Fp6<P> e6_mul_by_1(const Fp6<P>& a, const Fp2<P>& c1) {
  return Fp6<P>{e2_nr(f_mul(a.b2, c1)), f_mul(a.b0, c1), f_mul(a.b1, c1)};
}
// a * (c1 v + c2 v^2)
template <class P>
GMSM_TOWER Fp6<P> e6_mul_by_12(const Fp6<P>& a, const Fp2<P>& c1, const Fp2<P>& c2) {
  const Fp2<P> t1 = f_mul(a.b1, c1), t2 = f_mul(a.b2, c2);
  Fp6<P> z;
  z.b0 = e2_nr(f_sub(f_sub(f_mul(f_add(a.b1, a.b2), f_add(c1, c2)), t1), t2));
  z.b1 = f_add(f_mul(a.b0, c1), e2_nr(t2));
  z.b2 = f_add(f_mul(a.b0, c2), t1);
  return z;
}
template <class P>
GMSM_TOWER Fp6<P> e6_inv(const Fp6<P>& a) {
  const Fp2<P> t0 = f_sub(f_sqr(a.b0), e2_nr(f_mul(a.b1, a.b2)));
  const Fp2<P> t1 = f_sub(e2_nr(f_sqr(a.b2)), f_mul(a.b0, a.b1));
  const Fp2<P> t2 = f_sub(f_sqr(a.b1), f_mul(a.b0, a.b2));
  const Fp2<P> d = f_add(f_mul(a.b0, t0), e2_nr(f_add(f_mul(a.b2, t1), f_mul(a.b1, t2))));
  const Fp2<P> di = f_inv(d);
  return Fp6<P>{f_mul(t0, di), f_mul(t1, di), f_mul(t2, di)};
}

// ---- Fp12 ----
template <class P>
GMSM_TOWER Fp12<P> e12_mul(const Fp12<P>& a, const Fp12<P>& b) {
  const Fp6<P> t0 = e6_mul(a.c0, b.c0), t1 = e6_mul(a.c1, b.c1);
  Fp12<P> z;
  z.c1 = e6_sub(e6_sub(e6_mul(e6_add(a.c0, a.c1), e6_add(b.c0, b.c1)), t0), t1);
  z.c0 = e6_add(t0, e6_nr(t1));
  return z;
}
// complex squaring: 2 Fp6 products
template <class P>
GMSM_TOWER Fp12<P> e12_sqr(const Fp12<P>& a) {
  const Fp6<P> t = e6_mul(a.c0, a.c1);
  Fp12<P> z;
  z.c0 = e6_sub(e6_sub(e6_mul(e6_add(a.c0, a.c1), e6_add(a.c0, e6_nr(a.c1))), t), e6_nr(t));
  z.c1 = e6_dbl(t);
  return z;
}
template <class P>
GMSM_HD Fp12<P> e12_conj(const Fp12<P>& a) { return Fp12<P>{a.c0, e6_neg(a.c1)}; }
template <class P>
GMSM_TOWER Fp12<P> e12_inv(const Fp12<P>& a) {   // the inverse of zero is zero, as in the reference
  const Fp6<P> t = e6_inv(e6_sub(e6_mul(a.c0, a.c0), e6_nr(e6_mul(a.c1, a.c1))));
  return Fp12<P>{e6_mul(a.c0, t), e6_neg(e6_mul(a.c1, t))};
}
// a^(p^K): the coefficient of w^e (C0.B0, C0.B1, C0.B2, C1.B0, C1.B1, C1.B2: e = 0, 2, 4, 1, 3, 5), conjugated for odd K, times
// gamma[K][e].  Frobenius, FrobeniusSquare and FrobeniusCube are K = 1, 2, 3.
template <int K, class P>
GMSM_TOWER Fp12<P> e12_frob(const Fp12<P>& a) {
  auto c = [](const Fp2<P>& x) { return (K & 1) ? e2_conj(x) : x; };
  Fp12<P> z;
  z.c0.b0 = c(a.c0.b0);
  z.c0.b1 = f_mul(c(a.c0.b1), frob_coeff<P>(K, 2));
  z.c0.b2 = f_mul(c(a.c0.b2), frob_coeff<P>(K, 4));
  z.c1.b0 = f_mul(c(a.c1.b0), frob_coeff<P>(K, 1));
  z.c1.b1 = f_mul(c(a.c1.b1), frob_coeff<P>(K, 3));
  z.c1.b2 = f_mul(c(a.c1.b2), frob_coeff<P>(K, 5));
  return z;
}

// Granger-Scott squaring in the cyclotomic subgroup (e12.go CyclotomicSquare)
template <class P>
GMSM_TOWER Fp12<P> e12_cyclo_sqr(const Fp12<P>& x) {
  Fp2<P> t0 = f_sqr(x.c1.b1), t1 = f_sqr(x.c0.b0);
  const Fp2<P> t6 = f_sub(f_sub(f_sqr(f_add(x.c1.b1, x.c0.b0)), t0), t1);
  Fp2<P> t2 = f_sqr(x.c0.b2), t3 = f_sqr(x.c1.b0);
  const Fp2<P> t7 = f_sub(f_sub(f_sqr(f_add(x.c0.b2, x.c1.b0)), t2), t3);
  Fp2<P> t4 = f_sqr(x.c1.b2), t5 = f_sqr(x.c0.b1);
  const Fp2<P> t8 = e2_nr(f_sub(f_sub(f_sqr(f_add(x.c1.b2, x.c0.b1)), t4), t5));
  t0 = f_add(e2_nr(t0), t1);
  t2 = f_add(e2_nr(t2), t3);
  t4 = f_add(e2_nr(t4), t5);
  Fp12<P> z;
  z.c0.b0 = f_add(f_dbl(f_sub(t0, x.c0.b0)), t0);
  z.c0.b1 = f_add(f_dbl(f_sub(t2, x.c0.b1)), t2);
  z.c0.b2 = f_add(f_dbl(f_sub(t4, x.c0.b2)), t4);
  z.c1.b0 = f_add(f_dbl(f_add(t8, x.c1.b0)), t8);
  z.c1.b1 = f_add(f_dbl(f_add(t6, x.c1.b1)), t6);
  z.c1.b2 = f_add(f_dbl(f_add(t7, x.c1.b2)), t7);
  return z;
}
// Karabina's compressed squaring (e12.go CyclotomicSquareCompressed): updates C0.B1, C0.B2, C1.B0, C1.B2 and keeps the others
template <class P>
GMSM_TOWER Fp12<P> e12_cyclo_sqr_compressed(const Fp12<P>& x) {
  const Fp2<P> t0 = f_sqr(x.c0.b1), t1 = f_sqr(x.c1.b2);
  const Fp2<P> t5 = f_sub(f_sqr(f_add(x.c0.b1, x.c1.b2)), f_add(t0, t1));
  const Fp2<P> t3 = f_sqr(f_add(x.c1.b0, x.c0.b2));
  const Fp2<P> t2 = f_sqr(x.c1.b0);
  Fp12<P> z = x;
  const Fp2<P> t6 = e2_nr(t5);
  z.c1.b0 = f_add(f_dbl(f_add(t6, x.c1.b0)), t6);
  const Fp2<P> s5 = f_add(t0, e2_nr(t1));
  z.c0.b2 = f_add(f_dbl(f_sub(s5, x.c0.b2)), s5);
  const Fp2<P> u1 = f_sqr(x.c0.b2);
  const Fp2<P> s6 = f_add(t2, e2_nr(u1));
  z.c0.b1 = f_add(f_dbl(f_sub(s6, x.c0.b1)), s6);
  const Fp2<P> s7 = f_sub(t3, f_add(t2, u1));
  z.c1.b2 = f_add(s7, f_dbl(f_add(s7, x.c1.b2)));
  return z;
}
// e12.go DecompressKarabina (BatchDecompressKarabina gives the same values)
template <class P>
GMSM_TOWER Fp12<P> e12_decompress_karabina(const Fp12<P>& x) {
  Fp2<P> t0, t1;
  if (x.c1.b2.is_zero()) {
    t0 = f_dbl(f_mul(x.c0.b1, x.c1.b2));
    t1 = x.c0.b2;
    if (t1.is_zero()) return Fp12<P>::one();
  } else {
    t0 = f_sqr(x.c0.b1);
    t1 = f_add(f_dbl(f_sub(t0, x.c0.b2)), t0);
    t0 = f_add(e2_nr(f_sqr(x.c1.b2)), t1);
    t1 = f_dbl(f_dbl(x.c1.b0));
  }
  Fp12<P> z = x;
  z.c1.b1 = f_mul(t0, f_inv(t1));
  t1 = f_mul(x.c0.b2, x.c0.b1);
  Fp2<P> t2 = f_sub(f_dbl(f_sub(f_sqr(z.c1.b1), t1)), t1);
  t2 = f_add(t2, f_mul(x.c1.b0, x.c1.b2));
  z.c0.b0 = f_add(e2_nr(t2), Fp2<P>::one());
  return z;
}
template <class P>
GMSM_TOWER Fp12<P> e12_nsqr(Fp12<P> x, int n) {
  for (int i = 0; i < n; i++) x = e12_cyclo_sqr(x);
  return x;
}

// x^x0 (bn254, e12_pairing.go Expt); x^(x0 / 2) (bls12-381 ExptHalf) and its square
template <class P>
GMSM_TOWER Fp12<P> e12_expt_half(const Fp12<P>& x) {
  Fp12<P> r = x;
  for (int i = 0; i < 15; i++) r = e12_cyclo_sqr_compressed(r);
  const Fp12<P> t0 = r;
  for (int i = 0; i < 32; i++) r = e12_cyclo_sqr_compressed(r);
  Fp12<P> b1 = e12_decompress_karabina(r);
  Fp12<P> res = e12_mul(e12_decompress_karabina(t0), b1);
  b1 = e12_nsqr(b1, 9);
  res = e12_mul(res, b1);
  b1 = e12_nsqr(b1, 3);
  res = e12_mul(res, b1);
  b1 = e12_nsqr(b1, 2);
  res = e12_mul(res, b1);
  b1 = e12_cyclo_sqr(b1);
  res = e12_mul(res, b1);
  return e12_conj(res);
}
template <class P>
GMSM_TOWER Fp12<P> e12_expt(const Fp12<P>& x) {
  if constexpr (std::is_same<P, bls12381_fp>::value) {
    return e12_cyclo_sqr(e12_expt_half(x));
  } else {
    Fp12<P> t3 = e12_cyclo_sqr(x);
    Fp12<P> t5 = e12_cyclo_sqr(t3);
    const Fp12<P> result = e12_cyclo_sqr(t5);
    Fp12<P> t0 = e12_cyclo_sqr(result);
    Fp12<P> t2 = e12_mul(x, t0);
    t0 = e12_mul(t3, t2);
    Fp12<P> t1 = e12_mul(x, t0);
    Fp12<P> t4 = e12_mul(result, t2);
    Fp12<P> t6 = e12_cyclo_sqr(t2);
    t1 = e12_mul(t0, t1);
    t0 = e12_mul(t3, t1);
    t6 = e12_nsqr(t6, 6);
    t5 = e12_mul(t5, t6);
    t5 = e12_mul(t4, t5);
    t5 = e12_nsqr(t5, 7);
    t4 = e12_mul(t4, t5);
    t4 = e12_nsqr(t4, 8);
    t4 = e12_mul(t0, t4);
    t3 = e12_mul(t3, t4);
    t3 = e12_nsqr(t3, 6);
    t2 = e12_mul(t2, t3);
    t2 = e12_nsqr(t2, 8);
    t2 = e12_mul(t0, t2);
    t2 = e12_nsqr(t2, 6);
    t2 = e12_mul(t0, t2);
    t2 = e12_nsqr(t2, 10);
    t1 = e12_mul(t1, t2);
    t1 = e12_nsqr(t1, 6);
    t0 = e12_mul(t0, t1);
    return e12_mul(result, t0);
  }
}

// ---- sparse products of the Miller loops ----
// bn254 (D-twist): a line is c0 + (c3 + c4 v) w, at positions 0, 3, 4
template <class P>
GMSM_TOWER Fp12<P> e12_mul_by_034(const Fp12<P>& f, const Fp2<P>& c0, const Fp2<P>& c3, const Fp2<P>& c4) {
  const Fp6<P> a = e6_by_e2(f.c0, c0);
  const Fp6<P> b = e6_mul_by_01(f.c1, c3, c4);
  const Fp6<P> d = e6_mul_by_01(e6_add(f.c0, f.c1), f_add(c0, c3), c4);
  return Fp12<P>{e6_add(e6_nr(b), a), e6_sub(d, e6_add(a, b))};
}
// the product of two such lines: positions 0, 1, 2 (C0) and 3, 4 (C1.B0, C1.B1)
template <class P>
GMSM_TOWER void e2_mul_034_by_034(const Fp2<P>& d0, const Fp2<P>& d3, const Fp2<P>& d4, const Fp2<P>& c0, const Fp2<P>& c3, const Fp2<P>& c4,
                               Fp2<P> (&z)[5]) {
  const Fp2<P> x0 = f_mul(c0, d0), x3 = f_mul(c3, d3), x4 = f_mul(c4, d4);
  z[4] = f_sub(f_sub(f_mul(f_add(d0, d4), f_add(c0, c4)), x0), x4);
  z[3] = f_sub(f_sub(f_mul(f_add(d0, d3), f_add(c0, c3)), x0), x3);
  z[2] = f_sub(f_sub(f_mul(f_add(d3, d4), f_add(c3, c4)), x3), x4);
  z[1] = x3;
  z[0] = f_add(e2_nr(x4), x0);
}
template <class P>
GMSM_TOWER Fp12<P> e12_mul_by_01234(const Fp12<P>& f, const Fp2<P> (&x)[5]) {
  const Fp6<P> c0{x[0], x[1], x[2]};
  const Fp6<P> a = e6_mul(e6_add(f.c0, f.c1), Fp6<P>{f_add(x[0], x[3]), f_add(x[1], x[4]), x[2]});
  const Fp6<P> b = e6_mul(f.c0, c0);
  const Fp6<P> c = e6_mul_by_01(f.c1, x[3], x[4]);
  return Fp12<P>{e6_add(e6_nr(c), b), e6_sub(e6_sub(a, b), c)};
}
// bls12-381 (M-twist): a line is (c0 + c1 v) + (c4 v) w, at positions 0, 1, 4
template <class P>
GMSM_TOWER Fp12<P> e12_mul_by_014(const Fp12<P>& f, const Fp2<P>& c0, const Fp2<P>& c1, const Fp2<P>& c4) {
  const Fp6<P> a = e6_mul_by_01(f.c0, c0, c1);
  const Fp6<P> b = e6_mul_by_1(f.c1, c4);
  const Fp6<P> d = e6_mul_by_01(e6_add(f.c0, f.c1), c0, f_add(c1, c4));
  return Fp12<P>{e6_add(e6_nr(b), a), e6_sub(d, e6_add(a, b))};
}
// the product of two such lines: positions 0, 1, 2 (C0) and 4, 5 (C1.B1, C1.B2)
template <class P>
GMSM_TOWER void e2_mul_014_by_014(const Fp2<P>& d0, const Fp2<P>& d1, const Fp2<P>& d4, const Fp2<P>& c0, const Fp2<P>& c1, const Fp2<P>& c4,
                               Fp2<P> (&z)[5]) {
  const Fp2<P> x0 = f_mul(c0, d0), x1 = f_mul(c1, d1), x4 = f_mul(c4, d4);
  z[3] = f_sub(f_sub(f_mul(f_add(d0, d4), f_add(c0, c4)), x0), x4);
  z[1] = f_sub(f_sub(f_mul(f_add(d0, d1), f_add(c0, c1)), x0), x1);
  z[4] = f_sub(f_sub(f_mul(f_add(d1, d4), f_add(c1, c4)), x1), x4);
  z[2] = x1;
  z[0] = f_add(e2_nr(x4), x0);
}
template <class P>
GMSM_TOWER Fp12<P> e12_mul_by_01245(const Fp12<P>& f, const Fp2<P> (&x)[5]) {
  const Fp6<P> c0{x[0], x[1], x[2]};
  const Fp6<P> a = e6_mul(e6_add(f.c0, f.c1), Fp6<P>{x[0], f_add(x[1], x[3]), f_add(x[2], x[4])});
  const Fp6<P> b = e6_mul(f.c0, c0);
  const Fp6<P> c = e6_mul_by_12(f.c1, x[3], x[4]);
  return Fp12<P>{e6_add(e6_nr(c), b), e6_sub(e6_sub(a, b), c)};
}

}  // namespace gmsm
