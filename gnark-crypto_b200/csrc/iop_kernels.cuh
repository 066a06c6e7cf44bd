// Device side of the iop package (ecc/bn254/fr/iop; the iop packages of the other pairing curves are the same generated code):
// the accumulating ratios of BuildRatioShuffledVectors and BuildRatioCopyConstraint, the barycentric evaluation of a Lagrange-form
// polynomial, the interpreter behind Evaluate and the division by X^n - 1 of DivideByXMinusOne.  In a header of their own, like
// perm_kernels.cuh, so that the CPU kernel emulation of tests/emu/ compiles and runs them too (tests/test_emu_iop_cpu.py); fft.cu
// includes this file and holds the entry points.  The batch inversion (perm_tree_invert) and the exclusive prefix product
// (perm_prefix_schedule over poly_levels) are those of perm_kernels.cuh.
//
// Accumulating ratios (ratios.go:45-246).  The reference forms the prefix products of the numerators and of the denominators
// separately and multiplies by fr.BatchInvert of the second (zero -> zero).  Here r[i] = b_i d_i^-1 (zero -> zero) is formed per
// position with the tile inversion, then Z[0] = 1, Z[k] = prod_{i<k} r[i] by the exclusive prefix product.  A zero d_m makes the
// reference's t[k] zero for every k > m, so it zeroes exactly Z[k] for k > m; the ratio form zeroes exactly the same entries (r[m] = 0).
//   shuffled vectors:  b_i = prod_c (beta - P_c[i]),  d_i = prod_c (beta - Q_c[i])                       for i < n - 1
//   copy constraint:   b_i = prod_c (P_c[i] + beta g^c w^i + gamma),  d_i = prod_c (P_c[i] + beta ID[sigma(cn + i)] + gamma)
// with ID[s] = g^(s / n) w^(s mod n) formed on the fly from the domain's twiddles (w^(j + n/2) = -w^j, as in k_perm_numerator) and
// the host's beta g^c: the k n support table of getSupportIdentityPermutation is never materialised.  Columns are read at storage
// index i, or rev(i) for a BitReverse column; shift and size are ignored, as in the reference.
//
// Lagrange evaluation (evalLagrange, polynomial.go:204-241): p(x) = (x^n - 1) / n sum_i w^i (x - w^i)^-1 c[idx(i)].  One block per
// tile inverts its (x - w^i) with the tile inversion (zero -> zero) and sums its terms; k_iop_sum adds the tile sums and applies
// (x^n - 1) / n.  For x on the domain the factor is zero, so the result is zero, as in the reference.
//
// Field arithmetic is exact and every fp_* result is fully reduced, so any grouping gives the reference's limbs.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "field.cuh"
#include "perm_kernels.cuh"
#include "vec_io.cuh"

using namespace gmsm;

namespace {

constexpr int IOP_MAX_COLUMNS = 32;     // polynomials per list of a ratio builder
constexpr int IOP_MAX_PROGRAM = 256;    // instructions of an Evaluate program
constexpr int IOP_MAX_REGISTERS = 16;   // live values of an Evaluate program
constexpr int IOP_MAX_INPUTS = 32;      // input polynomials of Evaluate
constexpr int IOP_MAX_CONSTS = 32;      // distinct constants of an Evaluate program
constexpr int IOP_MAX_RHO = 64;         // len / size of DivideByXMinusOne's input

// storage index of element s of a vector of n entries: s, or Reverse64(s) >> (64 - TrailingZeros(n)) for a BitReverse layout
GMSM_HD uint64_t iop_index(uint64_t s, int tz, bool bitrev) {
#ifdef __CUDA_ARCH__
  const uint64_t b = __brevll(s);
#else
  uint64_t b = 0;
  for (int k = 0; k < 64; k++) b |= ((s >> k) & 1ull) << (63 - k);
#endif
  return bitrev ? (tz ? b >> (64 - tz) : 0ull) : s;
}

// w^i from the domain's twiddles tw[j] = w^j, j < n / 2
template <class P>
GMSM_D Fp<P> iop_root(const Fp<P>* tw, uint64_t i, uint64_t half) {
  return i == 0 ? Fp<P>::one() : i < half ? load_vec(tw + i) : fp_neg(load_vec(tw + (i - half)));
}

template <class P>
struct IopColumns {
  const Fp<P>* p[IOP_MAX_COLUMNS];
  uint32_t bitrev;   // bit c: column c has the BitReverse layout
  int k;
};

// r[i] = prod_c (beta - num_c[i]) (prod_c (beta - den_c[i]))^-1 (0 -> 0) for i < n - 1, r[n - 1] = 1 (never read by the exclusive
// prefix).  One block per tile of 2^log_t, blockDim.x >= 2^log_t / 32, dynamic shared memory perm_inv_smem_bytes.  r must not
// overlap a column.
template <class P>
__global__ void k_iop_ratio_shuffled(IopColumns<P> num, IopColumns<P> den, uint64_t n, int logn, Fp<P> beta, int log_t, Fp<P>* r) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Fp<P>* s = reinterpret_cast<Fp<P>*>(smem_raw);
  const uint32_t T = 1u << log_t, B = blockDim.x, tid = threadIdx.x;
  const uint64_t base = (uint64_t)blockIdx.x * T;
  uint32_t zero = 0;
  for (uint32_t j = tid, q = 0; j < T; j += B, q++) {
    const uint64_t i = base + j;
    Fp<P> d = Fp<P>::one();
    if (i + 1 < n)
      for (int c = 0; c < den.k; c++) d = fp_mul(d, fp_sub(beta, load_vec(den.p[c] + iop_index(i, logn, (den.bitrev >> c) & 1u))));
    if (d.is_zero()) zero |= 1u << q;
    store_vec(s + T + j, d.is_zero() ? Fp<P>::one() : d);
  }
  __syncthreads();
  perm_tree_invert(s, T);
  for (uint32_t j = tid, q = 0; j < T; j += B, q++) {
    const uint64_t i = base + j;
    if (i >= n) continue;
    Fp<P> v = Fp<P>::one();
    if (i + 1 < n) {
      if ((zero >> q) & 1u) {
        v = Fp<P>::zero();
      } else {
        Fp<P> b = Fp<P>::one();
        for (int c = 0; c < num.k; c++) b = fp_mul(b, fp_sub(beta, load_vec(num.p[c] + iop_index(i, logn, (num.bitrev >> c) & 1u))));
        v = fp_mul(b, load_vec(s + T + j));
      }
    }
    store_vec(r + i, v);
  }
}

template <class P>
struct IopCopyConsts {
  const Fp<P>* p[IOP_MAX_COLUMNS];
  Fp<P> bg[IOP_MAX_COLUMNS];   // beta g^c, g = FrMultiplicativeGen
  Fp<P> gamma;
  uint32_t bitrev;
  int k;
};

// sigma[j] outside [0, limit) for some j < m -> *bad = 1 (every writer stores the same value)
__global__ void k_iop_check_sigma(const int64_t* sigma, uint64_t m, int64_t limit, uint32_t* bad) {
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < m; j += (uint64_t)gridDim.x * blockDim.x) {
    const int64_t v = sigma[j];
    if (v < 0 || v >= limit) *bad = 1;
  }
}

// r[i] of BuildRatioCopyConstraint for i < n - 1 (header comment), r[n - 1] = 1; tw: the domain's twiddles.  Launch shape as
// k_iop_ratio_shuffled; every sigma entry must lie in [0, k n) (k_iop_check_sigma).  r must not overlap a column.
template <class P>
__global__ void k_iop_ratio_copy(IopCopyConsts<P> k, const int64_t* sigma, uint64_t n, int logn, const Fp<P>* tw, int log_t, Fp<P>* r) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Fp<P>* s = reinterpret_cast<Fp<P>*>(smem_raw);
  const uint32_t T = 1u << log_t, B = blockDim.x, tid = threadIdx.x;
  const uint64_t base = (uint64_t)blockIdx.x * T, half = n >> 1;
  uint32_t zero = 0;
  for (uint32_t j = tid, q = 0; j < T; j += B, q++) {
    const uint64_t i = base + j;
    Fp<P> d = Fp<P>::one();
    if (i + 1 < n)
      for (int c = 0; c < k.k; c++) {
        const uint64_t sg = (uint64_t)sigma[(uint64_t)c * n + i];
        const Fp<P> id = fp_mul(k.bg[sg >> logn], iop_root(tw, sg & (n - 1), half));   // beta ID[sigma]
        const Fp<P> pv = load_vec(k.p[c] + iop_index(i, logn, (k.bitrev >> c) & 1u));
        d = fp_mul(d, fp_add(fp_add(pv, id), k.gamma));
      }
    if (d.is_zero()) zero |= 1u << q;
    store_vec(s + T + j, d.is_zero() ? Fp<P>::one() : d);
  }
  __syncthreads();
  perm_tree_invert(s, T);
  for (uint32_t j = tid, q = 0; j < T; j += B, q++) {
    const uint64_t i = base + j;
    if (i >= n) continue;
    Fp<P> v = Fp<P>::one();
    if (i + 1 < n) {
      if ((zero >> q) & 1u) {
        v = Fp<P>::zero();
      } else {
        const Fp<P> wi = iop_root(tw, i, half);
        Fp<P> b = Fp<P>::one();
        for (int c = 0; c < k.k; c++) {
          const Fp<P> pv = load_vec(k.p[c] + iop_index(i, logn, (k.bitrev >> c) & 1u));
          b = fp_mul(b, fp_add(fp_add(pv, fp_mul(k.bg[c], wi)), k.gamma));
        }
        v = fp_mul(b, load_vec(s + T + j));
      }
    }
    store_vec(r + i, v);
  }
}

// partial[tile] = sum over the tile's i < n of w^i (x - w^i)^-1 c[idx(i)] (a zero x - w^i contributes zero).  Launch shape as
// k_iop_ratio_shuffled (blockDim.x a power of two, at most 2^(log_t + 1)).
template <class P>
__global__ void k_iop_lagrange_terms(const Fp<P>* c, uint64_t n, int logn, int bitrev, Fp<P> x, const Fp<P>* tw, int log_t, Fp<P>* partial) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Fp<P>* s = reinterpret_cast<Fp<P>*>(smem_raw);
  const uint32_t T = 1u << log_t, B = blockDim.x, tid = threadIdx.x;
  const uint64_t base = (uint64_t)blockIdx.x * T, half = n >> 1;
  uint32_t zero = 0;
  for (uint32_t j = tid, q = 0; j < T; j += B, q++) {
    const uint64_t i = base + j;
    const Fp<P> d = i < n ? fp_sub(x, iop_root(tw, i, half)) : Fp<P>::one();
    if (d.is_zero()) zero |= 1u << q;
    store_vec(s + T + j, d.is_zero() ? Fp<P>::one() : d);
  }
  __syncthreads();
  perm_tree_invert(s, T);
  Fp<P> acc = Fp<P>::zero();
  for (uint32_t j = tid, q = 0; j < T; j += B, q++) {
    const uint64_t i = base + j;
    if (i >= n || ((zero >> q) & 1u)) continue;
    const Fp<P> t = fp_mul(iop_root(tw, i, half), load_vec(s + T + j));
    acc = fp_add(acc, fp_mul(t, load_vec(c + iop_index(i, logn, bitrev != 0))));
  }
  __syncthreads();
  store_vec(s + tid, acc);
  __syncthreads();
  for (uint32_t h = B >> 1; h >= 1; h >>= 1) {
    if (tid < h) store_vec(s + tid, fp_add(load_vec(s + tid), load_vec(s + tid + h)));
    __syncthreads();
  }
  if (tid == 0) store_vec(partial + blockIdx.x, load_vec(s));
}

// *out = scale sum_{t<m} partial[t].  One block, blockDim.x a power of two, dynamic shared memory blockDim.x elements.
template <class P>
__global__ void k_iop_sum(const Fp<P>* partial, uint64_t m, Fp<P> scale, Fp<P>* out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Fp<P>* s = reinterpret_cast<Fp<P>*>(smem_raw);
  const uint32_t B = blockDim.x, tid = threadIdx.x;
  Fp<P> acc = Fp<P>::zero();
  for (uint64_t t = tid; t < m; t += B) acc = fp_add(acc, load_vec(partial + t));
  store_vec(s + tid, acc);
  __syncthreads();
  for (uint32_t h = B >> 1; h >= 1; h >>= 1) {
    if (tid < h) store_vec(s + tid, fp_add(load_vec(s + tid), load_vec(s + tid + h)));
    __syncthreads();
  }
  if (tid == 0) store_vec(out, fp_mul(load_vec(s), scale));
}

// ---- the Evaluate interpreter ----
// instruction word: op | dst << 8 | a << 16 | b << 24.  INPUT: reg[dst] = x_a.GetCoeff(i); CONST: reg[dst] = consts[a]; INDEX:
// reg[dst] = i as an fr.Element; ADD / SUB / MUL: reg[dst] = reg[a] op reg[b]; NEG: reg[dst] = -reg[a].
enum : uint32_t { IOP_OP_INPUT = 0, IOP_OP_CONST = 1, IOP_OP_INDEX = 2, IOP_OP_ADD = 3, IOP_OP_SUB = 4, IOP_OP_MUL = 5, IOP_OP_NEG = 6 };

template <class P>
struct IopProgram {
  uint32_t code[IOP_MAX_PROGRAM];
  Fp<P> consts[IOP_MAX_CONSTS];
  int len, out;   // instructions; the register that holds the result
};

struct IopInputs {
  const void* p[IOP_MAX_INPUTS];
  uint64_t off[IOP_MAX_INPUTS];   // (rho shift) mod n of GetCoeff
  uint32_t bitrev;
  int m;
};

// r[idx(i)] = f(i, x_0.GetCoeff(i), ...) for i < n, idx(i) = i or its bit reversal (out_bitrev).  Grid-stride, any launch shape.  The
// register file is indexed by the program, so it lives in local memory.  r must not overlap an input.
template <class P>
__global__ void k_iop_evaluate(IopProgram<P> prog, IopInputs in, uint64_t n, int tz, int out_bitrev, Fp<P>* r) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    Fp<P> reg[IOP_MAX_REGISTERS];
    for (int pc = 0; pc < prog.len; pc++) {
      const uint32_t w = prog.code[pc], op = w & 0xff, dst = (w >> 8) & 0xff, a = (w >> 16) & 0xff, b = w >> 24;
      switch (op) {
        case IOP_OP_INPUT: {
          uint64_t sx = i + in.off[a];
          if (sx >= n) sx -= n;
          reg[dst] = load_vec(reinterpret_cast<const Fp<P>*>(in.p[a]) + iop_index(sx, tz, (in.bitrev >> a) & 1u));
          break;
        }
        case IOP_OP_CONST: reg[dst] = prog.consts[a]; break;
        case IOP_OP_INDEX: {
          Fp<P> v = Fp<P>::zero();
          v.l[0] = (uint32_t)i;
          v.l[1] = (uint32_t)(i >> 32);
          reg[dst] = fp_to_mont(v);
          break;
        }
        case IOP_OP_ADD: reg[dst] = fp_add(reg[a], reg[b]); break;
        case IOP_OP_SUB: reg[dst] = fp_sub(reg[a], reg[b]); break;
        case IOP_OP_MUL: reg[dst] = fp_mul(reg[a], reg[b]); break;
        default: reg[dst] = fp_neg(reg[a]); break;
      }
    }
    store_vec(r + iop_index(i, tz, out_bitrev != 0), reg[prog.out]);
  }
}

template <class P>
struct IopXnInv {
  Fp<P> inv[IOP_MAX_RHO];   // (g^s (w_big^s)^j - 1)^-1, s the small domain's cardinality
  uint32_t rho;             // a power of two
};

// out[rev(i)] = a.GetCoeff(i) inv[i mod rho] for i < n = 2^logn (DivideByXMinusOne, quotient.go:40-47).  Grid-stride, any launch
// shape.  out must not overlap a.
template <class P>
__global__ void k_iop_div_xn_minus_one(const Fp<P>* a, uint64_t n, int logn, uint64_t off, int bitrev, IopXnInv<P> k, Fp<P>* out) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t sx = i + off;
    if (sx >= n) sx -= n;
    store_vec(out + iop_index(i, logn, true), fp_mul(load_vec(a + iop_index(sx, logn, bitrev != 0)), k.inv[i & (k.rho - 1)]));
  }
}

}  // namespace
