// Device side of permutation.Prove's Fr steps (ecc/bn254/fr/permutation/permutation.go; the permutation packages of the other
// pairing curves are the same generated code): batch inversion, the accumulation polynomial Z as an exclusive prefix product, and
// the quotient numerator on the coset.  In a header of their own, like poly_kernels.cuh, so that the CPU kernel emulation of
// tests/emu/ compiles and runs them too (tests/test_emu_perm_cpu.py); fft.cu includes this file and holds the entry points.  The
// launch schedule of the scan below is shared by both.
//
// Batch inversion (fr.BatchInvert, fr/element.go:658-687, zero -> zero).  Inversions are independent, so no global scan is needed:
// a block owns a tile of T = 2^log_t elements and runs Montgomery's trick on it as a product tree in shared memory (leaf j at slot
// T + j, node k = leaves 2k and 2k + 1, root at slot 1): an up-sweep of products, one fp_inv of the root, a down-sweep that hands
// each child (its parent's inverse) x (its sibling's product).  Three products per element and one inversion per tile; a zero
// leaf enters the tree as one and leaves as zero.
//
// Accumulation polynomial (evaluateAccumulationPolynomialBitReversed, permutation.go:52-75): z_lin[k] = prod_{j<k} r[j] with
// r[j] = (eps - t1[j]) (eps - t2[j])^-1 (zero -> zero).  The reference's prefix-then-BatchInvert zeroes every z_lin[k] past the
// first k with eps = t2[k-1]; the ratio form zeroes exactly the same entries.  k_perm_ratio writes r (tile inversion as above);
// the exclusive prefix product has the multi-level shape of poly_div_schedule over poly_levels: tile products level by level
// (k_perm_prod_heads) until a level fits in one tile, then a top-down write pass (k_perm_prod_write) whose carry-in for tile t is
// entry t of the level above, already rewritten to its exclusive prefix.  z_lin is written in natural order, in place of r; the
// caller's k_fft_bit_reverse then moves it to the bit-reversed layout of the reference.
//
// Quotient numerator (evaluateFirstPartNumReverse, evaluateSecondPartNumReverse and the omega-fold, permutation.go:78-121,
// 206-214): one elementwise kernel over the storage index p of the bit-reversed DIF outputs lt1, lt2, lz; with i = rev(p)
//   out[p] = omega (lz[p] - 1) u[i] + ((eps - lt2[p]) lz[rev(i + 1 mod n)] - (eps - lt1[p]) lz[p]) (g^n - 1)^-1,
// u[i] = (g w^i - 1)^-1 by the tile inversion (the set of leaves a tile inverts need not be consecutive i).  The reference's
// factor (g^n - 1) on the second part and (g^n - 1)^-1 on the sum cancel exactly in the first term.
// Field arithmetic is exact and every fp_* result is fully reduced, so any grouping gives the reference's limbs.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "field.cuh"
#include "poly_kernels.cuh"
#include "vec_io.cuh"

using namespace gmsm;

namespace {

// tile of the batch inversion: 2^PERM_INV_LOG_T elements, 2T shared slots (32 KB for the 32-byte fields, 40 KB for bw6-633,
// 48 KB for bw6-761: within the default dynamic shared-memory limit), PERM_INV_THREADS threads walking the tree levels
constexpr int PERM_INV_LOG_T = 9;
constexpr unsigned PERM_INV_THREADS = 256;
constexpr int PERM_INV_MAX_LEAVES_PER_THREAD = 32;   // bit mask of zero leaves per thread: T <= 32 blockDim.x

template <class P>
constexpr size_t perm_inv_smem_bytes(int log_t) {
  return (size_t(2) << log_t) * sizeof(Fp<P>);
}

// leaves s[T .. 2T) -> their inverses (a leaf must not be zero: callers substitute one); s[1 .. T) are overwritten
template <class P>
GMSM_D void perm_tree_invert(Fp<P>* s, uint32_t T) {
  const uint32_t B = blockDim.x, tid = threadIdx.x;
  for (uint32_t c = T >> 1; c >= 1; c >>= 1) {
    for (uint32_t k = c + tid; k < 2 * c; k += B) store_vec(s + k, fp_mul(load_vec(s + 2 * k), load_vec(s + 2 * k + 1)));
    __syncthreads();
  }
  if (tid == 0) store_vec(s + 1, fp_inv(load_vec(s + 1)));
  __syncthreads();
  for (uint32_t c = 1; c < T; c <<= 1) {
    for (uint32_t k = c + tid; k < 2 * c; k += B) {
      const Fp<P> inv = load_vec(s + k), a = load_vec(s + 2 * k), b = load_vec(s + 2 * k + 1);
      store_vec(s + 2 * k, fp_mul(inv, b));
      store_vec(s + 2 * k + 1, fp_mul(inv, a));
    }
    __syncthreads();
  }
}

// out[i] = a[i]^-1 (0 -> 0) for i < n.  One block per tile of 2^log_t elements, blockDim.x >= 2^log_t / 32, dynamic shared memory
// perm_inv_smem_bytes.  out may equal a (each block reads its tile before it writes it).
template <class P>
__global__ void k_fr_batch_invert(const Fp<P>* a, uint64_t n, int log_t, Fp<P>* out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Fp<P>* s = reinterpret_cast<Fp<P>*>(smem_raw);
  const uint32_t T = 1u << log_t, B = blockDim.x, tid = threadIdx.x;
  const uint64_t base = (uint64_t)blockIdx.x * T;
  uint32_t zero = 0;
  for (uint32_t j = tid, q = 0; j < T; j += B, q++) {
    const Fp<P> v = base + j < n ? load_vec(a + base + j) : Fp<P>::one();
    if (v.is_zero()) zero |= 1u << q;
    store_vec(s + T + j, v.is_zero() ? Fp<P>::one() : v);
  }
  __syncthreads();
  perm_tree_invert(s, T);
  for (uint32_t j = tid, q = 0; j < T; j += B, q++)
    if (base + j < n) store_vec(out + base + j, (zero >> q) & 1u ? Fp<P>::zero() : load_vec(s + T + j));
}

// r[j] = (eps - t1[j]) (eps - t2[j])^-1 (0 -> 0) for j < n; launch shape as k_fr_batch_invert.  r must not overlap t1 or t2.
template <class P>
__global__ void k_perm_ratio(const Fp<P>* t1, const Fp<P>* t2, uint64_t n, Fp<P> eps, int log_t, Fp<P>* r) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Fp<P>* s = reinterpret_cast<Fp<P>*>(smem_raw);
  const uint32_t T = 1u << log_t, B = blockDim.x, tid = threadIdx.x;
  const uint64_t base = (uint64_t)blockIdx.x * T;
  uint32_t zero = 0;
  for (uint32_t j = tid, q = 0; j < T; j += B, q++) {
    const Fp<P> d = base + j < n ? fp_sub(eps, load_vec(t2 + base + j)) : Fp<P>::one();
    if (d.is_zero()) zero |= 1u << q;
    store_vec(s + T + j, d.is_zero() ? Fp<P>::one() : d);
  }
  __syncthreads();
  perm_tree_invert(s, T);
  for (uint32_t j = tid, q = 0; j < T; j += B, q++)
    if (base + j < n)
      store_vec(r + base + j, (zero >> q) & 1u ? Fp<P>::zero() : fp_mul(fp_sub(eps, load_vec(t1 + base + j)), load_vec(s + T + j)));
}

// Stages tile blockIdx.x of x (m elements, one past the end) in the padded layout of poly_kernels.cuh (element j at slot
// j + j / L, thread t's pad slot after its chunk), forms each chunk's product in its pad slot and runs the up-sweep of a
// right-rooted product tree: afterwards the pad slot of thread t with t = -1 mod 2^k holds the product of the 2^k chunks that end
// at chunk t; thread B - 1's holds the tile product.
template <class P>
GMSM_D void perm_tile_up(Fp<P>* s, const Fp<P>* x, uint64_t m, int log_l) {
  const uint32_t B = blockDim.x, tid = threadIdx.x, L = 1u << log_l, T = B << log_l;
  const uint64_t base = (uint64_t)blockIdx.x * T;
  for (uint32_t j = tid; j < T; j += B) {
    const uint64_t i = base + j;
    store_vec(s + j + (j >> log_l), i < m ? load_vec(x + i) : Fp<P>::one());
  }
  __syncthreads();
  Fp<P>* c = s + tid * (L + 1);
  Fp<P> acc = load_vec(c);
  for (uint32_t j = 1; j < L; j++) acc = fp_mul(acc, load_vec(c + j));
  store_vec(c + L, acc);
  __syncthreads();
  for (uint32_t d = 1; d < B; d <<= 1) {
    if ((tid & (2 * d - 1)) == 2 * d - 1) store_vec(c + L, fp_mul(load_vec(s + (tid - d) * (L + 1) + L), load_vec(c + L)));
    __syncthreads();
  }
}

// tile-product pass: heads[tile] = product of the tile's elements.  blockDim.x = B, dynamic shared memory poly_smem_bytes, one
// block per tile.
template <class P>
__global__ void k_perm_prod_heads(const Fp<P>* x, uint64_t m, int log_l, Fp<P>* heads) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Fp<P>* s = reinterpret_cast<Fp<P>*>(smem_raw);
  perm_tile_up(s, x, m, log_l);
  const uint32_t B = blockDim.x, L = 1u << log_l;
  if (threadIdx.x == B - 1) store_vec(heads + blockIdx.x, load_vec(s + (B - 1) * (L + 1) + L));
}

// write pass: x[i] <- carry[tile] * prod_{tile start <= j < i} x[j] for i < m (the exclusive prefix product; carry == NULL: one),
// in place.  Launch shape as k_perm_prod_heads.
template <class P>
__global__ void k_perm_prod_write(Fp<P>* x, uint64_t m, int log_l, const Fp<P>* carry) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Fp<P>* s = reinterpret_cast<Fp<P>*>(smem_raw);
  const uint32_t B = blockDim.x, tid = threadIdx.x, L = 1u << log_l, T = B << log_l;
  const uint64_t base = (uint64_t)blockIdx.x * T;
  const Fp<P> cin = carry ? load_vec(carry + blockIdx.x) : Fp<P>::one();
  perm_tile_up(s, x, m, log_l);
  Fp<P>* c = s + tid * (L + 1);
  // down-sweep: a segment's slot takes the product of everything before it (the root: the carry-in); its left half inherits it,
  // its right half gets (that product) x (left half's product)
  if (tid == B - 1) store_vec(c + L, cin);
  __syncthreads();
  for (uint32_t d = B >> 1; d >= 1; d >>= 1) {
    if ((tid & (2 * d - 1)) == 2 * d - 1) {
      Fp<P>* l = s + (tid - d) * (L + 1) + L;
      const Fp<P> e = load_vec(c + L), y = load_vec(l);
      store_vec(l, e);
      store_vec(c + L, fp_mul(e, y));
    }
    __syncthreads();
  }
  Fp<P> acc = load_vec(c + L);   // product of everything before this thread's chunk
  for (uint32_t j = 0; j < L; j++) {
    const Fp<P> v = load_vec(c + j);
    store_vec(c + j, acc);
    acc = fp_mul(acc, v);
  }
  __syncthreads();
  for (uint32_t j = tid; j < T; j += B) {
    const uint64_t i = base + j;
    if (i < m) store_vec(x + i, load_vec(s + j + (j >> log_l)));
  }
}

// the constants of the numerator, computed on the host from the domain
template <class P>
struct PermNumConsts {
  Fp<P> eps, omega;   // the challenges "epsilon" and "omega"
  Fp<P> g;            // FrMultiplicativeGen (the coset shift)
  Fp<P> tn_inv;       // (g^n - 1)^-1
};

// out[p] for p < n (n = 2^logn), as in the header comment; tw[j] = w^j for j < n / 2 (the domain's twiddles).  Launch shape as
// k_fr_batch_invert.  out must not overlap lt1, lt2 or lz (lz is read at neighbouring positions).
template <class P>
__global__ void k_perm_numerator(const Fp<P>* lt1, const Fp<P>* lt2, const Fp<P>* lz, uint64_t n, int logn, PermNumConsts<P> k,
                                 const Fp<P>* tw, int log_t, Fp<P>* out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Fp<P>* s = reinterpret_cast<Fp<P>*>(smem_raw);
  const uint32_t T = 1u << log_t, B = blockDim.x, tid = threadIdx.x;
  const uint64_t base = (uint64_t)blockIdx.x * T, half = n >> 1;
  auto rev = [logn](uint64_t v) -> uint64_t { return logn ? (__brevll(v) >> (64 - logn)) : 0ull; };
  for (uint32_t j = tid; j < T; j += B) {
    const uint64_t p = base + j;
    Fp<P> v = Fp<P>::one();
    if (p < n) {
      const uint64_t i = rev(p);
      const Fp<P> wi = i == 0 ? Fp<P>::one() : i < half ? load_vec(tw + i) : fp_neg(load_vec(tw + (i - half)));   // w^(j + n/2) = -w^j
      v = fp_sub(fp_mul(k.g, wi), Fp<P>::one());   // never zero: g is outside the subgroup of order n
    }
    store_vec(s + T + j, v);
  }
  __syncthreads();
  perm_tree_invert(s, T);
  for (uint32_t j = tid; j < T; j += B) {
    const uint64_t p = base + j;
    if (p >= n) continue;
    const uint64_t i = rev(p), pn = rev(i + 1 == n ? 0 : i + 1);
    const Fp<P> z = load_vec(lz + p), zn = load_vec(lz + pn);
    const Fp<P> first = fp_sub(fp_mul(fp_sub(k.eps, load_vec(lt2 + p)), zn), fp_mul(fp_sub(k.eps, load_vec(lt1 + p)), z));
    const Fp<P> second = fp_mul(fp_sub(z, Fp<P>::one()), load_vec(s + T + j));
    store_vec(out + p, fp_add(fp_mul(k.omega, second), fp_mul(first, k.tn_inv)));
  }
}

// ---- launch schedule (host), shared by fft.cu and the CPU emulation ----

// x[k] <- prod_{j<k} x[j] for k < n, in place (the exclusive prefix product); work: poly_levels(n, log_l + log_b).work elements.
// heads(x, m, out, tiles) and write(x, m, carry, tiles) launch k_perm_prod_heads / k_perm_prod_write.
template <class P, class Heads, class Write>
void perm_prefix_schedule(Fp<P>* x, uint64_t n, Fp<P>* work, int log_l, int log_b, Heads&& heads, Write&& write) {
  const int log_t = log_l + log_b;
  const PolyLevels lv = poly_levels(n, log_t);
  auto level = [&](int l) { return l ? work + lv.off[l] : x; };
  auto tiles = [&](int l) { return ((lv.m[l] - 1) >> log_t) + 1; };
  for (int l = 0; l < lv.top; l++) heads(level(l), lv.m[l], level(l + 1), tiles(l));
  for (int l = lv.top; l >= 0; l--) write(level(l), lv.m[l], l < lv.top ? level(l + 1) : nullptr, tiles(l));
}

}  // namespace
