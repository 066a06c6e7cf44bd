// Device side of plookup.ProveLookupVector's Fr steps (ecc/bn254/fr/plookup/vector.go; the plookup packages of the other pairing
// curves are the same generated code): sort.Sort(fr.Vector), the accumulation polynomial z and the quotient numerator on the coset
// of size 2s.  In a header of their own, like perm_kernels.cuh, so that the CPU kernel emulation of tests/emu/ compiles and runs
// them too (tests/test_emu_plookup_cpu.py); fft.cu includes this file and holds the entry points.  The launch schedule of the sort
// below is shared by both.
//
// Sort (sort.Sort(fr.Vector): ascending by fr.Element.Cmp, the canonical value, fr/element.go:254).  Equal keys are bit-identical,
// so the result is unique.  The keys are converted to canonical form once, sorted by an LSD radix sort over their canonical bytes
// (8-bit digits, least significant byte first) and converted back to Montgomery form.  A byte position at which every key has the
// same byte is skipped: k_sort_diff ORs key ^ key[0] over the vector first, and only the bytes where that OR is non-zero are
// passes (range and XOR tables hold small values; the always-zero top bits of every field go too).  A pass is three steps:
//   k_sort_tile<false>: block b counts the digits of its tile of T = blockDim.x 2^log_r keys -> counts[d nb + b];
//   k_sort_row_totals / k_sort_row_scan: counts becomes its exclusive prefix sum in (digit, block) order, the first output slot of
//     block b's keys of digit d;
//   k_sort_tile<true>: block b walks its tile again and writes each key to counts[d nb + b] + (its rank among the tile's keys of
//     digit d), the rank taken without atomics: a round covers blockDim.x consecutive keys, __match_any_sync gives each lane its
//     peers of the same digit in the warp (rank in the warp: the peers below it), and one thread per digit turns the per-warp
//     counts into a prefix over the warps and the rounds before.  The rank follows the tile order, so every pass is stable and the
//     sort is exact and deterministic.
//
// Accumulation polynomial (evaluateAccumulationPolynomial, vector.go:52-95): z[0] = 1, z[i+1] = z[i] r[i] with
//   r[i] = (1+b)(g+f[i])(g(1+b)+t[i]+b t[i+1]) [(g(1+b)+h1[i]+b h1[i+1])(g(1+b)+h2[i]+b h2[i+1])]^-1   (0^-1 -> 0, fr.BatchInvert)
// k_plookup_ratio writes r with the tile inversion of perm_kernels.cuh; the exclusive prefix product is the permutation's scan
// (k_perm_prod_heads / k_perm_prod_write over poly_levels), in place.  z stays in natural order, as in the reference.
//
// Quotient numerator (evaluateNumBitReversed, evaluateZStartsByOneBitReversed, evaluateZEndsByOneBitReversed,
// evaluateOverlapH1h2BitReversed and computeQuotientCanonical up to its FFTInverse, vector.go:97-335): one elementwise kernel over
// the storage index p of the bit-reversed DIF outputs on the coset of size n = 2s.  With i = rev(p), q = rev(i + 2 mod n) (the
// neighbour x g of x = c w^i, g = w^2 the small domain's generator), gg = g^(s-1), A = g(1+b):
//   m   = (1+b) lz[p] (g+lf[p]) (A + lt[p] + b lt[q]),   nn = lz[q] (A + lh1[p] + b lh1[q]) (A + lh2[p] + b lh2[q])
//   out = ((alpha (lh1[p] - lh2[q]) dn + (lz[p] - 1) dn) alpha + (lz[p] - 1) d0) alpha + (m - nn)(x - gg) (x^s - 1)^-1
// with d0 = (x - 1)^-1, dn = (x - gg)^-1, both from one tile inversion of (x - 1)(x - gg), and (x^s - 1)^-1 one of two host
// constants (x^s = c^s (-1)^i).  The reference multiplies the three boundary terms by (x^s - 1) and the fold by (x^s - 1)^-1; the
// pair cancels exactly.  Field arithmetic is exact and every fp_* result is fully reduced, so any grouping gives the reference's
// limbs.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "field.cuh"
#include "perm_kernels.cuh"
#include "vec_io.cuh"

using namespace gmsm;

namespace {

// the sort's tile: blockDim.x = 2^SORT_LOG_B threads (a multiple of 32), 2^SORT_LOG_R rounds of blockDim.x keys
constexpr int SORT_LOG_B = 8;
constexpr int SORT_LOG_R = 4;
constexpr int SORT_MAX_WARPS = 8;   // blockDim.x <= 256
constexpr int SORT_DIGITS = 256;

template <class P>
GMSM_D uint32_t sort_digit(const Fp<P>& k, int byte) {
  uint32_t limb = 0;
#pragma unroll
  for (int w = 0; w < Fp<P>::N; w++)   // a select, not a dynamic register index (which would go through local memory)
    if (w == (byte >> 2)) limb = k.l[w];
  return (limb >> ((byte & 3) * 8)) & 0xffu;
}

// part[b N + j] = OR over block b's tile of 2^log_t keys of (canonical(in[i]) ^ canonical(in[0])), limb j
template <class P>
__global__ void k_sort_diff(const Fp<P>* in, uint64_t n, int log_t, uint32_t* part) {
  __shared__ uint32_t acc[Fp<P>::N];
  const uint32_t T = 1u << log_t, B = blockDim.x, tid = threadIdx.x;
  const uint64_t base = (uint64_t)blockIdx.x << log_t;
  if (tid < (uint32_t)Fp<P>::N) acc[tid] = 0;
  __syncthreads();
  const Fp<P> k0 = fp_from_mont(load_vec(in));
  uint32_t d[Fp<P>::N] = {};
  for (uint32_t j = tid; j < T && base + j < n; j += B) {
    const Fp<P> k = fp_from_mont(load_vec(in + base + j));
#pragma unroll
    for (int w = 0; w < Fp<P>::N; w++) d[w] |= k.l[w] ^ k0.l[w];
  }
#pragma unroll
  for (int w = 0; w < Fp<P>::N; w++)
    if (d[w]) atomicOr(&acc[w], d[w]);
  __syncthreads();
  if (tid < (uint32_t)Fp<P>::N) part[(uint64_t)blockIdx.x * Fp<P>::N + tid] = acc[tid];
}

// mask[j] = OR of the `parts` rows of part (one block)
template <class P>
__global__ void k_sort_diff_reduce(const uint32_t* part, uint64_t parts, uint32_t* mask) {
  __shared__ uint32_t acc[Fp<P>::N];
  const uint32_t tid = threadIdx.x;
  if (tid < (uint32_t)Fp<P>::N) acc[tid] = 0;
  __syncthreads();
  for (uint64_t b = tid; b < parts; b += blockDim.x)
    for (int w = 0; w < Fp<P>::N; w++)
      if (part[b * Fp<P>::N + w]) atomicOr(&acc[w], part[b * Fp<P>::N + w]);
  __syncthreads();
  if (tid < (uint32_t)Fp<P>::N) mask[tid] = acc[tid];
}

// out[i] = canonical(in[i]) (TO_MONT false) or Montgomery(in[i]) (true); out may equal in
template <class P, bool TO_MONT>
__global__ void k_sort_convert(const Fp<P>* in, uint64_t n, Fp<P>* out) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const Fp<P> v = load_vec(in + i);
    store_vec(out + i, TO_MONT ? fp_to_mont(v) : fp_from_mont(v));
  }
}

// SCATTER false: counts[d nb + b] = keys of digit d in block b's tile.  SCATTER true: dst[counts[d nb + b] + rank] = key for every
// key of the tile (counts already scanned).  blockDim.x a multiple of 32, at most 32 SORT_MAX_WARPS threads; tile = blockDim.x << log_r.
template <class P, bool SCATTER>
__global__ void k_sort_tile(const Fp<P>* src, uint64_t n, int byte, int log_r, uint32_t* counts, uint64_t nb, Fp<P>* dst) {
  __shared__ uint32_t run[SORT_DIGITS];                   // keys of each digit before this round (plus the block's first slot)
  __shared__ uint32_t wcnt[SORT_MAX_WARPS][SORT_DIGITS];  // this round: keys of digit d in warp w (zero between rounds)
  __shared__ uint32_t woff[SORT_MAX_WARPS][SORT_DIGITS];  // this round: first slot of warp w's keys of digit d
  const uint32_t B = blockDim.x, tid = threadIdx.x, lane = tid & 31u, w = tid >> 5, W = B >> 5;
  const uint64_t base = ((uint64_t)blockIdx.x * B) << log_r;
  for (uint32_t d = tid; d < SORT_DIGITS; d += B) {
    run[d] = SCATTER ? counts[d * nb + blockIdx.x] : 0u;
    for (uint32_t v = 0; v < W; v++) wcnt[v][d] = 0;
  }
  __syncthreads();
  for (uint32_t r = 0; r < (1u << log_r); r++) {
    const uint64_t i = base + (uint64_t)r * B + tid;
    const bool valid = i < n;
    const uint32_t dig = valid ? sort_digit(load_vec(src + i), byte) : SORT_DIGITS;   // past-the-end lanes: a group of their own
    const uint32_t peers = __match_any_sync(0xffffffffu, dig);
    const uint32_t rank = __popc(peers & ((1u << lane) - 1u));
    if (valid && rank == 0) wcnt[w][dig] = __popc(peers);
    __syncthreads();
    for (uint32_t d = tid; d < SORT_DIGITS; d += B) {
      uint32_t acc = run[d];
      for (uint32_t v = 0; v < W; v++) {
        woff[v][d] = acc;
        acc += wcnt[v][d];
        wcnt[v][d] = 0;
      }
      run[d] = acc;
    }
    __syncthreads();
    // the key is loaded again (a cache hit) rather than kept across the barriers: for the 40- and 48-byte fields a live key
    // would be placed in local memory
    if (SCATTER && valid) store_vec(dst + woff[w][dig] + rank, load_vec(src + i));
  }
  if (!SCATTER) {
    __syncthreads();
    for (uint32_t d = tid; d < SORT_DIGITS; d += B) counts[d * nb + blockIdx.x] = run[d];
  }
}

// totals[d] = sum of row d of counts (nb entries); one block per digit
__global__ void k_sort_row_totals(const uint32_t* counts, uint64_t nb, uint32_t* totals) {
  __shared__ uint32_t acc;
  if (threadIdx.x == 0) acc = 0;
  __syncthreads();
  uint32_t s = 0;
  for (uint64_t b = threadIdx.x; b < nb; b += blockDim.x) s += counts[blockIdx.x * nb + b];
  atomicAdd(&acc, s);
  __syncthreads();
  if (threadIdx.x == 0) totals[blockIdx.x] = acc;
}

// row d of counts -> its exclusive prefix sum plus the keys of every smaller digit; one block per digit, blockDim.x <= 256
__global__ void k_sort_row_scan(uint32_t* counts, uint64_t nb, const uint32_t* totals) {
  __shared__ uint32_t part[256];
  __shared__ uint32_t start;
  const uint32_t B = blockDim.x, tid = threadIdx.x, d = blockIdx.x;
  if (tid == 0) {
    uint32_t s = 0;
    for (uint32_t e = 0; e < d; e++) s += totals[e];
    start = s;
  }
  uint32_t* row = counts + d * nb;
  const uint64_t chunk = (nb + B - 1) / B, lo = tid * chunk < nb ? tid * chunk : nb, hi = lo + chunk < nb ? lo + chunk : nb;
  uint32_t s = 0;
  for (uint64_t b = lo; b < hi; b++) s += row[b];
  part[tid] = s;
  __syncthreads();
  for (uint32_t off = 1; off < B; off <<= 1) {   // inclusive Hillis-Steele scan of the thread sums
    const uint32_t v = tid >= off ? part[tid - off] : 0u;
    __syncthreads();
    part[tid] += v;
    __syncthreads();
  }
  uint32_t acc = start + part[tid] - s;
  for (uint64_t b = lo; b < hi; b++) {
    const uint32_t c = row[b];
    row[b] = acc;
    acc += c;
  }
}

// ---- the sort's workspace and launch schedule (host), shared by fft.cu and the CPU emulation ----

struct SortLayout {
  uint64_t tiles = 0;       // blocks of the digit passes
  uint64_t diff_tiles = 0;  // blocks of k_sort_diff
  size_t keys = 0, counts = 0, totals = 0, part = 0, mask = 0, bytes = 0;   // byte offsets into the workspace, total bytes
};
constexpr int SORT_DIFF_LOG_T = 12;

inline size_t sort_align(size_t b) { return (b + 255) & ~size_t(255); }

template <class P>
SortLayout sort_layout(uint64_t n, int log_r, int log_b) {
  SortLayout s;
  s.tiles = ((n - 1) >> (log_r + log_b)) + 1;
  s.diff_tiles = ((n - 1) >> SORT_DIFF_LOG_T) + 1;
  s.counts = sort_align(n * sizeof(Fp<P>));
  s.totals = s.counts + sort_align(s.tiles * SORT_DIGITS * 4);
  s.part = s.totals + sort_align(SORT_DIGITS * 4);
  s.mask = s.part + sort_align(s.diff_tiles * Fp<P>::N * 4);
  s.bytes = s.mask + sort_align(Fp<P>::N * 4);
  return s;
}

// out = in sorted ascending by canonical value (n >= 1; out may equal in; work: sort_layout(...).bytes).  launch(kernel, grid,
// block, args...) launches a kernel on the caller's stream; read_mask(host, device, words) copies the difference mask to the host
// once the kernels before it have run.
template <class P, class Launch, class ReadMask>
void fr_sort_schedule(const Fp<P>* in, uint64_t n, Fp<P>* out, unsigned char* work, int log_r, int log_b, Launch&& launch,
                      ReadMask&& read_mask) {
  using F = Fp<P>;
  const SortLayout L = sort_layout<P>(n, log_r, log_b);
  F* keys = reinterpret_cast<F*>(work);
  uint32_t* counts = reinterpret_cast<uint32_t*>(work + L.counts);
  uint32_t* totals = reinterpret_cast<uint32_t*>(work + L.totals);
  uint32_t* part = reinterpret_cast<uint32_t*>(work + L.part);
  uint32_t* dmask = reinterpret_cast<uint32_t*>(work + L.mask);
  launch(k_sort_diff<P>, (unsigned)L.diff_tiles, 256u, in, n, SORT_DIFF_LOG_T, part);
  launch(k_sort_diff_reduce<P>, 1u, 256u, (const uint32_t*)part, L.diff_tiles, dmask);
  uint32_t mask[F::N];
  read_mask(mask, dmask, F::N);
  int bytes[4 * F::N], passes = 0;
  for (int b = 0; b < 4 * F::N; b++)
    if ((mask[b >> 2] >> ((b & 3) * 8)) & 0xffu) bytes[passes++] = b;
  // ping-pong between out and keys, starting where the last pass lands in out
  F* src = passes & 1 ? keys : out;
  F* dst = passes & 1 ? out : keys;
  const unsigned conv_blocks = (unsigned)((n + 255) / 256 < 8192 ? (n + 255) / 256 : 8192);
  launch(k_sort_convert<P, false>, conv_blocks, 256u, in, n, src);
  for (int k = 0; k < passes; k++) {
    launch(k_sort_tile<P, false>, (unsigned)L.tiles, 1u << log_b, (const F*)src, n, bytes[k], log_r, counts, L.tiles, (F*)nullptr);
    launch(k_sort_row_totals, (unsigned)SORT_DIGITS, 1u << log_b, (const uint32_t*)counts, L.tiles, totals);
    launch(k_sort_row_scan, (unsigned)SORT_DIGITS, 1u << log_b, counts, L.tiles, (const uint32_t*)totals);
    launch(k_sort_tile<P, true>, (unsigned)L.tiles, 1u << log_b, (const F*)src, n, bytes[k], log_r, counts, L.tiles, dst);
    F* t = src;
    src = dst;
    dst = t;
  }
  launch(k_sort_convert<P, true>, conv_blocks, 256u, (const F*)out, n, out);
}

// ---- accumulation polynomial and quotient numerator ----

// the challenges and their combinations, computed on the host
template <class P>
struct PlookupConsts {
  Fp<P> beta, gamma;
  Fp<P> opb;    // 1 + beta
  Fp<P> gopb;   // gamma (1 + beta)
};

// r[i] for i < n - 1 as in the header comment, r[n - 1] = 1 (the exclusive prefix product never reads it).  Launch shape as
// k_fr_batch_invert.  r must not overlap f, t, h1 or h2.
template <class P>
__global__ void k_plookup_ratio(const Fp<P>* f, const Fp<P>* t, const Fp<P>* h1, const Fp<P>* h2, uint64_t n, PlookupConsts<P> k,
                                int log_t, Fp<P>* r) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Fp<P>* s = reinterpret_cast<Fp<P>*>(smem_raw);
  const uint32_t T = 1u << log_t, B = blockDim.x, tid = threadIdx.x;
  const uint64_t base = (uint64_t)blockIdx.x * T;
  uint32_t zero = 0;
  for (uint32_t j = tid, q = 0; j < T; j += B, q++) {
    const uint64_t i = base + j;
    Fp<P> d = Fp<P>::one();
    if (i + 1 < n) {
      const Fp<P> a = fp_add(fp_add(k.gopb, load_vec(h1 + i)), fp_mul(k.beta, load_vec(h1 + i + 1)));
      const Fp<P> b = fp_add(fp_add(k.gopb, load_vec(h2 + i)), fp_mul(k.beta, load_vec(h2 + i + 1)));
      d = fp_mul(a, b);
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
        const Fp<P> u = fp_add(fp_add(k.gopb, load_vec(t + i)), fp_mul(k.beta, load_vec(t + i + 1)));
        v = fp_mul(fp_mul(fp_mul(k.opb, fp_add(k.gamma, load_vec(f + i))), u), load_vec(s + T + j));
      }
    }
    store_vec(r + i, v);
  }
}

// the constants of the numerator, computed on the host from the big domain
template <class P>
struct PlookupNumConsts {
  PlookupConsts<P> c;
  Fp<P> alpha;
  Fp<P> shift;      // FrMultiplicativeGen (the coset shift)
  Fp<P> gg;         // g^(s-1), g = w^2 the small domain's generator
  Fp<P> xs_inv[2];  // (shift^s - 1)^-1, (-shift^s - 1)^-1: (x^s - 1)^-1 for even and odd i
};

// out[p] for p < n (n = 2s = 2^logn), as in the header comment; tw[j] = w^j for j < n / 2 (the big domain's twiddles).  Launch
// shape as k_fr_batch_invert.  out must not overlap the inputs (they are read at neighbouring positions).
template <class P>
__global__ void k_plookup_numerator(const Fp<P>* lz, const Fp<P>* lh1, const Fp<P>* lh2, const Fp<P>* lt, const Fp<P>* lf, uint64_t n,
                                    int logn, PlookupNumConsts<P> k, const Fp<P>* tw, int log_t, Fp<P>* out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Fp<P>* s = reinterpret_cast<Fp<P>*>(smem_raw);
  const uint32_t T = 1u << log_t, B = blockDim.x, tid = threadIdx.x;
  const uint64_t base = (uint64_t)blockIdx.x * T, half = n >> 1;
  auto rev = [logn](uint64_t v) -> uint64_t { return logn ? (__brevll(v) >> (64 - logn)) : 0ull; };
  auto point = [&](uint64_t i) -> Fp<P> {   // x = shift w^i (w^(j + n/2) = -w^j)
    const Fp<P> wi = i == 0 ? Fp<P>::one() : i < half ? load_vec(tw + i) : fp_neg(load_vec(tw + (i - half)));
    return fp_mul(k.shift, wi);
  };
  for (uint32_t j = tid; j < T; j += B) {
    const uint64_t p = base + j;
    Fp<P> v = Fp<P>::one();
    if (p < n) {
      const Fp<P> x = point(rev(p));
      v = fp_mul(fp_sub(x, Fp<P>::one()), fp_sub(x, k.gg));   // never zero: the shift is outside the subgroup of order n
    }
    store_vec(s + T + j, v);
  }
  __syncthreads();
  perm_tree_invert(s, T);
  for (uint32_t j = tid; j < T; j += B) {
    const uint64_t p = base + j;
    if (p >= n) continue;
    const uint64_t i = rev(p), q = rev(i + 2 >= n ? i + 2 - n : i + 2);
    const Fp<P> x = point(i), inv = load_vec(s + T + j);
    const Fp<P> xg = fp_sub(x, k.gg);
    const Fp<P> d0 = fp_mul(xg, inv), dn = fp_mul(fp_sub(x, Fp<P>::one()), inv);
    const Fp<P> z = load_vec(lz + p), zq = load_vec(lz + q);
    const Fp<P> h1 = load_vec(lh1 + p), h2q = load_vec(lh2 + q);
    Fp<P> m = fp_mul(fp_mul(k.c.opb, z), fp_add(k.c.gamma, load_vec(lf + p)));
    m = fp_mul(m, fp_add(fp_add(k.c.gopb, load_vec(lt + p)), fp_mul(k.c.beta, load_vec(lt + q))));
    Fp<P> nn = fp_add(fp_add(k.c.gopb, h1), fp_mul(k.c.beta, load_vec(lh1 + q)));
    nn = fp_mul(nn, fp_add(fp_add(k.c.gopb, load_vec(lh2 + p)), fp_mul(k.c.beta, h2q)));
    nn = fp_mul(nn, zq);
    const Fp<P> lh = fp_mul(fp_mul(fp_sub(m, nn), xg), (i & 1) ? k.xs_inv[1] : k.xs_inv[0]);
    const Fp<P> z1 = fp_sub(z, Fp<P>::one());
    Fp<P> acc = fp_mul(fp_mul(k.alpha, fp_sub(h1, h2q)), dn);
    acc = fp_mul(fp_add(acc, fp_mul(z1, dn)), k.alpha);
    acc = fp_mul(fp_add(acc, fp_mul(z1, d0)), k.alpha);
    store_vec(out + p, fp_add(acc, lh));
  }
}

}  // namespace
