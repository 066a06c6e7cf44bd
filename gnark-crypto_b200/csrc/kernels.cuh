// sm_90a kernels of the Pippenger bucket method.  One template instantiation per (curve, group).
//
// Pipeline (replaces ecc/bn254/multiexp.go:148-209 `_innerMsmG1` and its callees):
//   K1  k_digits_hist      partitionScalars (multiexp.go:709-803) fused with a bucket histogram
//   K1b k_scan_*           exclusive scan of the histogram -> bucket offsets
//   K1c k_scatter_window   digits -> entries grouped by bucket (positions from K1's ranks, or from a returning atomic)
//   K2  k_accumulate       bucket accumulation (processChunk, multiexp_jacobian.go:20-39) as a
//                          load-balanced segmented reduction over the bucket-ordered entry list
//   K2b k_carry_level      joins partial sums of buckets that span several chunks
//   K3  k_bucket_segments  bucket reduction sum (k+1)*B[k] (multiexp_jacobian.go:44-52), parallel form
//       k_sum_groups       tree sum of segment results -> one partial per window
//   K4  k_finalize         sum over ranks, Horner over windows (msmReduceChunk, multiexp.go:302-315),
//                          xyzz -> Jacobian -> affine normal form (g1.go:726-731, 150-166)
#pragma once
#include <cuda_runtime.h>

#include "groups.cuh"
#include "quad.cuh"
#include "testops.cuh"
#include "vec_io.cuh"

namespace gmsm {

static constexpr uint32_t ID_NONE = 0xFFFFFFFFu;

// out-of-line copies of the rare / cold group operations keep the hot loops small (one mixed add is
// ~2k SASS instructions; the instruction cache is 32 KB L1.5)
template <class F>
__device__ __noinline__ void xyzz_add_cold(XYZZ<F>& p, const XYZZ<F>& q) {
  xyzz_add(p, q);
}
template <class F>
__device__ __noinline__ XYZZ<F> xyzz_double_cold(const XYZZ<F>& q) {
  return xyzz_double(q);
}
// lane-parallel twins (quad.cuh): one point operation per QUAD of lanes
template <class F>
__device__ __noinline__ void xyzz_add_quad_cold(Quad q, XYZZ<F>& p, const XYZZ<F>& a) {
  xyzz_add_quad(q, p, a);
}
template <class F>
__device__ __noinline__ XYZZ<F> xyzz_double_quad_cold(Quad q, const XYZZ<F>& a) {
  return xyzz_double_quad(q, a);
}
// The tail kernels below exist in two forms selected by the template flag Q: Q = false, one thread per work item (serial
// chain); Q = true, one quad per work item (4x the threads, ~3x shorter chains).  The host picks Q = true whenever the
// 4x grid still fits the machine in about one wave -- these stages are then bound by the latency of the chain, not by
// the multiplier pipe.
template <bool Q, class F>
GMSM_D void tail_add(const Quad& q, XYZZ<F>& p, const XYZZ<F>& a) {
  if constexpr (Q) xyzz_add_quad_cold(q, p, a); else xyzz_add_cold(p, a);
}
template <bool Q, class F>
GMSM_D XYZZ<F> tail_double(const Quad& q, const XYZZ<F>& a) {
  if constexpr (Q) return xyzz_double_quad_cold(q, a); else return xyzz_double_cold(a);
}

// ------------------------------------------------------------------------------------------
// K1: signed-digit recoding.  Calls fn(window, magnitude >= 1, sign) for every non-zero digit.
// Semantics of partitionScalars (multiexp.go:743-800): zero scalars skipped; digit = carry + c bits;
// windows 0..W-2 borrow (digit > 2^(c-1)-1 -> digit -= 2^c, carry 1); last window never borrows.
// ------------------------------------------------------------------------------------------
// One scalar's signed digits, window by window (next() must be called for j = 0, 1, ..., W-1 in order).
template <class G>
struct DigitStream {
  static constexpr int N = G::Fr::N;
  uint32_t v[N];
  uint32_t carry, mask, maxd;
  int c, nwin;
  GMSM_D void init(const typename G::Fr& s_mont, int c_, int nwin_) {
    const typename G::Fr k = fp_from_mont(s_mont);            // Bits(), fr/element.go:855-859
#pragma unroll
    for (int i = 0; i < N; i++) v[i] = k.l[i];
    c = c_;
    nwin = nwin_;
    mask = (1u << c_) - 1u;
    maxd = (1u << (c_ - 1)) - 1u;
    carry = 0;
  }
  GMSM_D uint32_t next(int j) {
    uint32_t d = (v[0] & mask) + carry;
    // 256-bit logical shift right by c (c < 32)
#pragma unroll
    for (int i = 0; i < N - 1; i++) v[i] = __funnelshift_r(v[i], v[i + 1], c);
    v[N - 1] >>= c;
    if (j < nwin - 1) {
      carry = 0;
      if (d > maxd) {
        // negative digit d - 2^c, magnitude 2^c - d  (0 when an all-ones window meets a carry:
        // digit 0 with a carry out, nothing to add)
        const uint32_t mag = (1u << c) - d;
        carry = 1;
        return mag ? (((mag - 1u) << 1) | 1u) : 0u;
      }
      return d << 1;
    }
    return d << 1;  // multiexp.go:788-800: the last window never borrows
  }
};

template <class G, class Fn>
GMSM_D void for_each_digit(const typename G::Fr& s_mont, int c, int nwin, Fn fn) {
  if (s_mont.is_zero()) {                 // IsZero() on the Montgomery limbs, multiexp.go:743
    for (int j = 0; j < nwin; j++) fn(j, 0u);
    return;
  }
  DigitStream<G> ds;
  ds.init(s_mont, c, nwin);
  for (int j = 0; j < nwin; j++) fn(j, ds.next(j));
}

// bucket index inside its window for a non-zero code: magnitude - 1
GMSM_D uint32_t code_bucket(uint32_t code) { return (code >> 1) - 1u + (code & 1u); }

// K1: digits (stored chunk-major, digits[j*n + i], the reference's layout multiexp.go:785) + bucket histogram.
//
// The counting sort that follows needs, for every entry, its position inside its bucket.  Two modes, chosen per call by a
// sampling pass over the scalars (k_skew_probe -> flag in device memory, read by K1 and by the scatter kernels):
//   * plain mode (flag = 0, random-looking scalars): K1 counts with fire-and-forget atomics (RED) and the scatter takes the
//     positions with a returning atomicSub per entry -- most of the scatter runs on the auxiliary stream underneath the
//     accumulate kernel, so its atomics are off the critical path.
//   * rank mode (flag = 1, skewed scalars): K1's atomic RETURNS, which numbers the entry inside its bucket (ranks[j*n + i]),
//     and is warp-aggregated -- lanes of a warp that hit the same bucket (__match_any_sync) send ONE atomicAdd of their count and
//     number themselves locally; the scatter then needs no atomics at all.  Skewed inputs -- the reference's "redundancy"
//     benchmark (runs of 100 equal scalars) or "smallvalues" (n/5 equal scalars), multiexp_test.go:316-334 -- otherwise put
//     millions of atomics on a handful of addresses, one window per scatter launch; here all W hot addresses are in flight at
//     once and 32 equal lanes cost one atomic.
// Why not always rank mode: MATCH.ANY iterates over the DISTINCT keys of a warp (~32 rounds for random digits) and returning
// atomics cost about twice a RED: both the aggregated and the plain returning form were slower than the RED histogram at
// n = 2^24, W = 15.  In rank mode the returning atomics of DIGIT_BATCH windows are issued back to
// back and consumed afterwards (one L2 round trip per batch).  Lanes past the end walk the loop with a zero scalar so that
// every lane of a warp reaches the collectives.
static constexpr int DIGIT_BATCH = 8;
static constexpr uint32_t PROBE_SAMPLES = 16384, PROBE_BINS = 2048;

// flag[0] |= 1 if, in this block's strided sample of the scalars (PROBE_BLOCKS blocks x PROBE_PER_BLOCK samples), one digit value
// of window 0 owns more than 1/32 of the sample (a global hot spot) or more than 1/32 of the sampled scalars equal their
// successor (runs of equal scalars).  flag[] is cleared with the histogram before every call.
static constexpr uint32_t PROBE_BLOCKS = 16, PROBE_PER_BLOCK = PROBE_SAMPLES / PROBE_BLOCKS;
template <class G>
__global__ void __launch_bounds__(256) k_skew_probe(const typename G::Fr* __restrict__ scalars, uint32_t n, int c, int nwin, uint32_t* __restrict__ flag) {
  __shared__ uint32_t bins[PROBE_BINS];
  __shared__ uint32_t maxc, pairs;
  for (uint32_t k = threadIdx.x; k < PROBE_BINS; k += blockDim.x) bins[k] = 0;
  if (threadIdx.x == 0) { maxc = 0; pairs = 0; }
  __syncthreads();
  const uint32_t S = n < PROBE_SAMPLES ? n : PROBE_SAMPLES;          // samples of the whole grid
  const uint64_t stride = S ? (uint64_t)n / S : 1;
  const uint32_t k_lo = blockIdx.x * PROBE_PER_BLOCK, k_hi = (k_lo + PROBE_PER_BLOCK < S) ? k_lo + PROBE_PER_BLOCK : S;
  const uint32_t mine = k_hi > k_lo ? k_hi - k_lo : 0;
  for (uint32_t k = k_lo + threadIdx.x; k < k_hi; k += blockDim.x) {
    const size_t i = (size_t)((uint64_t)k * stride);
    typename G::Fr s = load_vec_ro(scalars + i);
    if (s.is_zero()) continue;                    // zero scalars produce no entries
    if (i + 1 < n) {
      typename G::Fr t = load_vec_ro(scalars + i + 1);
      if (t == s) atomicAdd(&pairs, 1u);
    }
    DigitStream<G> ds;
    ds.init(s, c, nwin);
    const uint32_t code = ds.next(0);
    if (code) atomicAdd(&bins[(code * 2654435761u) >> 21], 1u);
  }
  __syncthreads();
  uint32_t m = 0;
  for (uint32_t k = threadIdx.x; k < PROBE_BINS; k += blockDim.x) m = max(m, bins[k]);
  atomicMax(&maxc, m);
  __syncthreads();
  if (threadIdx.x == 0 && mine >= 256u && (maxc * 32u > mine || pairs * 32u > mine)) atomicOr(flag, 1u);
}

template <class G>
__global__ void k_digits_hist(const typename G::Fr* __restrict__ scalars, uint32_t n, int c, int nwin,
                              uint32_t nb, uint32_t* __restrict__ digits, uint32_t* __restrict__ ranks, uint32_t* __restrict__ hist,
                              const uint32_t* __restrict__ skew_flag) {
  using Fr = typename G::Fr;
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t lt = (1u << lane) - 1u;
  const bool rank_mode = skew_flag[0] != 0;
  for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x; base < n; base += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t i64 = base + threadIdx.x;
    const bool valid = i64 < n;
    const uint32_t i = (uint32_t)i64;
    Fr s = Fr::zero();
    if (valid) s = load_vec_ro(scalars + i);
    if (!rank_mode) {
      // plain mode: count only (the scatter numbers the entries)
      if (valid)
        for_each_digit<G>(s, c, nwin, [&](int j, uint32_t code) {
          digits[(size_t)j * n + i] = code;
          if (code) atomicAdd(&hist[(uint32_t)j * nb + code_bucket(code)], 1u);
        });
      continue;
    }
    DigitStream<G> ds;
    ds.init(s, c, nwin);       // (a zero scalar walks the windows like any other: all its digits are 0, multiexp.go:743)
    for (int j0 = 0; j0 < nwin; j0 += DIGIT_BATCH) {
      uint32_t code[DIGIT_BATCH], first[DIGIT_BATCH];
      unsigned peers[DIGIT_BATCH];
#pragma unroll
      for (int b = 0; b < DIGIT_BATCH; b++) {
        const int j = j0 + b;
        code[b] = (j < nwin) ? ds.next(j) : 0u;
        const uint32_t key = code[b] ? (uint32_t)j * nb + code_bucket(code[b]) : ID_NONE;
        peers[b] = __match_any_sync(0xffffffffu, key);
        first[b] = 0;
        if (code[b] && (int)lane == __ffs((int)peers[b]) - 1) first[b] = atomicAdd(&hist[key], (uint32_t)__popc(peers[b]));
      }
#pragma unroll
      for (int b = 0; b < DIGIT_BATCH; b++) {
        const int j = j0 + b;
        if (code[b]) first[b] = __shfl_sync(peers[b], first[b], __ffs((int)peers[b]) - 1) + (uint32_t)__popc(peers[b] & lt);
        if (j < nwin && valid) {
          if (code[b]) ranks[(size_t)j * n + i] = first[b];
          digits[(size_t)j * n + i] = code[b];
        }
      }
    }
  }
}

// K1c: scatter of ONE window: entries[position] = (i << 1) | sign.  The engine launches it after k_scan_final_ends, which
// turned the window's counters hist_w[] into bucket END pointers (offsets_w == nullptr): in plain mode the returning
// atomicSub on the counter IS the position (buckets fill from the back, each counter ends at its bucket's offset), so an
// entry costs one atomic and one store; in rank mode the position is end - 1 - rank.  With offsets_w the counters hold
// counts and the positions are offsets_w[b] + (count - 1, count - 2, ...) or offsets_w[b] + rank (the counters then count
// down to zero): the form the CPU emulation of the pipeline drives (tests/emu/emu_engine.cpp, with a host scan).
// Launched window by window so that the randomly written slice of `entries` (<= 4n bytes) and the window's counters stay
// L2-resident and reach HBM once, as full lines, instead of one read-modify-write per 4-byte store.  H100 has 50 MB of L2, so
// the slice fits up to n ~ 2^23; at n = 2^24 (64 MiB) it spills partly, yet the exposed scatter still costs the same per point
// as at n = 2^20 (DESIGN.md section 3).  Well beyond that (2^26) the cost per point about doubles; a window split into bucket
// ranges that fit L2 (what k_scatter_shared does for the window-table mode) would address it and is not done here.
GMSM_D uint32_t scatter_position(uint32_t* __restrict__ counters, const uint32_t* __restrict__ offsets, uint32_t b, bool rank_mode,
                                 uint32_t rk) {
  if (offsets == nullptr) return rank_mode ? counters[b] - 1u - rk : atomicSub(&counters[b], 1u) - 1u;
  return offsets[b] + (rank_mode ? rk : atomicSub(&counters[b], 1u) - 1u);
}
// U independent entries per thread and iteration: the atomics of all U are in flight together
template <int U>
GMSM_D void scatter_window(const uint32_t* __restrict__ digits_w, const uint32_t* __restrict__ ranks_w, uint32_t n,
                           uint32_t* __restrict__ hist_w, const uint32_t* __restrict__ offsets_w, uint32_t* __restrict__ entries,
                           const uint32_t* __restrict__ skew_flag) {
  const bool rank_mode = skew_flag[0] != 0;
  const uint32_t tile = blockDim.x * U;
  for (uint64_t base = (uint64_t)blockIdx.x * tile; base < n; base += (uint64_t)gridDim.x * tile) {
    uint32_t code[U], rk[U], pos[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const uint64_t i = base + (uint64_t)u * blockDim.x + threadIdx.x;
      code[u] = (i < n) ? __ldg(digits_w + i) : 0u;
      rk[u] = (rank_mode && code[u]) ? __ldg(ranks_w + i) : 0u;
    }
#pragma unroll
    for (int u = 0; u < U; u++)
      if (code[u]) pos[u] = scatter_position(hist_w, offsets_w, code_bucket(code[u]), rank_mode, rk[u]);
#pragma unroll
    for (int u = 0; u < U; u++) {
      if (code[u]) {
        const uint32_t i = (uint32_t)(base + (uint64_t)u * blockDim.x + threadIdx.x);
        entries[pos[u]] = (i << 1) | (code[u] & 1u);
      }
    }
  }
}
// on the call's stream, where the scatter has the machine to itself: SCATTER_BLOCKS_PER_SM blocks of 256 threads per SM
static constexpr int SCATTER_U = 4, SCATTER_BLOCKS_PER_SM = 8;
static __global__ void k_scatter_window(const uint32_t* __restrict__ digits_w, const uint32_t* __restrict__ ranks_w, uint32_t n,
                                        uint32_t* __restrict__ hist_w, const uint32_t* __restrict__ offsets_w, uint32_t* __restrict__ entries,
                                        const uint32_t* __restrict__ skew_flag) {
  scatter_window<SCATTER_U>(digits_w, ranks_w, n, hist_w, offsets_w, entries, skew_flag);
}
// on the auxiliary stream, underneath the accumulate: ONE block of 256 threads per SM with twice the entries per thread.  A window
// takes about as long as with the full grid (the scatter is bound by the L2's atomics, not by the threads in flight), and the
// block (44 registers per thread) fits beside three k_accumulate blocks of the 8-limb groups, which fill the register file at four.
static constexpr int SCATTER_AUX_U = 8, SCATTER_AUX_BLOCKS_PER_SM = 1;
static __global__ void k_scatter_window_aux(const uint32_t* __restrict__ digits_w, const uint32_t* __restrict__ ranks_w, uint32_t n,
                                            uint32_t* __restrict__ hist_w, const uint32_t* __restrict__ offsets_w, uint32_t* __restrict__ entries,
                                            const uint32_t* __restrict__ skew_flag) {
  scatter_window<SCATTER_AUX_U>(digits_w, ranks_w, n, hist_w, offsets_w, entries, skew_flag);
}

// K1c (window-table mode, see k_table_level): all W windows feed ONE bucket set -- the entry of (scalar i,
// window j) is the table point j*row_stride + i = 2^(c*j) * P_i, and hist / offsets / ranks are indexed by the bucket
// alone (hist holds end pointers when offsets is null, as in k_scatter_window).  The L2-residency argument of
// k_scatter_window is kept by passing over the digits once per BUCKET RANGE [blo, bhi): a range owns a contiguous slice of
// `entries` (~4n bytes for uniform digits), every pass streams all n*W digits (coalesced) and scatters only the ones of its
// range.  blockIdx.y = window.
static __global__ void k_scatter_shared(const uint32_t* __restrict__ digits, const uint32_t* __restrict__ ranks, uint32_t n, uint32_t row_stride,
                                        uint32_t* __restrict__ hist, const uint32_t* __restrict__ offsets, uint32_t* __restrict__ entries,
                                        uint32_t blo, uint32_t bhi, const uint32_t* __restrict__ skew_flag) {
  constexpr int U = 4;
  const bool rank_mode = skew_flag[0] != 0;
  const uint32_t tile = blockDim.x * U;
  const uint32_t j = blockIdx.y;
  const uint32_t* digits_w = digits + (size_t)j * n;
  const uint32_t* ranks_w = ranks + (size_t)j * n;
  const uint32_t idx0 = j * row_stride;      // (W * row_stride) < 2^31 is checked by the host
  for (uint64_t base = (uint64_t)blockIdx.x * tile; base < n; base += (uint64_t)gridDim.x * tile) {
    uint32_t code[U], rk[U], pos[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const uint64_t i = base + (uint64_t)u * blockDim.x + threadIdx.x;
      code[u] = (i < n) ? __ldg(digits_w + i) : 0u;
      if (code[u]) {
        const uint32_t b = code_bucket(code[u]);
        if (b < blo || b >= bhi) code[u] = 0u;
      }
      rk[u] = (rank_mode && code[u]) ? __ldg(ranks_w + i) : 0u;
    }
#pragma unroll
    for (int u = 0; u < U; u++)
      if (code[u]) pos[u] = scatter_position(hist, offsets, code_bucket(code[u]), rank_mode, rk[u]);
#pragma unroll
    for (int u = 0; u < U; u++) {
      if (code[u]) {
        const uint32_t i = (uint32_t)(base + (uint64_t)u * blockDim.x + threadIdx.x);
        entries[pos[u]] = ((idx0 + i) << 1) | (code[u] & 1u);
      }
    }
  }
}

// test hook: digits in the reference's encoding (multiexp.go:779-785), out[w*n + i]
template <class G>
__global__ void k_digits_dump(const typename G::Fr* __restrict__ scalars, uint32_t n, int c, int nwin,
                              uint32_t* __restrict__ out) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    typename G::Fr s = load_vec_ro(scalars + i);
    for_each_digit<G>(s, c, nwin, [&](int j, uint32_t code) { out[(size_t)j * n + i] = code; });
  }
}

// ------------------------------------------------------------------------------------------
// K1b: exclusive scan over the histogram (nb_total entries) -> offsets[0..nb_total]
// three-phase: per-block totals, scan of the totals (one block), per-block scan + prefix.
// ------------------------------------------------------------------------------------------

GMSM_D uint32_t warp_incl_scan(uint32_t v) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    uint32_t t = __shfl_up_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) >= o) v += t;
  }
  return v;
}

// block-wide exclusive scan of one value per thread; returns exclusive prefix, total in *total
GMSM_D uint32_t block_excl_scan(uint32_t v, uint32_t* smem /* >= 33 */, uint32_t* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t inc = warp_incl_scan(v);
  if (lane == 31) smem[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    uint32_t w = (lane < (int)(blockDim.x >> 5)) ? smem[lane] : 0;
    uint32_t wi = warp_incl_scan(w);
    smem[lane] = wi - w;
    if (lane == 31) smem[32] = wi;
  }
  __syncthreads();
  uint32_t res = smem[warp] + inc - v;
  *total = smem[32];
  __syncthreads();
  return res;
}

static __global__ void k_scan_block_sums(const uint32_t* __restrict__ in, uint32_t n, uint32_t* __restrict__ block_sums) {
  __shared__ uint32_t smem[33];
  uint32_t base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
  uint32_t s = 0;
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; k++)
    if (base + k < n) s += in[base + k];
  uint32_t tot;
  block_excl_scan(s, smem, &tot);
  if (threadIdx.x == 0) block_sums[blockIdx.x] = tot;
}

// single block: exclusive scan in place over nblocks values, grand total -> *grand
static __global__ void k_scan_top(uint32_t* __restrict__ block_sums, uint32_t nblocks, uint32_t* __restrict__ grand) {
  __shared__ uint32_t smem[33];
  uint32_t running = 0;
  for (uint32_t base = 0; base < nblocks; base += blockDim.x) {
    uint32_t i = base + threadIdx.x;
    uint32_t v = (i < nblocks) ? block_sums[i] : 0;
    uint32_t tot;
    uint32_t ex = block_excl_scan(v, smem, &tot);
    if (i < nblocks) block_sums[i] = running + ex;
    running += tot;
  }
  if (threadIdx.x == 0) *grand = running;
}

template <bool ENDS>
GMSM_D void scan_final_tile(const uint32_t* in, uint32_t n, const uint32_t* __restrict__ block_sums, uint32_t* __restrict__ out,
                            uint32_t* ends) {
  __shared__ uint32_t smem[33];
  uint32_t base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
  uint32_t v[SCAN_ITEMS];
  uint32_t s = 0;
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; k++) {
    v[k] = (base + k < n) ? in[base + k] : 0;
    s += v[k];
  }
  uint32_t tot;
  uint32_t ex = block_excl_scan(s, smem, &tot) + block_sums[blockIdx.x];
#pragma unroll
  for (int k = 0; k < SCAN_ITEMS; k++) {
    if (base + k < n) {
      out[base + k] = ex;
      if constexpr (ENDS) ends[base + k] = ex + v[k];
    }
    ex += v[k];
  }
}
static __global__ void k_scan_final(const uint32_t* __restrict__ in, uint32_t n, const uint32_t* __restrict__ block_sums,
                             uint32_t* __restrict__ out) {
  scan_final_tile<false>(in, n, block_sums, out, nullptr);
}
// the same over the bucket histogram, which it also turns in place into bucket END pointers (offset + count): the scatter's
// returning atomic on a counter then yields the entry's position directly (k_scatter_window)
static __global__ void k_scan_final_ends(uint32_t* counts, uint32_t n, const uint32_t* __restrict__ block_sums,
                                         uint32_t* __restrict__ out) {
  scan_final_tile<true>(counts, n, block_sums, out, counts);
}

// first index in offsets[0..len) with offsets[idx] > key  (offsets non-decreasing)
GMSM_D uint32_t upper_bound_u32(const uint32_t* __restrict__ a, uint32_t len, uint32_t key) {
  uint32_t lo = 0, hi = len;
  while (lo < hi) {
    uint32_t mid = lo + ((hi - lo) >> 1);
    if (a[mid] <= key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// ------------------------------------------------------------------------------------------
// K2: bucket accumulation as a load-balanced segmented reduction.
// The bucket-ordered entry list (length M = offsets[nb_total]) is cut into chunks of K entries, one
// thread per chunk, so the work per thread is constant whatever the digit distribution (the
// reference needs chunkStat weights and a two-goroutine split for skewed windows, multiexp.go:185-203).
// A thread keeps the running bucket sum in registers (extended Jacobian, mixed adds with the
// reference's exact special cases) and flushes it at each bucket boundary:
//   * bucket begins inside the chunk  -> the thread owns it: buckets[b] = sum
//   * bucket began in an earlier chunk -> the partial goes to carries[t] (joined by k_carry_level)
// ------------------------------------------------------------------------------------------
// ---- bulk-asynchronous (TMA engine) staging of the NEXT base point -------------------------------------------------
// GMSM_ACC_TMA = 1: the software pipeline of k_accumulate keeps the prefetched point in shared memory instead of in
// registers.  Each thread owns one slot (one affine point) and one mbarrier; at the top of an iteration it posts
//   mbarrier.arrive.expect_tx + cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes   (SASS: UBLKCP)
// for the point of the following entry -- a 64..192-byte 1-D bulk copy executed by the TMA unit, no registers held while it
// is in flight -- runs the mixed addition on the current point, then waits on the barrier's phase and reads the slot
// (LDS.128).  This frees the 16 (G1, 8 limbs) .. 48 (bls12-381 G2) registers of `pt_next`.
#ifndef GMSM_ACC_TMA
#define GMSM_ACC_TMA 0
#endif
// GMSM_ACC_NOPREFETCH = 1 (experimental): no software pipeline at all -- each iteration loads its own point and relies on the
// other resident warps to cover the gather latency; frees the registers of the prefetched point without extra instructions.
#ifndef GMSM_ACC_NOPREFETCH
#define GMSM_ACC_NOPREFETCH 0
#endif
#if GMSM_ACC_TMA && defined(__CUDA_ARCH__)
GMSM_D uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
GMSM_D void tma_bar_init(uint32_t bar) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
GMSM_D void tma_load_1d(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // earlier generic reads of the slot are ordered before the async write
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(__cvta_generic_to_global(src)), "r"(bytes), "r"(bar) : "memory");
}
GMSM_D void tma_bar_wait(uint32_t bar, uint32_t phase) {
  uint32_t ok;
  do {
    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                 : "=r"(ok) : "r"(bar), "r"(phase) : "memory");
  } while (!ok);
}
#endif

#ifndef GMSM_ACC_MINBLOCKS_BIG
#define GMSM_ACC_MINBLOCKS_BIG 1
#endif
#ifndef GMSM_ACC_MINBLOCKS_SMALL
#define GMSM_ACC_MINBLOCKS_SMALL 4
#endif
#ifndef GMSM_ACC_PREFETCH_BEND
#define GMSM_ACC_PREFETCH_BEND 1
#endif
template <class G>
__global__ void __launch_bounds__(128, (sizeof(typename G::F) <= 32) ? GMSM_ACC_MINBLOCKS_SMALL : GMSM_ACC_MINBLOCKS_BIG)
k_accumulate(const Affine<typename G::F>* __restrict__ points, const uint32_t* __restrict__ entries,
             const uint32_t* __restrict__ offsets, uint32_t nb_total, uint32_t K, uint32_t nchunks,
             XYZZ<typename G::F>* __restrict__ buckets, XYZZ<typename G::F>* __restrict__ carries,
             uint32_t* __restrict__ carry_ids, int part, uint32_t split_bucket) {
  using F = typename G::F;
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nchunks) return;
  const uint32_t M = offsets[nb_total];
  const uint64_t start64 = (uint64_t)t * K;
  // The launch can be split in two parts so that the scatter of the later windows overlaps the first
  // part: part 1 takes the chunks that end inside the first `split_bucket` buckets (whose entries are
  // already scattered), part 2 the rest (after the whole scatter); part 0 = everything.
  if (part != 0) {
    const uint32_t split = offsets[split_bucket];
    const bool early = (start64 + K <= split);
    if ((part == 1) != early) return;
  }
  if (start64 >= M) {
    carry_ids[t] = ID_NONE;
    return;
  }
  const uint32_t start = (uint32_t)start64;
  const uint32_t end = (M - start < K) ? M : start + K;

  uint32_t b = upper_bound_u32(offsets, nb_total + 1, start) - 1u;
  uint32_t bend = offsets[b + 1];
  // end of the NEXT bucket, fetched one bucket ahead so that a boundary costs no dependent load (the warp is
  // divergent there: every lane waits for it).  offsets[] is padded past nb_total; the pad is never consumed.
#if GMSM_ACC_PREFETCH_BEND
  uint32_t bend2 = offsets[b + 2];
#endif
  bool owner = (offsets[b] == start);
  uint32_t my_carry = ID_NONE;
  XYZZ<F> acc = XYZZ<F>::inf();

  uint32_t e = entries[start];
  Affine<F> pt = load_vec_ro(points + (e >> 1));
#if GMSM_ACC_TMA && defined(__CUDA_ARCH__)
  __shared__ __align__(128) Affine<F> tma_slot[128];
  __shared__ __align__(8) unsigned long long tma_bar[128];
  const uint32_t slot_a = smem_u32(&tma_slot[threadIdx.x]), bar_a = smem_u32(&tma_bar[threadIdx.x]);
  tma_bar_init(bar_a);
  uint32_t tma_phase = 0;
#endif
  for (uint32_t pos = start; pos < end; pos++) {
    // software pipeline: issue the next entry / point loads before the arithmetic of this one
    uint32_t e_next = 0;
    const bool has_next = (pos + 1 < end);
#if GMSM_ACC_TMA && defined(__CUDA_ARCH__)
    if (has_next) {
      e_next = entries[pos + 1];
      tma_load_1d(slot_a, points + (e_next >> 1), (uint32_t)sizeof(Affine<F>), bar_a);
    }
#elif GMSM_ACC_NOPREFETCH
    if (has_next) e_next = entries[pos + 1];
#else
    Affine<F> pt_next;
    if (has_next) {
      e_next = entries[pos + 1];
      pt_next = load_vec_ro(points + (e_next >> 1));
    }
#endif
    if (pos == bend) {
      // bucket boundary: flush, move to the bucket that contains `pos`
      if (owner) {
        store_vec(buckets + b, acc);
      } else {
        store_vec(carries + t, acc);
        my_carry = b;
      }
      b++;
#if GMSM_ACC_PREFETCH_BEND
      bend = bend2;
      if (bend == pos) {   // skip empty buckets
        b = upper_bound_u32(offsets, nb_total + 1, pos) - 1u;
        bend = offsets[b + 1];
      }
      bend2 = offsets[b + 2];
#else
      if (offsets[b + 1] == pos) b = upper_bound_u32(offsets, nb_total + 1, pos) - 1u;  // skip empty buckets
      bend = offsets[b + 1];
#endif
      owner = true;
      acc = XYZZ<F>::inf();
    }
    xyzz_add_mixed(acc, pt, (e & 1u) != 0);
    if (has_next) {
      e = e_next;
#if GMSM_ACC_TMA && defined(__CUDA_ARCH__)
      tma_bar_wait(bar_a, tma_phase);
      tma_phase ^= 1u;
      pt = load_vec(&tma_slot[threadIdx.x]);
#elif GMSM_ACC_NOPREFETCH
      pt = load_vec_ro(points + (e >> 1));
#else
      pt = pt_next;
#endif
    }
  }
  if (owner) {
    store_vec(buckets + b, acc);
  } else {
    store_vec(carries + t, acc);
    my_carry = b;
  }
  carry_ids[t] = my_carry;
}

// K2b: one level of the carry join.  Input: (id, partial) items ordered by id, ID_NONE = empty slot;
// the items of one bucket are contiguous.  A thread walks K2 consecutive items, sums runs of equal id;
// a run that starts in this thread's range is owned (bucket[id] += sum, exclusive within a level);
// a run continued from the previous range is forwarded to the next level.
template <class G, bool Q>
__global__ void __launch_bounds__(128)
k_carry_level(const XYZZ<typename G::F>* __restrict__ in_pts, const uint32_t* __restrict__ in_ids, uint32_t n_in,
              uint32_t K2, XYZZ<typename G::F>* __restrict__ buckets, XYZZ<typename G::F>* __restrict__ out_pts,
              uint32_t* __restrict__ out_ids) {
  using F = typename G::F;
  const uint32_t gid = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t t = Q ? gid >> 2 : gid;
  const Quad qd = quad_of_thread();
  const bool writer = !Q || qd.ql == 0;
  const uint32_t n_out = (n_in + K2 - 1) / K2;
  if (t >= n_out) return;
  const uint32_t start = t * K2;
  const uint32_t end = (n_in - start < K2) ? n_in : start + K2;
  uint32_t cur = ID_NONE, out_id = ID_NONE;
  bool owner = true;
  XYZZ<F> acc = XYZZ<F>::inf();
  for (uint32_t i = start; i <= end; i++) {
    uint32_t id = (i < end) ? in_ids[i] : ID_NONE;
    if (id == cur && id != ID_NONE) {
      XYZZ<F> q = load_vec(in_pts + i);
      tail_add<Q>(qd, acc, q);
      continue;
    }
    if (cur != ID_NONE) {  // run ended: flush
      if (owner) {
        XYZZ<F> old = load_vec(buckets + cur);
        if constexpr (Q) __syncwarp(qd.mask);   // every lane of the quad has read the bucket before lane 0 rewrites it
        tail_add<Q>(qd, old, acc);
        if (writer) store_vec(buckets + cur, old);
      } else {
        if (writer) store_vec(out_pts + t, acc);
        out_id = cur;
      }
      cur = ID_NONE;
    }
    if (id != ID_NONE) {
      cur = id;
      acc = load_vec(in_pts + i);
      owner = !(i == start && start > 0 && in_ids[start - 1] == id);
    }
  }
  if (writer) out_ids[t] = out_id;
}

// dst[b] += src[b] for every bucket (joins the buckets of a pipelined batch into the running ones)
template <class G>
__global__ void __launch_bounds__(128)
k_merge_buckets(XYZZ<typename G::F>* __restrict__ dst, const XYZZ<typename G::F>* __restrict__ src, uint32_t nb) {
  using F = typename G::F;
  const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= nb) return;
  XYZZ<F> q = load_vec(src + b);
  if (q.is_inf()) return;
  XYZZ<F> p = load_vec(dst + b);
  xyzz_add_cold(p, q);
  store_vec(dst + b, p);
}

// ------------------------------------------------------------------------------------------
// K3: bucket reduction.  Window total = sum_k (k+1) * B[k]  (multiexp_jacobian.go:44-52, a serial
// running sum in the reference).  Parallel form: segment s covers buckets [sL, sL+L):
//   sum_{k in seg} (k+1) B[k] = tot_s + (sL) * run_s,   run_s = sum B[k], tot_s = local running-sum
// each thread also applies the small scalar sL by double-and-add, so segments are independent and the
// window total is a plain sum of the segment results (k_sum_groups).
// ------------------------------------------------------------------------------------------
template <class G, bool Q>
__global__ void __launch_bounds__(128)
k_bucket_segments(const XYZZ<typename G::F>* __restrict__ buckets, int nwin, uint32_t nb, uint32_t nb_last,
                  uint32_t L, uint32_t S, XYZZ<typename G::F>* __restrict__ seg_out) {
  using F = typename G::F;
  const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t gid = Q ? tid >> 2 : tid;
  const Quad qd = quad_of_thread();
  const bool writer = !Q || qd.ql == 0;
  if (gid >= (uint32_t)nwin * S) return;
  const uint32_t j = gid / S, s = gid % S;
  const uint32_t nbj = (j == (uint32_t)nwin - 1) ? nb_last : nb;
  const uint32_t lo = s * L;
  if (lo >= nbj) {
    if (writer) store_vec(seg_out + gid, XYZZ<F>::inf());
    return;
  }
  const uint32_t hi = (nbj - lo < L) ? nbj : lo + L;
  const XYZZ<F>* base = buckets + (size_t)j * nb;
  XYZZ<F> run = XYZZ<F>::inf(), tot = XYZZ<F>::inf();
  for (uint32_t k = hi; k-- > lo;) {
    XYZZ<F> bk = load_vec(base + k);
    tail_add<Q>(qd, run, bk);
    tail_add<Q>(qd, tot, run);
  }
  if (lo > 0 && !run.is_inf()) {
    XYZZ<F> acc = XYZZ<F>::inf();
    for (int bit = 31 - __clz(lo); bit >= 0; bit--) {
      acc = tail_double<Q>(qd, acc);
      if ((lo >> bit) & 1u) tail_add<Q>(qd, acc, run);
    }
    tail_add<Q>(qd, tot, acc);
  }
  if (writer) store_vec(seg_out + gid, tot);
}

// out[j][g] = sum_{i in [gR, gR+R)} in[j][i]
template <class G, bool Q>
__global__ void __launch_bounds__(128)
k_sum_groups(const XYZZ<typename G::F>* __restrict__ in, uint32_t in_per_win, uint32_t R, uint32_t out_per_win,
             int nwin, XYZZ<typename G::F>* __restrict__ out) {
  using F = typename G::F;
  const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t gid = Q ? tid >> 2 : tid;
  const Quad qd = quad_of_thread();
  if (gid >= (uint32_t)nwin * out_per_win) return;
  const uint32_t j = gid / out_per_win, g = gid % out_per_win;
  uint32_t lo = g * R, hi = lo + R;
  if (hi > in_per_win) hi = in_per_win;
  XYZZ<F> acc = XYZZ<F>::inf();
  for (uint32_t i = lo; i < hi; i++) {
    XYZZ<F> q = load_vec(in + (size_t)j * in_per_win + i);
    tail_add<Q>(qd, acc, q);
  }
  if (!Q || qd.ql == 0) store_vec(out + (size_t)j * out_per_win + g, acc);
}

// out[j][g] = sum of in[j][128 g .. 128 g + 128): a block-level binary tree (each thread adds two inputs, then six
// shared-memory levels), so a launch shortens every window's list 128-fold along a chain of only 7 additions -- the
// group sums above walk 16 additions per 16-fold level (48 for 2048 segment results, against 14 here).
static constexpr int TREE_THREADS = 64;
template <class G>
__global__ void __launch_bounds__(TREE_THREADS)
k_sum_tree(const XYZZ<typename G::F>* __restrict__ in, uint32_t in_per_win, uint32_t out_per_win, XYZZ<typename G::F>* __restrict__ out) {
  using F = typename G::F;
  __shared__ XYZZ<F> sm[TREE_THREADS];
  const uint32_t j = blockIdx.y, g = blockIdx.x, t = threadIdx.x;
  const uint32_t base = g * 2u * TREE_THREADS;
  const XYZZ<F>* src = in + (size_t)j * in_per_win;
  XYZZ<F> acc = XYZZ<F>::inf();
  if (base + t < in_per_win) acc = load_vec(src + base + t);
  if (base + t + TREE_THREADS < in_per_win) {
    XYZZ<F> q = load_vec(src + base + t + TREE_THREADS);
    xyzz_add_cold(acc, q);
  }
  for (uint32_t s = TREE_THREADS / 2; s >= 1; s >>= 1) {
    store_vec(&sm[t], acc);
    __syncthreads();
    if (t < s) {
      XYZZ<F> q = load_vec(&sm[t + s]);
      xyzz_add_cold(acc, q);
    }
    __syncthreads();
  }
  if (t == 0) store_vec(out + (size_t)j * out_per_win + g, acc);
}

// ------------------------------------------------------------------------------------------
// K4: finalize (one block of FIN_THREADS).  partials[r][j], r < nranks, j < nwin.  Lanes sum over the ranks, window-parallel;
// then ONE thread runs the Horner chain -- c * (W - 1) dependent doublings, the longest serial chain of an MSM.  Q = true is
// the lane-parallel form (quad.cuh: three product steps per doubling instead of seven); it is SLOWER for the 8- and 12-limb
// groups (a lone warp is bound by the ~5 cycles per dependent instruction, and the operand
// selects and shuffles of a lane-parallel step cost as many instructions as they save) and is kept behind GMSM_QUAD=1.
// ------------------------------------------------------------------------------------------
static constexpr int FIN_THREADS = 64;
template <class F>
__device__ __noinline__ Jac<F> jac_double_quad_cold(Quad q, const Jac<F>& p) {
  return jac_double_quad(q, p);
}
template <class F>
__device__ __noinline__ Jac<F> jac_double_cold1(const Jac<F>& p) {
  return jac_double(p);
}
template <class G, bool Q>
__global__ void __launch_bounds__(FIN_THREADS)
k_finalize(const XYZZ<typename G::F>* __restrict__ partials, int nranks, int nwin, int c,
           XYZZ<typename G::F>* __restrict__ scratch /* nwin */, Jac<typename G::F>* __restrict__ out) {
  using F = typename G::F;
  const Quad qd = quad_of_thread();
  // sum over the ranks, window-parallel (one lane -- or one quad -- per window)
  const int stride = Q ? (int)(blockDim.x >> 2) : (int)blockDim.x;
  for (int j = Q ? (int)(threadIdx.x >> 2) : (int)threadIdx.x; j < nwin; j += stride) {
    XYZZ<F> acc = load_vec(partials + j);
    for (int r = 1; r < nranks; r++) {
      XYZZ<F> q = load_vec(partials + (size_t)r * nwin + j);
      tail_add<Q>(qd, acc, q);
    }
    if (!Q || qd.ql == 0) store_vec(scratch + j, acc);
  }
  __syncthreads();
  if (threadIdx.x >= (Q ? 4u : 1u)) return;
  // Horner over the windows, high -> low: acc = 2^c * acc + T_j.  The c doublings run in Jacobian
  // coordinates (2M + 5S each instead of 6M + 3S); the addition of T_j in extended Jacobian.
  XYZZ<F> acc = load_vec(scratch + (nwin - 1));
  for (int j = nwin - 2; j >= 0; j--) {
    if constexpr (Q) {
      Jac<F> dj = xyzz_to_jac_quad(qd, acc);
      for (int l = 0; l < c; l++) dj = jac_double_quad_cold(qd, dj);
      acc = jac_to_xyzz_quad(qd, dj);
    } else {
      Jac<F> dj = xyzz_to_jac(acc);
      for (int l = 0; l < c; l++) dj = jac_double_cold1(dj);
      acc = jac_to_xyzz(dj);
    }
    XYZZ<F> q = load_vec(scratch + j);
    tail_add<Q>(qd, acc, q);
  }
  Jac<F> jac = xyzz_to_jac(acc);
  Affine<F> a = jac_to_affine(jac);
  Jac<F> o;
  if (jac.z.is_zero()) {
    o = Jac<F>{F::zero(), F::zero(), F::zero()};
  } else {
    o = Jac<F>{a.x, a.y, F::one()};
  }
  if (!Q || qd.ql == 0) store_vec(out, o);
}

// ------------------------------------------------------------------------------------------
// base generator: out[t*m + i] = [start + t*m + i] * base  (affine), one thread per m consecutive
// multiples: double-and-add to the first one, mixed adds for the rest, one inversion per thread
// (Montgomery trick over ZZZ; 1/ZZ = ZZ^2 / ZZZ^2).
// ------------------------------------------------------------------------------------------
static constexpr int GEN_M = 16;
template <class G>
__global__ void __launch_bounds__(128)
k_generate_multiples(const Affine<typename G::F>* __restrict__ base_p, uint64_t start, uint64_t n,
                     Affine<typename G::F>* __restrict__ out) {
  using F = typename G::F;
  const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint64_t first = t * GEN_M;
  if (first >= n) return;
  const Affine<F> base = load_vec_ro(base_p);
  uint64_t k = start + first;
  XYZZ<F> acc = XYZZ<F>::inf();
  for (int bit = 63; bit >= 0; bit--) {
    acc = xyzz_double_cold(acc);
    if ((k >> bit) & 1ull) xyzz_add_mixed(acc, base, false);
  }
  XYZZ<F> pts[GEN_M];
  F pref[GEN_M];
  F prod = F::one();
  const int cnt = (n - first < (uint64_t)GEN_M) ? (int)(n - first) : GEN_M;
  for (int i = 0; i < cnt; i++) {
    pts[i] = acc;
    pref[i] = prod;  // product of ZZZ of points before i (infinity contributes 1)
    if (!acc.is_inf()) prod = f_mul(prod, acc.zzz);
    xyzz_add_mixed(acc, base, false);
  }
  F inv = f_inv(prod);
  for (int i = cnt - 1; i >= 0; i--) {
    Affine<F> a = Affine<F>::inf();
    if (!pts[i].is_inf()) {
      F i3 = f_mul(inv, pref[i]);        // 1/ZZZ_i
      inv = f_mul(inv, pts[i].zzz);
      F i2 = f_mul(f_sqr(pts[i].zz), f_sqr(i3));  // 1/ZZ_i
      a.x = f_mul(pts[i].x, i2);
      a.y = f_mul(pts[i].y, i3);
    }
    store_vec(out + first + i, a);
  }
}

// ------------------------------------------------------------------------------------------
// Window tables for resident bases: out[i] = 2^c * in[i] (affine).  Row j of a table holds 2^(c*j) * P_i, so
//   sum_i s_i P_i = sum_j sum_i d_ij * (2^(c*j) P_i)
// becomes ONE bucket problem over n*W table points with the digits of partitionScalars (multiexp.go:709-803)
// -- no per-window bucket sets, no Horner (msmReduceChunk, multiexp.go:302-315, degenerates to one window),
// which lets c grow to ~22 (W = 12 instead of 15 -> 20 % fewer bucket additions).  The reference has no
// counterpart: its bases are re-read per call; this is the "static SRS" flow of kzg.Commit (kzg/kzg.go:159-176).
// One thread takes TAB_M consecutive points (table_level_batch, curve.cuh): c Jacobian doublings each (dbl-2009-l),
// one shared inversion (Montgomery's trick over the Z's), affine normal forms out.  Infinity stays (0, 0).
// ------------------------------------------------------------------------------------------
template <class F>
__device__ __noinline__ Jac<F> jac_double_cold(const Jac<F>& p) {
  return jac_double(p);
}
template <class G>
__global__ void __launch_bounds__(128)
k_table_level(const Affine<typename G::F>* __restrict__ in, uint32_t n, int c, Affine<typename G::F>* __restrict__ out) {
  using F = typename G::F;
  const uint64_t first = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) * TAB_M;
  if (first >= n) return;
  const int cnt = (n - first < (uint64_t)TAB_M) ? (int)(n - first) : TAB_M;
  table_level_batch<F>(
      cnt, c, [&](int i) { return load_vec_ro(in + first + i); }, [&](int i, const Affine<F>& a) { store_vec(out + first + i, a); },
      [](const Jac<F>& j) { return jac_double_cold(j); });
}

// ------------------------------------------------------------------------------------------
// N1: fixed-base batch scalar multiplication (BatchScalarMultiplicationG1, ecc/bn254/g1.go:1039-1118;
// G2 g2.go:1001+).  table[k] = [k+1]*base in affine (k < 2^(max(c,lastC)-1)); one thread per scalar:
// signed digits as in partitionScalars, Horner from the top window (c doublings + one mixed add of
// +-table[|d|-1] per window), then the affine normal form (BatchJacobianToAffineG1's result, :988-1034;
// here each thread inverts its own ZZZ: x = X*ZZ^2/ZZZ^2, y = Y/ZZZ).
// ------------------------------------------------------------------------------------------
static constexpr int BSM_MAX_WINDOWS = 64;   // c >= 4
template <class G>
__global__ void __launch_bounds__(128)
k_batch_scalar_mul(const Affine<typename G::F>* __restrict__ table, const typename G::Fr* __restrict__ scalars, uint32_t n,
                   int c, int nwin, Affine<typename G::F>* __restrict__ out) {
  using F = typename G::F;
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t codes[BSM_MAX_WINDOWS];
  typename G::Fr s = load_vec_ro(scalars + i);
  for_each_digit<G>(s, c, nwin, [&](int j, uint32_t code) { codes[j] = code; });
  XYZZ<F> p = XYZZ<F>::inf();
  for (int j = nwin - 1; j >= 0; j--) {
    if (j != nwin - 1)
      for (int l = 0; l < c; l++) p = xyzz_double_cold(p);
    const uint32_t code = codes[j];
    if (code == 0) continue;
    Affine<F> t = load_vec_ro(table + code_bucket(code));
    xyzz_add_mixed(p, t, (code & 1u) != 0);
  }
  Affine<F> a = Affine<F>::inf();
  if (!p.is_inf()) {
    F i3 = f_inv(p.zzz);
    F i2 = f_mul(f_sqr(p.zz), f_sqr(i3));
    a.x = f_mul(p.x, i2);
    a.y = f_mul(p.y, i3);
  }
  store_vec(out + i, a);
}

// test hook kernel (element-wise ops are defined in testops.cuh, shared with the host formula check)
#if defined(__CUDACC__)
template <class G>
__global__ void k_test_op(int op, const uint32_t* a, const uint32_t* b, uint32_t* o, uint32_t n) {
  int wa, wb, wo;
  test_op_sizes<G>(op, &wa, &wb, &wo);
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    test_op_one<G>(op, a + (size_t)i * wa, b + (size_t)i * wb, o + (size_t)i * wo);
}
#endif

}  // namespace gmsm
