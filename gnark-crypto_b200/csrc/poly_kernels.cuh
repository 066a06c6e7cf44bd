// Device side of the Fr polynomial steps of kzg.Open, kzg.BatchOpenSinglePoint and the SHPLONK / FFLONK batch openings:
// evaluation, division by (X - a) and the strided linear combination, of which the gamma-fold is the stride-1 case.  Reference:
// eval (ecc/bn254/kzg/kzg.go:55-63), dividePolyByXminusA (:567-582), the fold of BatchOpenSinglePoint (:302-319); the kzg
// packages of the other pairing curves are the same generated code.  In a header of their own, like
// fft_kernels.cuh, so that the CPU kernel emulation of tests/emu/ compiles and runs them too (tests/test_emu_poly_cpu.py);
// fft.cu includes this file and holds the entry points.  The launch schedules below are shared by both.
//
// One suffix recurrence gives both outputs of an opening: b[n-1] = f[n-1], b[i] = f[i] + a b[i+1]; then b[0] = f(a) (the
// ClaimedValue) and h[i] = b[i+1] (i < n-1) is dividePolyByXminusA(f, f(a), a) -- the reference's f[0] - f(a) changes only b[0].
// Parallel form, a linear-recurrence scan with a constant multiplier:
//   * a block owns a tile of T = B * L coefficients: B threads, each a chunk of L consecutive ones (B, L powers of two);
//     the tile is staged through shared memory so that global accesses stay coalesced;
//   * k_poly_heads writes each tile's head: its b at the tile's first index with carry-in 0;
//   * tile t's true carry-in is b at the next tile's first index, and these values obey the same recurrence over the heads with
//     multiplier a^T.  So k_poly_heads runs level by level on the heads (multipliers a^T, a^(T^2), ...) until a level fits in
//     one tile; then k_poly_write runs top-down: each tile recomputes its b from its true carry-in, read from the level above,
//     and stores them -- in place on the carry levels, shifted by one into h on the polynomial itself.
//   * evaluation only: one more k_poly_heads on the top level leaves f(a) as the head of its single tile.
// Inside a block the chunk values are joined by a work-efficient tree over the B threads (up-sweep, then down-sweep for the
// carries).  Field arithmetic is exact and every fp_* result is fully reduced, so any grouping gives the reference's limbs.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <vector>

#include "field.cuh"
#include "vec_io.cuh"

using namespace gmsm;

namespace {

constexpr int POLY_MAX_LOG_B = 10;   // at most 1024 threads per block
constexpr int POLY_FOLD_BATCH = 8;   // polynomials folded per k_poly_fold launch

// Tile shape per element size: log2 of the chunk length L and of the block size B.  Shared memory (poly_smem_bytes):
// 40 KB for the 32-byte fields (B = 256, L = 4), 45 KB for bw6-633 (B = 128, L = 8), 30 KB for bw6-761 (B = 128, L = 4) --
// all within the default 48 KB dynamic shared-memory limit, so no cudaFuncSetAttribute opt-in is needed.
template <class P>
constexpr int poly_log_l() { return sizeof(Fp<P>) == 40 ? 3 : 2; }
template <class P>
constexpr int poly_log_b() { return sizeof(Fp<P>) == 32 ? 8 : 7; }

// multipliers of one level: a = the level's A (Horner step inside a chunk); m[k] = A^(L 2^k) joins two neighbouring segments
// of 2^k chunks.  Computed on the host, passed by value.
template <class P>
struct PolyMults {
  Fp<P> a;
  Fp<P> m[POLY_MAX_LOG_B];
};

// Shared memory of a tile: coefficient j at slot j + j / L, so every chunk is followed by one pad slot.  The pad slot of chunk t
// holds thread t's tree value, and the L + 1 stride between chunks spreads the chunk walks over the banks.  The tree
// multipliers m[] follow the T + B slots.
template <class P>
constexpr size_t poly_smem_bytes(int log_l, int log_b) {
  return ((size_t(1) << (log_l + log_b)) + (size_t(1) << log_b) + POLY_MAX_LOG_B) * sizeof(Fp<P>);
}

// Stages tile blockIdx.x of x (m elements, zero past the end) and the multipliers, runs the thread's Horner with carry-in 0 and
// the up-sweep.  Afterwards the pad slot of thread t with t = 0 mod 2^k holds the value of the segment of 2^k chunks that
// starts at chunk t; thread 0's holds the tile head.  Returns log2(B).
template <class P>
GMSM_D int poly_tile_up(Fp<P>* s, const Fp<P>* x, uint64_t m, const PolyMults<P>& mu, int log_l) {
  const uint32_t B = blockDim.x, tid = threadIdx.x, L = 1u << log_l, T = B << log_l;
  const uint64_t base = (uint64_t)blockIdx.x * T;
  for (uint32_t j = tid; j < T; j += B) {
    const uint64_t i = base + j;
    store_vec(s + j + (j >> log_l), i < m ? load_vec(x + i) : Fp<P>::zero());
  }
  Fp<P>* sm = s + T + B;
#pragma unroll
  for (int k = 0; k < POLY_MAX_LOG_B; k++)   // unrolled: static indices keep mu in the parameter bank
    if (tid == (uint32_t)k) store_vec(sm + k, mu.m[k]);
  __syncthreads();
  Fp<P>* c = s + tid * (L + 1);
  Fp<P> acc = load_vec(c + L - 1);
  for (int j = (int)L - 2; j >= 0; j--) acc = fp_add(fp_mul(acc, mu.a), load_vec(c + j));
  store_vec(c + L, acc);
  __syncthreads();
  int k = 0;
  for (uint32_t d = 1; d < B; d <<= 1, k++) {
    if ((tid & (2 * d - 1)) == 0)
      store_vec(c + L, fp_add(load_vec(c + L), fp_mul(load_vec(sm + k), load_vec(s + (tid + d) * (L + 1) + L))));
    __syncthreads();
  }
  return k;
}

// chunk-head pass: heads[tile] = b at the tile's first index with carry-in 0.  blockDim.x = B, dynamic shared memory
// poly_smem_bytes, one block per tile.
template <class P>
__global__ void k_poly_heads(const Fp<P>* x, uint64_t m, PolyMults<P> mu, int log_l, Fp<P>* heads) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Fp<P>* s = reinterpret_cast<Fp<P>*>(smem_raw);
  poly_tile_up(s, x, m, mu, log_l);
  if (threadIdx.x == 0) store_vec(heads + blockIdx.x, load_vec(s + (1u << log_l)));
}

// write pass: tile t's carry-in is carry[t + 1] (b at the next tile's first index; 0 for the last tile or carry == NULL).
// Stores out[i - shift] = b[i] for shift <= i < m (out == NULL: nothing; out may equal x: in place) and, from block 0,
// *fa = b[0] (fa == NULL: nothing).  Launch shape as k_poly_heads.
template <class P>
__global__ void k_poly_write(const Fp<P>* x, uint64_t m, PolyMults<P> mu, int log_l, const Fp<P>* carry, Fp<P>* out, int shift,
                             Fp<P>* fa) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Fp<P>* s = reinterpret_cast<Fp<P>*>(smem_raw);
  const uint32_t B = blockDim.x, tid = threadIdx.x, L = 1u << log_l, T = B << log_l;
  const uint64_t base = (uint64_t)blockIdx.x * T, tiles = ((m - 1) >> (log_l + __ffs((int)B) - 1)) + 1;
  const Fp<P> cin = (carry && blockIdx.x + 1 < tiles) ? load_vec(carry + blockIdx.x + 1) : Fp<P>::zero();
  int k = poly_tile_up(s, x, m, mu, log_l);
  const Fp<P>* sm = s + T + B;
  Fp<P>* c = s + tid * (L + 1);
  // down-sweep: a segment's slot takes the b just past its end (the root: the tile's carry-in); its right half inherits it,
  // its left half gets (right half's value) + m[k] * (that b)
  if (tid == 0) store_vec(c + L, cin);
  __syncthreads();
  for (uint32_t d = B >> 1; d >= 1; d >>= 1) {
    k--;
    if ((tid & (2 * d - 1)) == 0) {
      Fp<P>* r = s + (tid + d) * (L + 1) + L;
      const Fp<P> e = load_vec(c + L), y = load_vec(r);
      store_vec(r, e);
      store_vec(c + L, fp_add(y, fp_mul(load_vec(sm + k), e)));
    }
    __syncthreads();
  }
  Fp<P> acc = load_vec(c + L);   // b just past this thread's chunk
  for (int j = (int)L - 1; j >= 0; j--) {
    acc = fp_add(fp_mul(acc, mu.a), load_vec(c + j));
    store_vec(c + j, acc);
  }
  __syncthreads();
  if (out) {
    for (uint32_t j = tid; j < T; j += B) {
      const uint64_t i = base + j;
      if (i >= (uint64_t)shift && i < m) store_vec(out + (i - shift), load_vec(s + j + (j >> log_l)));
    }
  }
  if (fa && blockIdx.x == 0 && tid == 0) store_vec(fa, load_vec(s));
}

// one batch of the linear combination: out[m stride[i] + offset[i]] (+)= g[i] p[i][m] for m < len[i].  stride and offset follow
// the fields of the stride-1 fold so that its kernel reads its parameters where it always did.
template <class P>
struct PolyFoldBatch {
  const Fp<P>* p[POLY_FOLD_BATCH];
  uint64_t len[POLY_FOLD_BATCH];
  Fp<P> g[POLY_FOLD_BATCH];
  int count;
  uint64_t stride[POLY_FOLD_BATCH];
  uint64_t offset[POLY_FOLD_BATCH];
};

// linear combination: out[j] = sum_i g[i] p[i][(j - offset[i]) / stride[i]] for j < out_len, over the inputs whose stride divides
// j - offset[i] (j >= offset[i]) with a quotient below len[i]; every input read once, out written once per batch of
// POLY_FOLD_BATCH inputs (accumulate != 0: add to out).  Grid-stride, no barrier.  STRIDED = false: every stride is 1 and every
// offset 0 (the gamma-fold), and the index arithmetic reduces to j < len[i].
template <class P, bool STRIDED = false>
__global__ void k_poly_fold(Fp<P>* __restrict__ out, uint64_t out_len, PolyFoldBatch<P> b, int accumulate) {
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < out_len; j += (uint64_t)gridDim.x * blockDim.x) {
    Fp<P> acc = accumulate ? load_vec(out + j) : Fp<P>::zero();
#pragma unroll
    for (int i = 0; i < POLY_FOLD_BATCH; i++) {
      if (i >= b.count) continue;
      if constexpr (STRIDED) {
        if (j < b.offset[i]) continue;
        const uint64_t d = j - b.offset[i], m = d / b.stride[i];
        if (m * b.stride[i] == d && m < b.len[i]) acc = fp_add(acc, fp_mul(load_vec(b.p[i] + m), b.g[i]));
      } else {
        if (j < b.len[i]) acc = fp_add(acc, fp_mul(load_vec(b.p[i] + j), b.g[i]));
      }
    }
    store_vec(out + j, acc);
  }
}

// ---- launch schedules (host), shared by fft.cu and the CPU emulation ----

// level 0 is the polynomial (n coefficients); level l + 1 holds the heads of the tiles of level l; the levels stop at the first
// one that fits in one tile.  Levels >= 1 live in the caller's workspace, one after the other.
struct PolyLevels {
  int top = 0;            // index of the last level
  uint64_t m[65] = {};    // elements per level
  uint64_t off[65] = {};  // workspace offset (elements) of levels >= 1
  uint64_t work = 0;      // workspace elements
};
inline PolyLevels poly_levels(uint64_t n, int log_t) {
  PolyLevels lv;
  lv.m[0] = n;
  while (lv.m[lv.top] > (1ull << log_t)) {
    const uint64_t next = ((lv.m[lv.top] - 1) >> log_t) + 1;
    lv.top++;
    lv.m[lv.top] = next;
    lv.off[lv.top] = lv.work;
    lv.work += next;
  }
  return lv;
}

template <class P>
PolyMults<P> poly_mults(Fp<P> A, int log_l) {
  PolyMults<P> mu;
  mu.a = A;
  for (int i = 0; i < log_l; i++) A = fp_sqr(A);
  for (int k = 0; k < POLY_MAX_LOG_B; k++) {
    mu.m[k] = A;
    A = fp_sqr(A);
  }
  return mu;
}

// *fa = f(a) and, when h != NULL, h = (f - f(a)) / (X - a) (n - 1 elements); work: poly_levels(n, ..).work elements.
// heads(x, m, mu, out, tiles) and write(x, m, mu, carry, out, shift, fa, tiles) launch k_poly_heads / k_poly_write.
template <class P, class Heads, class Write>
void poly_div_schedule(const Fp<P>* f, uint64_t n, const Fp<P>& a, Fp<P>* h, Fp<P>* fa, Fp<P>* work, int log_l, int log_b,
                       Heads&& heads, Write&& write) {
  const int log_t = log_l + log_b;
  const PolyLevels lv = poly_levels(n, log_t);
  std::vector<PolyMults<P>> mu;   // level l multiplies by a^(T^l)
  Fp<P> A = a;
  for (int l = 0; l <= lv.top; l++) {
    mu.push_back(poly_mults(A, log_l));
    for (int i = 0; i < log_t; i++) A = fp_sqr(A);
  }
  auto level = [&](int l) { return work + lv.off[l]; };
  auto input = [&](int l) -> const Fp<P>* { return l ? level(l) : f; };
  auto tiles = [&](int l) { return ((lv.m[l] - 1) >> log_t) + 1; };
  for (int l = 0; l < lv.top; l++) heads(input(l), lv.m[l], mu[l], level(l + 1), tiles(l));
  if (!h) {
    heads(input(lv.top), lv.m[lv.top], mu[lv.top], fa, 1);
    return;
  }
  for (int l = lv.top; l >= 0; l--)
    write(input(l), lv.m[l], mu[l], l < lv.top ? level(l + 1) : nullptr, l ? level(l) : h, l ? 0 : 1, l == lv.top ? fa : nullptr,
          tiles(l));
}

// out (+)= sum_i scalars[i] polys[i] placed at stride strides[i] from offsets[i] (strides / offsets NULL: 1 / 0); launch(batch,
// accumulate, strided) runs k_poly_fold<P, strided>, strided = false for a batch whose strides are all 1 and offsets all 0
template <class P, class Launch>
void poly_lincomb_schedule(const Fp<P>* const* polys, const uint64_t* lens, const Fp<P>* scalars, const uint64_t* strides,
                           const uint64_t* offsets, uint64_t k, int accumulate, Launch&& launch) {
  for (uint64_t i0 = 0; i0 < k; i0 += POLY_FOLD_BATCH) {
    PolyFoldBatch<P> b{};
    b.count = (int)(k - i0 < (uint64_t)POLY_FOLD_BATCH ? k - i0 : POLY_FOLD_BATCH);
    bool strided = false;
    for (int i = 0; i < b.count; i++) {
      b.p[i] = polys[i0 + i];
      b.len[i] = lens[i0 + i];
      b.g[i] = scalars[i0 + i];
      b.stride[i] = strides ? strides[i0 + i] : 1;
      b.offset[i] = offsets ? offsets[i0 + i] : 0;
      strided |= b.stride[i] != 1 || b.offset[i] != 0;
    }
    launch(b, i0 > 0 ? 1 : accumulate, strided);
  }
}

// out = sum_i gamma^i polys[i] (zero past lens[i]): the linear combination with scalars gamma^i, stride 1 and offset 0;
// launch(batch, accumulate) runs k_poly_fold<P, false>
template <class P, class Launch>
void poly_fold_schedule(const Fp<P>* const* polys, const uint64_t* lens, uint64_t k, const Fp<P>& gamma, Launch&& launch) {
  if (k == 0) return;
  std::vector<Fp<P>> g(k);
  g[0] = Fp<P>::one();
  for (uint64_t i = 1; i < k; i++) g[i] = fp_mul(g[i - 1], gamma);
  poly_lincomb_schedule<P>(polys, lens, g.data(), nullptr, nullptr, k, 0,
                           [&](const PolyFoldBatch<P>& b, int accumulate, bool) { launch(b, accumulate); });
}

}  // namespace
