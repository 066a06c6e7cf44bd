// TEST INFRASTRUCTURE ONLY -- the Fr polynomial kernels of a KZG opening (gnark-crypto_b200/csrc/poly_kernels.cuh) on the CPU
// for every scalar field, launched by the same schedules as fft.cu's gmsm_fr_poly_div_x_minus_a_device / gmsm_fr_poly_fold_device:
// k_poly_heads level by level, then k_poly_write top-down (both have barriers: cooperative launcher), and k_poly_fold.  The tile
// shape (log2 of the chunk length and of the block size) is a parameter, so that small polynomials reach several carry levels.
#include <cstring>
#include <vector>

#include "poly_kernels.cuh"

namespace {
// the dynamic shared memory of k_poly_heads / k_poly_write (`extern __shared__ smem_raw[]`)
constexpr size_t EMU_SMEM = 64 * 1024;
thread_local __attribute__((aligned(16))) unsigned char smem_raw[EMU_SMEM];

template <class P>
int emu_div(const uint32_t* f_words, uint64_t n, const uint32_t* a_words, uint32_t* h_words, uint32_t* fa_words, int log_l, int log_b) {
  using F = Fp<P>;
  if (n == 0 || log_b > POLY_MAX_LOG_B || poly_smem_bytes<P>(log_l, log_b) > EMU_SMEM) return 1;
  F a;
  std::memcpy(a.l, a_words, sizeof(F));
  std::vector<F> f(n), work(poly_levels(n, log_l + log_b).work + 1);
  std::memcpy(f.data(), f_words, n * sizeof(F));
  const unsigned B = 1u << log_b;
  poly_div_schedule<P>(
      f.data(), n, a, reinterpret_cast<F*>(h_words), reinterpret_cast<F*>(fa_words), work.data(), log_l, log_b,
      [&](const F* x, uint64_t m, const PolyMults<P>& mu, F* heads, uint64_t tiles) {
        emu_launch_coop(k_poly_heads<P>, dim3((unsigned)tiles), B, x, m, mu, log_l, heads);
      },
      [&](const F* x, uint64_t m, const PolyMults<P>& mu, const F* carry, F* out, int shift, F* fa, uint64_t tiles) {
        emu_launch_coop(k_poly_write<P>, dim3((unsigned)tiles), B, x, m, mu, log_l, carry, out, shift, fa);
      });
  return std::memcmp(f.data(), f_words, n * sizeof(F)) != 0 ? 2 : 0;   // the polynomial is left unchanged
}

template <class P>
int emu_fold(const uint32_t* const* polys, const uint64_t* lens, uint64_t k, const uint32_t* gamma_words, uint32_t* out, uint64_t out_len) {
  using F = Fp<P>;
  F g;
  std::memcpy(g.l, gamma_words, sizeof(F));
  const unsigned blocks = (unsigned)std::min<uint64_t>((out_len + 255) / 256, 8u);
  poly_fold_schedule<P>(reinterpret_cast<const F* const*>(polys), lens, k, g, [&](const PolyFoldBatch<P>& b, int accumulate) {
    emu_launch(k_poly_fold<P>, dim3(blocks), 256u, reinterpret_cast<F*>(out), out_len, b, accumulate);
  });
  return 0;
}

template <class Fn>
int with_field(int field, Fn&& fn) {
  switch (field) {
    case 0: return fn(bn254_fr{});
    case 1: return fn(bls12381_fr{});
    case 2: return fn(bls12377_fr{});
    case 3: return fn(bls24315_fr{});
    case 4: return fn(bls24317_fr{});
    case 5: return fn(bw6633_fr{});
    case 6: return fn(bw6761_fr{});
  }
  return 1;
}
}  // namespace

// field: GMSM_FR_* (0 bn254 ... 6 bw6-761); elements of fr.Limbs u64 (8 / 10 / 12 u32) Montgomery limbs.  *fa = f(a); h (n - 1
// elements, NULL: evaluation only) = (f - f(a)) / (X - a).  log_l, log_b < 0: the shape fft.cu uses for the field.
// Returns 0, or 2 if the kernels wrote to f.
extern "C" int emu_poly_div(int field, const uint32_t* f, uint64_t n, const uint32_t* a, uint32_t* h, uint32_t* fa, int log_l, int log_b) {
  return with_field(field, [&](auto p) {
    using P = decltype(p);
    return emu_div<P>(f, n, a, h, fa, log_l < 0 ? poly_log_l<P>() : log_l, log_b < 0 ? poly_log_b<P>() : log_b);
  });
}

// out[j] = sum_i gamma^i polys[i][j], j < out_len, polys[i] zero past lens[i]
extern "C" int emu_poly_fold(int field, const uint32_t* const* polys, const uint64_t* lens, uint64_t k, const uint32_t* gamma, uint32_t* out,
                             uint64_t out_len) {
  return with_field(field, [&](auto p) { return emu_fold<decltype(p)>(polys, lens, k, gamma, out, out_len); });
}
