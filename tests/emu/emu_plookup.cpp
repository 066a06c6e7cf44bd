// TEST INFRASTRUCTURE ONLY -- the Fr kernels of plookup.ProveLookupVector (gnark-crypto_b200/csrc/plookup_kernels.cuh) on the CPU for
// every scalar field, launched in the order of fft.cu's gmsm_fr_sort_device (through the same fr_sort_schedule),
// gmsm_fr_plookup_accumulate_device and gmsm_fft_plookup_numerator_device (the kernels have barriers and warp votes: cooperative
// launcher).  The tile shapes are parameters, so that short vectors spread over many blocks.
#include <cstring>
#include <vector>

#include "fft_kernels.cuh"
#include "plookup_kernels.cuh"

namespace {
// the dynamic shared memory of the kernels (`extern __shared__ smem_raw[]`)
constexpr size_t EMU_SMEM = 64 * 1024;
thread_local __attribute__((aligned(16))) unsigned char smem_raw[EMU_SMEM];

template <class P>
bool inv_shape_ok(int log_t, unsigned threads) {
  return log_t >= 0 && perm_inv_smem_bytes<P>(log_t) <= EMU_SMEM && (1u << log_t) <= 32 * threads;
}

template <class P>
int emu_sort(const uint32_t* in_words, uint64_t n, uint32_t* out_words, int log_r, int log_b, int* passes) {
  using F = Fp<P>;
  if (n == 0 || log_r < 0 || log_b < 5 || log_b > 8) return 1;
  std::vector<F> in(n);
  std::memcpy(in.data(), in_words, n * sizeof(F));
  std::vector<unsigned char> work(sort_layout<P>(n, log_r, log_b).bytes + 16);
  *passes = 0;
  fr_sort_schedule<P>(
      in.data(), n, reinterpret_cast<F*>(out_words), work.data(), log_r, log_b,
      [&](auto kernel, unsigned grid, unsigned block, auto... args) { emu_launch_coop(kernel, dim3(grid), block, args...); },
      [&](uint32_t* host, const uint32_t* dev, int words) {
        std::memcpy(host, dev, words * 4);
        for (int b = 0; b < 4 * words; b++) *passes += (host[b >> 2] >> ((b & 3) * 8)) & 0xffu ? 1 : 0;   // the byte passes that run
      });
  return std::memcmp(in.data(), in_words, n * sizeof(F)) != 0 ? 2 : 0;
}

// consts: beta, gamma
template <class P>
int emu_accumulate(const uint32_t* f, const uint32_t* t, const uint32_t* h1, const uint32_t* h2, uint64_t n, const uint32_t* consts,
                   uint32_t* z_words, int log_t, unsigned threads, int log_l, int log_b) {
  using F = Fp<P>;
  if (n == 0 || !inv_shape_ok<P>(log_t, threads) || log_b > POLY_MAX_LOG_B || poly_smem_bytes<P>(log_l, log_b) > EMU_SMEM) return 1;
  PlookupConsts<P> k;
  std::memcpy(k.beta.l, consts, sizeof(F));
  std::memcpy(k.gamma.l, consts + sizeof(F) / 4, sizeof(F));
  k.opb = fp_add(F::one(), k.beta);
  k.gopb = fp_mul(k.gamma, k.opb);
  std::vector<F> work(poly_levels(n, log_l + log_b).work + 1);
  F* z = reinterpret_cast<F*>(z_words);
  emu_launch_coop(k_plookup_ratio<P>, dim3((unsigned)(((n - 1) >> log_t) + 1)), threads, reinterpret_cast<const F*>(f),
                  reinterpret_cast<const F*>(t), reinterpret_cast<const F*>(h1), reinterpret_cast<const F*>(h2), n, k, log_t, z);
  const unsigned B = 1u << log_b;
  perm_prefix_schedule<P>(
      z, n, work.data(), log_l, log_b,
      [&](const F* x, uint64_t m, F* heads, uint64_t tiles) { emu_launch_coop(k_perm_prod_heads<P>, dim3((unsigned)tiles), B, x, m, log_l, heads); },
      [&](F* x, uint64_t m, const F* carry, uint64_t tiles) { emu_launch_coop(k_perm_prod_write<P>, dim3((unsigned)tiles), B, x, m, log_l, carry); });
  return 0;
}

// in: lz, lh1, lh2, lt, lf (n each); tw: the n / 2 twiddles w^j of the big domain; consts: beta, gamma, alpha, shift, w^-1
template <class P>
int emu_numerator(const uint32_t* in, uint64_t n, const uint32_t* tw, const uint32_t* consts, uint32_t* out, int log_t, unsigned threads) {
  using F = Fp<P>;
  if (n == 0 || (n & (n - 1)) || !inv_shape_ok<P>(log_t, threads)) return 1;
  auto c = [&](int i) {
    F v;
    std::memcpy(v.l, consts + i * sizeof(F) / 4, sizeof(F));
    return v;
  };
  int logn = 0;
  while (((uint64_t)1 << logn) < n) logn++;
  // the constants as gmsm_fft_plookup_numerator_device derives them
  PlookupNumConsts<P> k;
  k.c.beta = c(0);
  k.c.gamma = c(1);
  k.alpha = c(2);
  k.shift = c(3);
  k.c.opb = fp_add(F::one(), k.c.beta);
  k.c.gopb = fp_mul(k.c.gamma, k.c.opb);
  k.gg = fp_sqr(c(4));
  F ss = k.shift;
  for (int i = 1; i < logn; i++) ss = fp_sqr(ss);
  k.xs_inv[0] = fp_inv(fp_sub(ss, F::one()));
  k.xs_inv[1] = fp_inv(fp_neg(fp_add(ss, F::one())));
  const F* v = reinterpret_cast<const F*>(in);
  emu_launch_coop(k_plookup_numerator<P>, dim3((unsigned)(((n - 1) >> log_t) + 1)), threads, v, v + n, v + 2 * n, v + 3 * n, v + 4 * n, n,
                  logn, k, reinterpret_cast<const F*>(tw), log_t, reinterpret_cast<F*>(out));
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

// field: GMSM_FR_* (0 bn254 ... 6 bw6-761); elements of fr.Limbs u64 (8 / 10 / 12 u32) Montgomery limbs.  Negative shape
// parameters: the shapes fft.cu uses for the field.  Returns 0, 1 for a refused shape, or 2 if an input was written.
extern "C" int emu_plookup_sort(int field, const uint32_t* in, uint64_t n, uint32_t* out, int log_r, int log_b, int* passes) {
  return with_field(field, [&](auto p) {
    using P = decltype(p);
    return emu_sort<P>(in, n, out, log_r < 0 ? SORT_LOG_R : log_r, log_b < 0 ? SORT_LOG_B : log_b, passes);
  });
}

extern "C" int emu_plookup_accumulate(int field, const uint32_t* f, const uint32_t* t, const uint32_t* h1, const uint32_t* h2, uint64_t n,
                                      const uint32_t* consts, uint32_t* z, int log_t, unsigned threads, int log_l, int log_b) {
  return with_field(field, [&](auto p) {
    using P = decltype(p);
    return emu_accumulate<P>(f, t, h1, h2, n, consts, z, log_t < 0 ? PERM_INV_LOG_T : log_t, threads ? threads : PERM_INV_THREADS,
                             log_l < 0 ? poly_log_l<P>() : log_l, log_b < 0 ? poly_log_b<P>() : log_b);
  });
}

extern "C" int emu_plookup_numerator(int field, const uint32_t* in, uint64_t n, const uint32_t* tw, const uint32_t* consts, uint32_t* out,
                                     int log_t, unsigned threads) {
  return with_field(field, [&](auto p) {
    using P = decltype(p);
    return emu_numerator<P>(in, n, tw, consts, out, log_t < 0 ? PERM_INV_LOG_T : log_t, threads ? threads : PERM_INV_THREADS);
  });
}
