// TEST INFRASTRUCTURE ONLY -- the Fr kernels of permutation.Prove (gnark-crypto_b200/csrc/perm_kernels.cuh) on the CPU for every
// scalar field, launched in the order of fft.cu's gmsm_fr_batch_invert_device, gmsm_fr_permutation_accumulate_device and
// gmsm_fft_permutation_numerator_device (the kernels have barriers: cooperative launcher).  The tile shapes are parameters, so
// that short vectors reach several scan levels.
#include <cstring>
#include <vector>

#include "fft_kernels.cuh"
#include "perm_kernels.cuh"

namespace {
// the dynamic shared memory of the kernels (`extern __shared__ smem_raw[]`)
constexpr size_t EMU_SMEM = 64 * 1024;
thread_local __attribute__((aligned(16))) unsigned char smem_raw[EMU_SMEM];

template <class P>
bool inv_shape_ok(int log_t, unsigned threads) {
  return log_t >= 0 && perm_inv_smem_bytes<P>(log_t) <= EMU_SMEM && (1u << log_t) <= 32 * threads;
}

template <class P>
int emu_invert(const uint32_t* a_words, uint64_t n, uint32_t* out, int log_t, unsigned threads) {
  using F = Fp<P>;
  if (n == 0 || !inv_shape_ok<P>(log_t, threads)) return 1;
  std::vector<F> a(n);
  std::memcpy(a.data(), a_words, n * sizeof(F));
  emu_launch_coop(k_fr_batch_invert<P>, dim3((unsigned)(((n - 1) >> log_t) + 1)), threads, (const F*)a.data(), n, log_t,
                  reinterpret_cast<F*>(out));
  return std::memcmp(a.data(), a_words, n * sizeof(F)) != 0 ? 2 : 0;
}

template <class P>
int emu_accumulate(const uint32_t* t1_words, const uint32_t* t2_words, uint64_t n, const uint32_t* eps_words, uint32_t* z_words, int log_t,
                   unsigned threads, int log_l, int log_b) {
  using F = Fp<P>;
  if (n == 0 || (n & (n - 1)) || !inv_shape_ok<P>(log_t, threads) || log_b > POLY_MAX_LOG_B ||
      poly_smem_bytes<P>(log_l, log_b) > EMU_SMEM)
    return 1;
  F eps;
  std::memcpy(eps.l, eps_words, sizeof(F));
  std::vector<F> t1(n), t2(n), work(poly_levels(n, log_l + log_b).work + 1);
  std::memcpy(t1.data(), t1_words, n * sizeof(F));
  std::memcpy(t2.data(), t2_words, n * sizeof(F));
  F* z = reinterpret_cast<F*>(z_words);
  emu_launch_coop(k_perm_ratio<P>, dim3((unsigned)(((n - 1) >> log_t) + 1)), threads, (const F*)t1.data(), (const F*)t2.data(), n, eps,
                  log_t, z);
  const unsigned B = 1u << log_b;
  perm_prefix_schedule<P>(
      z, n, work.data(), log_l, log_b,
      [&](const F* x, uint64_t m, F* heads, uint64_t tiles) { emu_launch_coop(k_perm_prod_heads<P>, dim3((unsigned)tiles), B, x, m, log_l, heads); },
      [&](F* x, uint64_t m, const F* carry, uint64_t tiles) { emu_launch_coop(k_perm_prod_write<P>, dim3((unsigned)tiles), B, x, m, log_l, carry); });
  int logn = 0;
  while (((uint64_t)1 << logn) < n) logn++;
  emu_launch(k_fft_bit_reverse<P>, dim3(4), 64u, z, n, logn);
  const bool changed = std::memcmp(t1.data(), t1_words, n * sizeof(F)) || std::memcmp(t2.data(), t2_words, n * sizeof(F));
  return changed ? 2 : 0;
}

// tw: the n / 2 twiddles w^j of the domain (built by the caller); consts: eps, omega, g, (g^n - 1)^-1
template <class P>
int emu_numerator(const uint32_t* lt1, const uint32_t* lt2, const uint32_t* lz, uint64_t n, const uint32_t* tw, const uint32_t* consts,
                  uint32_t* out, int log_t, unsigned threads) {
  using F = Fp<P>;
  if (n == 0 || (n & (n - 1)) || !inv_shape_ok<P>(log_t, threads)) return 1;
  PermNumConsts<P> k;
  std::memcpy(k.eps.l, consts, sizeof(F));
  std::memcpy(k.omega.l, consts + 1 * sizeof(F) / 4, sizeof(F));
  std::memcpy(k.g.l, consts + 2 * sizeof(F) / 4, sizeof(F));
  std::memcpy(k.tn_inv.l, consts + 3 * sizeof(F) / 4, sizeof(F));
  int logn = 0;
  while (((uint64_t)1 << logn) < n) logn++;
  emu_launch_coop(k_perm_numerator<P>, dim3((unsigned)(((n - 1) >> log_t) + 1)), threads, reinterpret_cast<const F*>(lt1),
                  reinterpret_cast<const F*>(lt2), reinterpret_cast<const F*>(lz), n, logn, k, reinterpret_cast<const F*>(tw), log_t,
                  reinterpret_cast<F*>(out));
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

// field: GMSM_FR_* (0 bn254 ... 6 bw6-761); elements of fr.Limbs u64 (8 / 10 / 12 u32) Montgomery limbs.  log_t < 0 (and
// log_l, log_b < 0): the tile shapes fft.cu uses for the field.  Returns 0, 1 for a refused shape, or 2 if an input was written.
extern "C" int emu_perm_invert(int field, const uint32_t* a, uint64_t n, uint32_t* out, int log_t, unsigned threads) {
  return with_field(field, [&](auto p) {
    using P = decltype(p);
    return emu_invert<P>(a, n, out, log_t < 0 ? PERM_INV_LOG_T : log_t, threads ? threads : PERM_INV_THREADS);
  });
}

extern "C" int emu_perm_accumulate(int field, const uint32_t* t1, const uint32_t* t2, uint64_t n, const uint32_t* eps, uint32_t* z, int log_t,
                                   unsigned threads, int log_l, int log_b) {
  return with_field(field, [&](auto p) {
    using P = decltype(p);
    return emu_accumulate<P>(t1, t2, n, eps, z, log_t < 0 ? PERM_INV_LOG_T : log_t, threads ? threads : PERM_INV_THREADS,
                             log_l < 0 ? poly_log_l<P>() : log_l, log_b < 0 ? poly_log_b<P>() : log_b);
  });
}

extern "C" int emu_perm_numerator(int field, const uint32_t* lt1, const uint32_t* lt2, const uint32_t* lz, uint64_t n, const uint32_t* tw,
                                  const uint32_t* consts, uint32_t* out, int log_t, unsigned threads) {
  return with_field(field, [&](auto p) {
    using P = decltype(p);
    return emu_numerator<P>(lt1, lt2, lz, n, tw, consts, out, log_t < 0 ? PERM_INV_LOG_T : log_t, threads ? threads : PERM_INV_THREADS);
  });
}
