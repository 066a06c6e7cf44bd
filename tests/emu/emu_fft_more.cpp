// TEST INFRASTRUCTURE ONLY -- the Fr FFT kernels (gnark-crypto_b200/csrc/fft_kernels.cuh) on the CPU for every scalar field,
// with elements of 32, 40 (bw6-633) or 48 (bw6-761) bytes; launched in the order of fft.cu's domain_build / run_fft, like
// emu_fft.cpp does for the 32-byte fields: twiddle table by k_fft_powers, coset scaling, strided DIF / DIT stages, the
// shared-memory tile kernel (barriers: cooperative launcher), final scaling.  The domain constants (Generator, GeneratorInv,
// CardinalityInv, coset shift and its inverse; Montgomery limbs) are passed in by the test.
#include <algorithm>
#include <cstring>
#include <vector>

#include "fft_kernels.cuh"

namespace {
// the dynamic shared memory of k_fft_tile (`extern __shared__ smem_raw[]`): 1024 elements of up to 48 bytes
thread_local __attribute__((aligned(16))) unsigned char smem_raw[TILE * 48];

template <class P>
int emu_fft(uint32_t* a_words, uint64_t n, int logn, int inverse, int decimation, int coset, const uint32_t* consts5) {
  using F = Fp<P>;
  static_assert(sizeof(F) <= 48, "smem_raw holds 1024 elements of at most 48 bytes");
  constexpr int N = P::N;   // u32 limbs per element: consts5 is 5 rows of N
  F* a = reinterpret_cast<F*>(a_words);
  auto grid = [](uint64_t work) { return (unsigned)std::min<uint64_t>((work + 255) / 256, 8u); };
  F gen, gen_inv, card_inv, shift, shift_inv;
  std::memcpy(gen.l, consts5, sizeof(F)); std::memcpy(gen_inv.l, consts5 + N, sizeof(F)); std::memcpy(card_inv.l, consts5 + 2 * N, sizeof(F));
  std::memcpy(shift.l, consts5 + 3 * N, sizeof(F)); std::memcpy(shift_inv.l, consts5 + 4 * N, sizeof(F));
  // domain_build: pw[0..63] = shift^(2^k), pw[64..127] = shift^-(2^k), pw[128..191] = w^(2^k); tw[j] = w^j, j < n/2
  std::vector<F> pw(192);
  {
    F x = shift, y = shift_inv, w = inverse ? gen_inv : gen;
    for (int k = 0; k < 64; k++) { pw[k] = x; pw[64 + k] = y; pw[128 + k] = w; x = fp_sqr(x); y = fp_sqr(y); w = fp_sqr(w); }
  }
  const uint64_t half = n >> 1;
  std::vector<F> tw(std::max<uint64_t>(half, 1));
  if (half) emu_launch(k_fft_powers<P>, dim3(grid(half)), 256u, tw.data(), half, (const F*)(pw.data() + 128), logn > 0 ? logn - 1 : 0);
  // run_fft
  const F one = F::one();
  if (!inverse && coset) emu_launch(k_fft_scale<P>, dim3(grid(n)), 256u, a, n, logn, (const F*)pw.data(), 1, (int)(decimation == 0), one, 0);
  if (n > 1) {
    const uint32_t tile = (uint32_t)std::min<uint64_t>(n, TILE);
    if (decimation == 1) {
      for (uint64_t h = half; h >= tile; h >>= 1) emu_launch(k_fft_dif_stage<P>, dim3(grid(half)), 256u, a, (const F*)tw.data(), half, h, half / h);
      emu_launch_coop(k_fft_tile<P, true>, dim3((unsigned)(n / tile)), tile / 2, a, (const F*)tw.data(), n, tile);
    } else {
      emu_launch_coop(k_fft_tile<P, false>, dim3((unsigned)(n / tile)), tile / 2, a, (const F*)tw.data(), n, tile);
      for (uint64_t h = tile; h <= half; h <<= 1) emu_launch(k_fft_dit_stage<P>, dim3(grid(half)), 256u, a, (const F*)tw.data(), half, h, half / h);
    }
  }
  if (inverse) emu_launch(k_fft_scale<P>, dim3(grid(n)), 256u, a, n, logn, (const F*)(pw.data() + 64), coset ? 1 : 0, (int)(decimation == 1), card_inv, 1);
  return 0;
}
}  // namespace

// field: GMSM_FR_* (0 bn254, 1 bls12-381, 2 bls12-377, 3 bls24-315, 4 bls24-317, 5 bw6-633, 6 bw6-761); a: n elements of
// fr.Limbs u64 (8 / 10 / 12 u32) Montgomery limbs, transformed in place; consts5: 5 such elements
extern "C" int emu_fft_more_run(int field, uint32_t* a, uint64_t n, int logn, int inverse, int decimation, int coset, const uint32_t* consts5) {
  if (n == 0 || (n & (n - 1)) || (1ull << logn) != n) return 1;
  switch (field) {
    case 0: return emu_fft<bn254_fr>(a, n, logn, inverse, decimation, coset, consts5);
    case 1: return emu_fft<bls12381_fr>(a, n, logn, inverse, decimation, coset, consts5);
    case 2: return emu_fft<bls12377_fr>(a, n, logn, inverse, decimation, coset, consts5);
    case 3: return emu_fft<bls24315_fr>(a, n, logn, inverse, decimation, coset, consts5);
    case 4: return emu_fft<bls24317_fr>(a, n, logn, inverse, decimation, coset, consts5);
    case 5: return emu_fft<bw6633_fr>(a, n, logn, inverse, decimation, coset, consts5);
    case 6: return emu_fft<bw6761_fr>(a, n, logn, inverse, decimation, coset, consts5);
  }
  return 1;
}
