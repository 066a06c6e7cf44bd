// TEST INFRASTRUCTURE ONLY -- the strided linear combination of gnark-crypto_b200/csrc/poly_kernels.cuh (k_poly_fold, both
// instantiations) on the CPU for every scalar field, launched by poly_lincomb_schedule exactly as fft.cu's
// gmsm_fr_poly_lincomb_device launches it.
#include <cstring>
#include <vector>

#include "poly_kernels.cuh"

namespace {
template <class P>
int emu_lincomb(const uint32_t* const* polys, const uint64_t* lens, const uint32_t* scalar_words, const uint64_t* strides,
                const uint64_t* offsets, uint64_t k, uint32_t* out, uint64_t out_len, int accumulate) {
  using F = Fp<P>;
  std::vector<F> s(k);
  for (uint64_t i = 0; i < k; i++) std::memcpy(s[i].l, scalar_words + i * (sizeof(F) / 4), sizeof(F));
  const unsigned blocks = (unsigned)std::min<uint64_t>((out_len + 255) / 256, 8u);
  F* o = reinterpret_cast<F*>(out);
  poly_lincomb_schedule<P>(reinterpret_cast<const F* const*>(polys), lens, s.data(), strides, offsets, k, accumulate,
                           [&](const PolyFoldBatch<P>& b, int acc, bool strided) {
                             if (strided)
                               emu_launch(k_poly_fold<P, true>, dim3(blocks), 256u, o, out_len, b, acc);
                             else
                               emu_launch(k_poly_fold<P, false>, dim3(blocks), 256u, o, out_len, b, acc);
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

// field: GMSM_FR_* (0 bn254 ... 6 bw6-761); elements of fr.Limbs u64 Montgomery limbs; scalars: k elements.
// out[m strides[i] + offsets[i]] (+)= scalars[i] polys[i][m] for m < lens[i], indices below out_len (accumulate = 0: the rest 0)
extern "C" int emu_poly_lincomb(int field, const uint32_t* const* polys, const uint64_t* lens, const uint32_t* scalars,
                                const uint64_t* strides, const uint64_t* offsets, uint64_t k, uint32_t* out, uint64_t out_len,
                                int accumulate) {
  return with_field(field, [&](auto p) {
    return emu_lincomb<decltype(p)>(polys, lens, scalars, strides, offsets, k, out, out_len, accumulate);
  });
}
