// Next-row N3: radix-2 FFT over Fr on the GPU, behind gnark-crypto's fft.Domain interface.
//
// Replaces (reference tree; the fr/fft packages of bls12-381, bls12-377, bls24-315, bls24-317, bw6-633 and bw6-761 are the same
// generated code with their own constants):
//   fft.NewDomain / Domain{Cardinality, CardinalityInv, Generator, GeneratorInv, FrMultiplicativeGen(Inv)}
//                                                             ecc/bn254/fr/fft/domain.go:24-110
//   fr.Generator(m) (2-adic root of unity, maxOrderRoot)      ecc/bn254/fr/generator.go:18-36
//   (*Domain).FFT / FFTInverse (DIF: natural in, bit-reversed out; DIT: bit-reversed in, natural out; coset
//   option; FFTInverse scales by CardinalityInv)              ecc/bn254/fr/fft/fft.go:31-190, difFFT :195+, ditFFT :262+
//   BitReverse                                                 ecc/bn254/fr/fft/bitreverse.go:17-42
//
// Data is the reference's []fr.Element image (fr.Limbs u64 Montgomery limbs: 4; 5 for bw6-633, 6 for bw6-761).  Kernels: one launch per butterfly
// stage for the strided stages, one shared-memory kernel for the last (DIF) / first (DIT) TILE_LOG stages,
// twiddles w^j (j < n/2) precomputed per domain like the reference's Domain.twiddles; coset powers are
// computed on the fly from u^(2^k).  HBM-bound streaming work: fr.Bytes (32 / 40 / 48) per element per pass.
//
// Also the Fr polynomial steps of a KZG opening on device vectors (kernels and schedules in poly_kernels.cuh):
//   eval                          ecc/bn254/kzg/kzg.go:55-63
//   dividePolyByXminusA           ecc/bn254/kzg/kzg.go:567-582
//   the gamma-fold of BatchOpenSinglePoint   ecc/bn254/kzg/kzg.go:302-319
//   the strided linear combinations of shplonk.BatchOpen / fflonk.Fold (gmsm_fr_poly_lincomb_device)
// and the Fr steps of permutation.Prove (kernels and schedule in perm_kernels.cuh):
//   fr.BatchInvert                                ecc/bn254/fr/element.go:658-687
//   evaluateAccumulationPolynomialBitReversed     ecc/bn254/fr/permutation/permutation.go:52-75
//   the quotient numerator and its omega-fold     ecc/bn254/fr/permutation/permutation.go:78-121, 206-214
// and the Fr steps of plookup.ProveLookupVector (kernels and the sort's schedule in plookup_kernels.cuh):
//   sort.Sort(fr.Vector)                          ecc/bn254/fr/element.go:254 (fr.Element.Cmp)
//   evaluateAccumulationPolynomial                ecc/bn254/fr/plookup/vector.go:52-95
//   the quotient numerator and its alpha-fold     ecc/bn254/fr/plookup/vector.go:97-335
// and the O(n) steps of the iop package (kernels in iop_kernels.cuh; the FFTs are the ones above):
//   BuildRatioShuffledVectors / BuildRatioCopyConstraint   ecc/bn254/fr/iop/ratios.go:45-246
//   evalLagrange of Polynomial.Evaluate                    ecc/bn254/fr/iop/polynomial.go:204-241
//   Evaluate (an interpreted straight-line program)        ecc/bn254/fr/iop/expressions.go:26-73
//   DivideByXMinusOne                                      ecc/bn254/fr/iop/quotient.go:21-53
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>

#include "engine.h"
#include "field.cuh"

using namespace gmsm;

#include "fft_kernels.cuh"
#include "poly_kernels.cuh"
#include "perm_kernels.cuh"
#include "plookup_kernels.cuh"
#include "iop_kernels.cuh"

namespace {

// ---- host-side field helpers (portable path of field.cuh) ----
template <class P>
Fp<P> host_from_u64(uint64_t v) {
  Fp<P> c = Fp<P>::zero();
  c.l[0] = (uint32_t)v;
  c.l[1] = (uint32_t)(v >> 32);
  return fp_to_mont(c);
}
template <class P>
Fp<P> host_from_decimal(const char* dec) {  // canonical integer < q given in decimal -> Montgomery
  Fp<P> acc = Fp<P>::zero(), ten = host_from_u64<P>(10);
  for (const char* p = dec; *p; p++) acc = fp_add(fp_mul(acc, ten), host_from_u64<P>((uint64_t)(*p - '0')));
  return acc;
}
template <class P>
Fp<P> host_pow2k(Fp<P> x, int k) {  // x^(2^k)
  for (int i = 0; i < k; i++) x = fp_sqr(x);
  return x;
}

struct FrConsts {
  const char* root;   // fr.Generator's rootOfUnity (decimal), generator.go:23
  int max_order;      // maxOrderRoot, generator.go:24
  uint64_t mult_gen;  // GeneratorFullMultiplicativeGroup, fft/domain.go:55-63
};
// one row per scalar field id (GMSM_FR_*), in the order of the ids
const FrConsts FR_CONSTS[] = {
    {"19103219067921713944291392827692070036145651957329286315305642004821462161904", 28, 5},     // bn254
    {"10238227357739495823651030575849232062558860180284477541189508159991286009131", 32, 7},     // bls12-381
    // ecc/bls12-377/fr/generator.go:23-24, fr/fft/domain.go:59
    {"8065159656716812877374967518403273466521432693661810619979959746626482506078", 47, 22},
    // ecc/{bls24-315,bls24-317,bw6-633,bw6-761}/fr/generator.go:23-24, fr/fft/domain.go:59.  Each root is
    // GeneratorFullMultiplicativeGroup^((r - 1) >> maxOrderRoot), of order exactly 2^maxOrderRoot.
    {"1792993287828780812362846131493071959406149719416102105453370749552622525216", 22, 7},      // bls24-315
    {"16532287748948254263922689505213135976137839535221842169193829039521719560631", 60, 7},     // bls24-317
    {"4991787701895089137426454739366935169846548798279261157172811661565882460884369603588700158257", 20, 13},   // bw6-633
    {"32863578547254505029601261939868325669770508939375122462904745766352256812585773382134936404344547323199885654433", 46,
     15},                                                                                           // bw6-761
};
static_assert(sizeof(FR_CONSTS) / sizeof(FR_CONSTS[0]) == GMSM_FR_BW6761 + 1, "one row per scalar field id");

const FrConsts* fr_consts(int field) { return field >= 0 && field <= GMSM_FR_BW6761 ? &FR_CONSTS[field] : nullptr; }

// log2 of ecc.NextPowerOfTwo(m) into *logn, refused past maxOrderRoot as fr.Generator refuses it (generator.go:29)
int domain_log(const FrConsts& fc, uint64_t m, int* logn) {
  int k = 0;
  while (k <= fc.max_order && ((uint64_t)1 << k) < m) k++;
  if (k > fc.max_order)
    return set_err(GMSM_EINVAL, "m (%llu) is too big: the required root of unity does not exist", (unsigned long long)m);
  *logn = k;
  return GMSM_OK;
}

template <class P>
struct FrTag {
  using type = P;
};
// calls fn(FrTag<P>{}) with the Fp parameters of a scalar field id (checked by the caller)
template <class Fn>
int with_fr(int field, Fn&& fn) {
  switch (field) {
    case GMSM_FR_BN254: return fn(FrTag<bn254_fr>{});
    case GMSM_FR_BLS12381: return fn(FrTag<bls12381_fr>{});
    case GMSM_FR_BLS12377: return fn(FrTag<bls12377_fr>{});
    case GMSM_FR_BLS24315: return fn(FrTag<bls24315_fr>{});
    case GMSM_FR_BLS24317: return fn(FrTag<bls24317_fr>{});
    case GMSM_FR_BW6633: return fn(FrTag<bw6633_fr>{});
    case GMSM_FR_BW6761: return fn(FrTag<bw6761_fr>{});
  }
  return set_err(GMSM_EINVAL, "unknown scalar field %d", field);
}
constexpr int FR_MAX_WORDS = 6;   // u64 limbs of the widest scalar field (bw6-761)

}  // namespace

struct gmsm_fft_domain {
  int field = 0, device = 0, logn = 0;
  int words = 0;                // u64 limbs per element (fr.Limbs); elements are 8 * words bytes
  uint64_t n = 0;
  uint64_t consts[5][FR_MAX_WORDS] = {};   // Generator, GeneratorInv, CardinalityInv, FrMultiplicativeGen, FrMultiplicativeGenInv
  void *d_tw = nullptr, *d_tw_inv = nullptr;       // w^j, w^-j for j < n/2
  void *d_pw = nullptr;                            // [0..63]: u^(2^k); [64..127]: u^-(2^k); [128..191]: scratch for twiddle builds
  void* d_buf = nullptr;                           // staging for the host entry points
  std::mutex mu;
};

template <class P>
static int domain_build(gmsm_fft_domain* d, const FrConsts& fc, const uint64_t* shift_mont) {
  using F = Fp<P>;
  F gen = host_pow2k(host_from_decimal<P>(fc.root), fc.max_order - d->logn);
  F gen_inv = fp_inv(gen);
  F card_inv = fp_inv(host_from_u64<P>(d->n));
  static_assert(sizeof(F) <= sizeof(d->consts[0]), "consts row too small");
  F shift;
  if (shift_mont) memcpy(shift.l, shift_mont, sizeof(F)); else shift = host_from_u64<P>(fc.mult_gen);
  F shift_inv = fp_inv(shift);
  memcpy(d->consts[0], gen.l, sizeof(F)); memcpy(d->consts[1], gen_inv.l, sizeof(F)); memcpy(d->consts[2], card_inv.l, sizeof(F));
  memcpy(d->consts[3], shift.l, sizeof(F)); memcpy(d->consts[4], shift_inv.l, sizeof(F));
  F pw[192];
  F a = shift, b = shift_inv, g = gen, gi = gen_inv;
  for (int k = 0; k < 64; k++) { pw[k] = a; pw[64 + k] = b; a = fp_sqr(a); b = fp_sqr(b); }
  CK(cudaMalloc(&d->d_pw, sizeof(pw)));
  const uint64_t half = d->n >> 1;
  CK(cudaMalloc(&d->d_tw, (half ? half : 1) * sizeof(F)));
  CK(cudaMalloc(&d->d_tw_inv, (half ? half : 1) * sizeof(F)));
  for (int pass = 0; pass < 2; pass++) {
    F w = pass ? gi : g;
    for (int k = 0; k < 64; k++) { pw[128 + k] = w; w = fp_sqr(w); }
    CK(cudaMemcpy(d->d_pw, pw, sizeof(pw), cudaMemcpyHostToDevice));
    if (half) {
      unsigned blocks = (unsigned)std::min<uint64_t>((half + 255) / 256, GMSM_NUM_SMS * 16u);
      k_fft_powers<P><<<blocks, 256>>>(reinterpret_cast<F*>(pass ? d->d_tw_inv : d->d_tw), half,
                                       reinterpret_cast<const F*>(d->d_pw) + 128, d->logn > 0 ? d->logn - 1 : 0);
      CK(cudaGetLastError());
      CK(cudaDeviceSynchronize());
    }
  }
  return GMSM_OK;
}

template <class P>
static int run_fft(gmsm_fft_domain* d, void* d_a, int inverse, int decimation, int coset, cudaStream_t st) {
  using F = Fp<P>;
  F* a = reinterpret_cast<F*>(d_a);
  const uint64_t n = d->n, half = n >> 1;
  const F* pw = reinterpret_cast<const F*>(d->d_pw);
  const F* tw = reinterpret_cast<const F*>(inverse ? d->d_tw_inv : d->d_tw);
  auto grid = [](uint64_t work) { return (unsigned)std::min<uint64_t>((work + 255) / 256, GMSM_NUM_SMS * 32u); };
  F one = F::one();
  if (!inverse && coset) {
    // FFT: a[i] *= u^i (DIF, natural input) or u^bitrev(i) (DIT, bit-reversed input)   fft.go:44-86
    k_fft_scale<P><<<grid(n), 256, 0, st>>>(a, n, d->logn, pw, 1, decimation == 0 /*DIT*/, one, 0);
  }
  if (n > 1) {
    const uint32_t tile = (uint32_t)std::min<uint64_t>(n, TILE);
    const size_t smem = (size_t)tile * sizeof(F);
    if (decimation == 1) {  // DIF: large strides first, then the tile kernel
      for (uint64_t h = half; h >= tile; h >>= 1) k_fft_dif_stage<P><<<grid(half), 256, 0, st>>>(a, tw, half, h, half / h);
      k_fft_tile<P, true><<<(unsigned)(n / tile), tile / 2, smem, st>>>(a, tw, n, tile);
    } else {                // DIT: the tile kernel first, then growing strides
      k_fft_tile<P, false><<<(unsigned)(n / tile), tile / 2, smem, st>>>(a, tw, n, tile);
      for (uint64_t h = tile; h <= half; h <<= 1) k_fft_dit_stage<P><<<grid(half), 256, 0, st>>>(a, tw, half, h, half / h);
    }
  }
  if (inverse) {
    // FFTInverse: scale by CardinalityInv, and on a coset by u^-i (DIT, natural output) or u^-bitrev(i) (DIF)
    F ci;
    memcpy(ci.l, d->consts[2], sizeof(F));
    k_fft_scale<P><<<grid(n), 256, 0, st>>>(a, n, d->logn, pw + 64, coset ? 1 : 0, decimation == 1 /*DIF*/, ci, 1);
  }
  CK(cudaGetLastError());
  return GMSM_OK;
}

// the domain inverses of kzg.ToLagrangeG1 (computeTwiddlesInv, ecc/bn254/kzg/utils.go:66-93): the same root as a domain of n
int gmsm::fr_domain_inverses(int fr_field, uint64_t n, uint64_t* w_inv, uint64_t* n_inv) {
  const FrConsts* fcp = fr_consts(fr_field);
  if (!fcp) return set_err(GMSM_EINVAL, "unknown scalar field %d", fr_field);
  int logn = 0;
  if (int rc = domain_log(*fcp, n, &logn)) return rc;
  return with_fr(fr_field, [&](auto tag) -> int {
    using P = typename decltype(tag)::type;
    const Fp<P> wi = fp_inv(host_pow2k(host_from_decimal<P>(fcp->root), fcp->max_order - logn));
    const Fp<P> ni = fp_inv(host_from_u64<P>(n));
    memcpy(w_inv, wi.l, sizeof(Fp<P>));
    memcpy(n_inv, ni.l, sizeof(Fp<P>));
    return GMSM_OK;
  });
}

extern "C" gmsm_fft_domain_t* gmsm_fft_domain_create(int fr_field, uint64_t m, const uint64_t* shift, int device) {
  const FrConsts* fcp = fr_consts(fr_field);
  if (!fcp) { set_err(GMSM_EINVAL, "unknown scalar field %d", fr_field); return nullptr; }
  if (use_device(device, "device %d out of range") != GMSM_OK) return nullptr;
  const FrConsts& fc = *fcp;
  int logn = 0;
  if (domain_log(fc, m, &logn) != GMSM_OK) return nullptr;
  const uint64_t x = (uint64_t)1 << logn;
  gmsm_fft_domain* d = new gmsm_fft_domain();
  d->field = fr_field; d->device = device; d->n = x; d->logn = logn;
  d->words = (int)(gmsm_fft_fr_bytes(fr_field) / 8);
  int rc = with_fr(fr_field, [&](auto tag) { return domain_build<typename decltype(tag)::type>(d, fc, shift); });
  const uint64_t buf_bytes = x * 8 * (uint64_t)d->words;
  if (rc == GMSM_OK && cudaMalloc(&d->d_buf, buf_bytes) != cudaSuccess) rc = set_err(GMSM_ENOMEM, "cudaMalloc(%llu) failed", (unsigned long long)buf_bytes);
  if (rc != GMSM_OK) { cudaFree(d->d_tw); cudaFree(d->d_tw_inv); cudaFree(d->d_pw); cudaFree(d->d_buf); delete d; return nullptr; }
  return d;
}

extern "C" void gmsm_fft_domain_free(gmsm_fft_domain_t* d) {
  if (!d) return;
  cudaSetDevice(d->device);
  cudaFree(d->d_tw); cudaFree(d->d_tw_inv); cudaFree(d->d_pw); cudaFree(d->d_buf);
  delete d;
}

extern "C" size_t gmsm_fft_fr_bytes(int fr_field) {
  if (!fr_consts(fr_field)) return 0;   // (with_fr would set an error)
  return (size_t)with_fr(fr_field, [](auto tag) { return (int)sizeof(Fp<typename decltype(tag)::type>); });
}

extern "C" uint64_t gmsm_fft_domain_cardinality(const gmsm_fft_domain_t* d) { return d ? d->n : 0; }

extern "C" int gmsm_fft_domain_constants(const gmsm_fft_domain_t* d, uint64_t* out) {
  if (!d) return set_err(GMSM_EINVAL, "null domain");
  for (int k = 0; k < 5; k++) memcpy(out + k * d->words, d->consts[k], 8 * (size_t)d->words);   // 5 x words limbs
  return GMSM_OK;
}

// unlocked dispatcher: callers hold d->mu
static int fft_dispatch(gmsm_fft_domain_t* d, void* d_a, int inverse, int decimation, int coset, cudaStream_t st) {
  CK(cudaSetDevice(d->device));
  return with_fr(d->field, [&](auto tag) { return run_fft<typename decltype(tag)::type>(d, d_a, inverse, decimation, coset, st); });
}

extern "C" int gmsm_fft_device(gmsm_fft_domain_t* d, void* d_a, size_t n, int inverse, int decimation, int coset, void* stream) {
  if (!d) return set_err(GMSM_EINVAL, "null domain");
  if (n != d->n) return set_err(GMSM_EINVAL, "len(a) = %zu must equal the domain cardinality %llu", n, (unsigned long long)d->n);
  if (decimation != 0 && decimation != 1) return set_err(GMSM_EINVAL, "not implemented");  // fft.go:108
  std::lock_guard<std::mutex> lk(d->mu);
  return fft_dispatch(d, d_a, inverse, decimation, coset, (cudaStream_t)stream);
}

// host vector in, host vector out: the domain's staging buffer d_buf is shared by all callers, so the domain mutex is held
// across the whole H2D -> transform -> D2H sequence (two concurrent calls used to interleave on the buffer)
static int fft_host(gmsm_fft_domain_t* d, uint64_t* a, size_t n, int inverse, int decimation, int coset) {
  if (!d) return set_err(GMSM_EINVAL, "null domain");
  if (n != d->n) return set_err(GMSM_EINVAL, "len(a) = %zu must equal the domain cardinality %llu", n, (unsigned long long)d->n);
  if (decimation != 0 && decimation != 1) return set_err(GMSM_EINVAL, "not implemented");  // fft.go:108
  std::lock_guard<std::mutex> lk(d->mu);
  CK(cudaSetDevice(d->device));
  const size_t bytes = n * 8 * (size_t)d->words;
  CK(cudaMemcpy(d->d_buf, a, bytes, cudaMemcpyHostToDevice));
  if (int rc = fft_dispatch(d, d->d_buf, inverse, decimation, coset, nullptr)) return rc;
  CK(cudaMemcpy(a, d->d_buf, bytes, cudaMemcpyDeviceToHost));
  return GMSM_OK;
}
extern "C" int gmsm_fft(gmsm_fft_domain_t* d, uint64_t* a, size_t n, int decimation, int coset) { return fft_host(d, a, n, 0, decimation, coset); }
extern "C" int gmsm_fft_inverse(gmsm_fft_domain_t* d, uint64_t* a, size_t n, int decimation, int coset) { return fft_host(d, a, n, 1, decimation, coset); }

extern "C" int gmsm_fft_bit_reverse_device(gmsm_fft_domain_t* d, void* d_a, size_t n, void* stream) {
  if (!d) return set_err(GMSM_EINVAL, "null domain");
  if (n != d->n) return set_err(GMSM_EINVAL, "len(a) must be the domain cardinality");
  std::lock_guard<std::mutex> lk(d->mu);
  CK(cudaSetDevice(d->device));
  unsigned blocks = (unsigned)std::min<uint64_t>((n + 255) / 256, GMSM_NUM_SMS * 32u);
  return with_fr(d->field, [&](auto tag) -> int {
    using P = typename decltype(tag)::type;
    k_fft_bit_reverse<P><<<blocks, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<Fp<P>*>(d_a), n, d->logn);
    CK(cudaGetLastError());
    return GMSM_OK;
  });
}

// ---- Fr polynomial steps of a KZG opening (kzg.go:55-63, 567-582, 302-319) on device vectors ----

extern "C" size_t gmsm_fr_poly_workspace_bytes(int fr_field, size_t n) {
  if (!gmsm_fft_fr_bytes(fr_field) || n == 0) return 0;
  size_t bytes = 0;
  with_fr(fr_field, [&](auto tag) {
    using P = typename decltype(tag)::type;
    bytes = poly_levels(n, poly_log_l<P>() + poly_log_b<P>()).work * sizeof(Fp<P>);
    return GMSM_OK;
  });
  return bytes;
}

extern "C" int gmsm_fr_poly_div_x_minus_a_device(int fr_field, const void* d_f, size_t n, const uint64_t* a, void* d_h, void* d_fa,
                                                 void* d_work, void* stream) {
  const size_t fb = gmsm_fft_fr_bytes(fr_field);
  if (!fb) return set_err(GMSM_EINVAL, "unknown scalar field %d", fr_field);
  if (n == 0) return set_err(GMSM_EINVAL, "empty polynomial (n = 0)");
  if (!d_f || !a || !d_fa) return set_err(GMSM_EINVAL, "null polynomial, point or value pointer");
  if (d_h) {
    const uintptr_t f0 = (uintptr_t)d_f, f1 = f0 + n * fb, h0 = (uintptr_t)d_h, h1 = h0 + (n - 1) * fb;
    if (h0 < f1 && f0 < h1) return set_err(GMSM_EINVAL, "the quotient must not overlap the polynomial");
  }
  if (!d_work && gmsm_fr_poly_workspace_bytes(fr_field, n)) return set_err(GMSM_EINVAL, "null workspace (gmsm_fr_poly_workspace_bytes)");
  return with_fr(fr_field, [&](auto tag) -> int {
    using P = typename decltype(tag)::type;
    using F = Fp<P>;
    F av;
    memcpy(av.l, a, sizeof(F));
    if (!fp_is_reduced(av)) return set_err(GMSM_EINVAL, "the point is not a reduced fr.Element");
    constexpr int log_l = poly_log_l<P>(), log_b = poly_log_b<P>();
    if (((n - 1) >> (log_l + log_b)) >= 0x7fffffffull) return set_err(GMSM_EINVAL, "polynomial too large (n = %zu)", n);
    const size_t smem = poly_smem_bytes<P>(log_l, log_b);
    cudaStream_t st = (cudaStream_t)stream;
    poly_div_schedule<P>(
        reinterpret_cast<const F*>(d_f), n, av, reinterpret_cast<F*>(d_h), reinterpret_cast<F*>(d_fa), reinterpret_cast<F*>(d_work),
        log_l, log_b,
        [&](const F* x, uint64_t m, const PolyMults<P>& mu, F* heads, uint64_t tiles) {
          k_poly_heads<P><<<(unsigned)tiles, 1u << log_b, smem, st>>>(x, m, mu, log_l, heads);
        },
        [&](const F* x, uint64_t m, const PolyMults<P>& mu, const F* carry, F* out, int shift, F* fa, uint64_t tiles) {
          k_poly_write<P><<<(unsigned)tiles, 1u << log_b, smem, st>>>(x, m, mu, log_l, carry, out, shift, fa);
        });
    CK(cudaGetLastError());
    return GMSM_OK;
  });
}

// launch(batch, accumulate, strided) of poly_lincomb_schedule: k_poly_fold over d_out[0, out_len) on `stream`
template <class P>
auto poly_fold_launcher(void* d_out, size_t out_len, void* stream) {
  const unsigned blocks = (unsigned)std::min<uint64_t>((out_len + 255) / 256, GMSM_NUM_SMS * 32u);
  return [=](const PolyFoldBatch<P>& b, int accumulate, bool strided) {
    Fp<P>* out = reinterpret_cast<Fp<P>*>(d_out);
    if (strided)
      k_poly_fold<P, true><<<blocks, 256, 0, (cudaStream_t)stream>>>(out, out_len, b, accumulate);
    else
      k_poly_fold<P, false><<<blocks, 256, 0, (cudaStream_t)stream>>>(out, out_len, b, accumulate);
  };
}

extern "C" int gmsm_fr_poly_fold_device(int fr_field, const void* const* d_polys, const size_t* lens, size_t k, const uint64_t* gamma,
                                        void* d_out, size_t out_len, void* stream) {
  if (!gmsm_fft_fr_bytes(fr_field)) return set_err(GMSM_EINVAL, "unknown scalar field %d", fr_field);
  if (k == 0 || out_len == 0) return set_err(GMSM_EINVAL, "nothing to fold (k = %zu, out_len = %zu)", k, out_len);
  if (!d_polys || !lens || !gamma || !d_out) return set_err(GMSM_EINVAL, "null argument");
  for (size_t i = 0; i < k; i++)
    if (lens[i] && !d_polys[i]) return set_err(GMSM_EINVAL, "polynomial %zu is null", i);
  return with_fr(fr_field, [&](auto tag) -> int {
    using P = typename decltype(tag)::type;
    using F = Fp<P>;
    F g;
    memcpy(g.l, gamma, sizeof(F));
    if (!fp_is_reduced(g)) return set_err(GMSM_EINVAL, "gamma is not a reduced fr.Element");
    std::vector<uint64_t> len(lens, lens + k);
    const auto launch = poly_fold_launcher<P>(d_out, out_len, stream);
    poly_fold_schedule<P>(reinterpret_cast<const F* const*>(d_polys), len.data(), k, g,
                          [&](const PolyFoldBatch<P>& b, int accumulate) { launch(b, accumulate, false); });
    CK(cudaGetLastError());
    return GMSM_OK;
  });
}

extern "C" int gmsm_fr_poly_lincomb_device(int fr_field, const void* const* d_polys, const size_t* lens, const uint64_t* scalars,
                                           const size_t* strides, const size_t* offsets, size_t k, void* d_out, size_t out_len,
                                           int accumulate, void* stream) {
  const size_t fb = gmsm_fft_fr_bytes(fr_field);
  if (!fb) return set_err(GMSM_EINVAL, "unknown scalar field %d", fr_field);
  if (k == 0 || out_len == 0) return set_err(GMSM_EINVAL, "nothing to combine (k = %zu, out_len = %zu)", k, out_len);
  if (!d_polys || !lens || !scalars || !strides || !offsets || !d_out) return set_err(GMSM_EINVAL, "null argument");
  const uintptr_t o0 = (uintptr_t)d_out, o1 = o0 + out_len * fb;
  for (size_t i = 0; i < k; i++) {
    if (strides[i] == 0) return set_err(GMSM_EINVAL, "stride of polynomial %zu is 0", i);
    if (!lens[i]) continue;
    if (!d_polys[i]) return set_err(GMSM_EINVAL, "polynomial %zu is null", i);
    const uintptr_t p0 = (uintptr_t)d_polys[i], p1 = p0 + lens[i] * fb;
    if (p0 < o1 && o0 < p1) return set_err(GMSM_EINVAL, "polynomial %zu overlaps the output", i);
  }
  return with_fr(fr_field, [&](auto tag) -> int {
    using P = typename decltype(tag)::type;
    using F = Fp<P>;
    std::vector<F> s(k);
    for (size_t i = 0; i < k; i++) {
      memcpy(s[i].l, scalars + i * (fb / 8), sizeof(F));
      if (!fp_is_reduced(s[i])) return set_err(GMSM_EINVAL, "scalar %zu is not a reduced fr.Element", i);
    }
    std::vector<uint64_t> len(lens, lens + k), str(strides, strides + k), off(offsets, offsets + k);
    poly_lincomb_schedule<P>(reinterpret_cast<const F* const*>(d_polys), len.data(), s.data(), str.data(), off.data(), k,
                             accumulate ? 1 : 0, poly_fold_launcher<P>(d_out, out_len, stream));
    CK(cudaGetLastError());
    return GMSM_OK;
  });
}

// ---- fr.BatchInvert and the Fr steps of permutation.Prove (permutation.go:52-121) on device vectors ----

namespace {

bool overlaps(const void* a, size_t a_bytes, const void* b, size_t b_bytes) {
  const uintptr_t a0 = (uintptr_t)a, b0 = (uintptr_t)b;
  return a0 < b0 + b_bytes && b0 < a0 + a_bytes;
}

// blocks of the tile inversion kernels (k_fr_batch_invert, k_perm_ratio, k_perm_numerator) over n elements
unsigned perm_inv_tiles(uint64_t n) { return (unsigned)(((n - 1) >> PERM_INV_LOG_T) + 1); }

template <class P>
bool read_reduced(const uint64_t* limbs, Fp<P>* out) {
  memcpy(out->l, limbs, sizeof(Fp<P>));
  return fp_is_reduced(*out);
}

}  // namespace

extern "C" int gmsm_fr_batch_invert_device(int fr_field, const void* d_a, size_t n, void* d_out, void* stream) {
  const size_t fb = gmsm_fft_fr_bytes(fr_field);
  if (!fb) return set_err(GMSM_EINVAL, "unknown scalar field %d", fr_field);
  if (n == 0) return set_err(GMSM_EINVAL, "empty vector (n = 0)");
  if (!d_a || !d_out) return set_err(GMSM_EINVAL, "null vector");
  if (d_out != d_a && overlaps(d_a, n * fb, d_out, n * fb)) return set_err(GMSM_EINVAL, "the output must equal the input or not overlap it");
  if (((n - 1) >> PERM_INV_LOG_T) >= 0x7fffffffull) return set_err(GMSM_EINVAL, "vector too large (n = %zu)", n);
  return with_fr(fr_field, [&](auto tag) -> int {
    using P = typename decltype(tag)::type;
    using F = Fp<P>;
    k_fr_batch_invert<P><<<perm_inv_tiles(n), PERM_INV_THREADS, perm_inv_smem_bytes<P>(PERM_INV_LOG_T), (cudaStream_t)stream>>>(
        reinterpret_cast<const F*>(d_a), n, PERM_INV_LOG_T, reinterpret_cast<F*>(d_out));
    CK(cudaGetLastError());
    return GMSM_OK;
  });
}

extern "C" size_t gmsm_fr_permutation_workspace_bytes(int fr_field, size_t n) {
  return gmsm_fr_poly_workspace_bytes(fr_field, n);   // the carry levels of the prefix product: the tile shape of the opening scan
}

extern "C" int gmsm_fr_permutation_accumulate_device(int fr_field, const void* d_t1, const void* d_t2, size_t n, const uint64_t* epsilon,
                                                     void* d_z, void* d_work, void* stream) {
  const size_t fb = gmsm_fft_fr_bytes(fr_field);
  if (!fb) return set_err(GMSM_EINVAL, "unknown scalar field %d", fr_field);
  if (n == 0 || (n & (n - 1))) return set_err(GMSM_EINVAL, "n (%zu) must be a power of 2", n);
  if (!d_t1 || !d_t2 || !d_z || !epsilon) return set_err(GMSM_EINVAL, "null vector or epsilon");
  if (overlaps(d_z, n * fb, d_t1, n * fb) || overlaps(d_z, n * fb, d_t2, n * fb)) return set_err(GMSM_EINVAL, "z must not overlap t1 or t2");
  if (!d_work && gmsm_fr_permutation_workspace_bytes(fr_field, n))
    return set_err(GMSM_EINVAL, "null workspace (gmsm_fr_permutation_workspace_bytes)");
  if (((n - 1) >> PERM_INV_LOG_T) >= 0x7fffffffull) return set_err(GMSM_EINVAL, "vector too large (n = %zu)", n);
  return with_fr(fr_field, [&](auto tag) -> int {
    using P = typename decltype(tag)::type;
    using F = Fp<P>;
    F eps;
    if (!read_reduced(epsilon, &eps)) return set_err(GMSM_EINVAL, "epsilon is not a reduced fr.Element");
    cudaStream_t st = (cudaStream_t)stream;
    F* z = reinterpret_cast<F*>(d_z);
    k_perm_ratio<P><<<perm_inv_tiles(n), PERM_INV_THREADS, perm_inv_smem_bytes<P>(PERM_INV_LOG_T), st>>>(
        reinterpret_cast<const F*>(d_t1), reinterpret_cast<const F*>(d_t2), n, eps, PERM_INV_LOG_T, z);
    constexpr int log_l = poly_log_l<P>(), log_b = poly_log_b<P>();
    const size_t smem = poly_smem_bytes<P>(log_l, log_b);
    perm_prefix_schedule<P>(
        z, n, reinterpret_cast<F*>(d_work), log_l, log_b,
        [&](const F* x, uint64_t m, F* heads, uint64_t tiles) {
          k_perm_prod_heads<P><<<(unsigned)tiles, 1u << log_b, smem, st>>>(x, m, log_l, heads);
        },
        [&](F* x, uint64_t m, const F* carry, uint64_t tiles) {
          k_perm_prod_write<P><<<(unsigned)tiles, 1u << log_b, smem, st>>>(x, m, log_l, carry);
        });
    // natural order -> the bit-reversed layout of the reference
    int logn = 0;
    while (((uint64_t)1 << logn) < n) logn++;
    k_fft_bit_reverse<P><<<(unsigned)std::min<uint64_t>((n + 255) / 256, GMSM_NUM_SMS * 32u), 256, 0, st>>>(z, n, logn);
    CK(cudaGetLastError());
    return GMSM_OK;
  });
}

extern "C" int gmsm_fft_permutation_numerator_device(gmsm_fft_domain_t* d, const void* d_lt1, const void* d_lt2, const void* d_lz, size_t n,
                                                     const uint64_t* epsilon, const uint64_t* omega, void* d_out, void* stream) {
  if (!d) return set_err(GMSM_EINVAL, "null domain");
  if (n != d->n) return set_err(GMSM_EINVAL, "len(a) = %zu must equal the domain cardinality %llu", n, (unsigned long long)d->n);
  if (!d_lt1 || !d_lt2 || !d_lz || !d_out || !epsilon || !omega) return set_err(GMSM_EINVAL, "null vector or challenge");
  const size_t bytes = n * 8 * (size_t)d->words;
  if (overlaps(d_out, bytes, d_lt1, bytes) || overlaps(d_out, bytes, d_lt2, bytes) || overlaps(d_out, bytes, d_lz, bytes))
    return set_err(GMSM_EINVAL, "the output must not overlap lt1, lt2 or lz");
  std::lock_guard<std::mutex> lk(d->mu);
  CK(cudaSetDevice(d->device));
  return with_fr(d->field, [&](auto tag) -> int {
    using P = typename decltype(tag)::type;
    using F = Fp<P>;
    PermNumConsts<P> k;
    if (!read_reduced(epsilon, &k.eps)) return set_err(GMSM_EINVAL, "epsilon is not a reduced fr.Element");
    if (!read_reduced(omega, &k.omega)) return set_err(GMSM_EINVAL, "omega is not a reduced fr.Element");
    memcpy(k.g.l, d->consts[3], sizeof(F));
    k.tn_inv = fp_inv(fp_sub(host_pow2k(k.g, d->logn), F::one()));   // (g^n - 1)^-1, permutation.go:208
    k_perm_numerator<P><<<perm_inv_tiles(n), PERM_INV_THREADS, perm_inv_smem_bytes<P>(PERM_INV_LOG_T), (cudaStream_t)stream>>>(
        reinterpret_cast<const F*>(d_lt1), reinterpret_cast<const F*>(d_lt2), reinterpret_cast<const F*>(d_lz), n, d->logn, k,
        reinterpret_cast<const F*>(d->d_tw), PERM_INV_LOG_T, reinterpret_cast<F*>(d_out));
    CK(cudaGetLastError());
    return GMSM_OK;
  });
}

// ---- sort.Sort(fr.Vector) and the Fr steps of plookup.ProveLookupVector (vector.go:52-335) on device vectors ----

extern "C" size_t gmsm_fr_sort_workspace_bytes(int fr_field, size_t n) {
  if (!gmsm_fft_fr_bytes(fr_field) || n == 0) return 0;
  size_t bytes = 0;
  with_fr(fr_field, [&](auto tag) {
    using P = typename decltype(tag)::type;
    bytes = sort_layout<P>(n, SORT_LOG_R, SORT_LOG_B).bytes;
    return GMSM_OK;
  });
  return bytes;
}

extern "C" int gmsm_fr_sort_device(int fr_field, const void* d_in, size_t n, void* d_out, void* d_work, void* stream) {
  const size_t fb = gmsm_fft_fr_bytes(fr_field);
  if (!fb) return set_err(GMSM_EINVAL, "unknown scalar field %d", fr_field);
  if (n == 0) return set_err(GMSM_EINVAL, "empty vector (n = 0)");
  if (!d_in || !d_out) return set_err(GMSM_EINVAL, "null vector");
  if (!d_work) return set_err(GMSM_EINVAL, "null workspace (gmsm_fr_sort_workspace_bytes)");
  if (n >= 0x80000000ull) return set_err(GMSM_EINVAL, "vector too large (n = %zu)", n);
  if (d_out != d_in && overlaps(d_in, n * fb, d_out, n * fb)) return set_err(GMSM_EINVAL, "the output must equal the input or not overlap it");
  const size_t wb = gmsm_fr_sort_workspace_bytes(fr_field, n);
  if (overlaps(d_work, wb, d_in, n * fb) || overlaps(d_work, wb, d_out, n * fb))
    return set_err(GMSM_EINVAL, "the workspace must not overlap the input or the output");
  return with_fr(fr_field, [&](auto tag) -> int {
    using P = typename decltype(tag)::type;
    using F = Fp<P>;
    cudaStream_t st = (cudaStream_t)stream;
    int err = GMSM_OK;
    fr_sort_schedule<P>(
        reinterpret_cast<const F*>(d_in), n, reinterpret_cast<F*>(d_out), reinterpret_cast<unsigned char*>(d_work), SORT_LOG_R, SORT_LOG_B,
        [&](auto kernel, unsigned grid, unsigned block, auto... args) { kernel<<<grid, block, 0, st>>>(args...); },
        [&](uint32_t* host, const uint32_t* dev, int words) {   // which byte positions vary decides the passes: one small copy
          if (err == GMSM_OK && (cudaMemcpyAsync(host, dev, words * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
                                 cudaStreamSynchronize(st) != cudaSuccess))
            err = set_err(GMSM_ECUDA, "reading the sort's difference mask: %s", cudaGetErrorString(cudaGetLastError()));
          if (err != GMSM_OK) memset(host, 0, words * 4);
        });
    if (err != GMSM_OK) return err;
    CK(cudaGetLastError());
    return GMSM_OK;
  });
}

extern "C" int gmsm_fr_plookup_accumulate_device(int fr_field, const void* d_f, const void* d_t, const void* d_h1, const void* d_h2,
                                                 size_t n, const uint64_t* beta, const uint64_t* gamma, void* d_z, void* d_work,
                                                 void* stream) {
  const size_t fb = gmsm_fft_fr_bytes(fr_field);
  if (!fb) return set_err(GMSM_EINVAL, "unknown scalar field %d", fr_field);
  if (n == 0) return set_err(GMSM_EINVAL, "empty vector (n = 0)");
  if (!d_f || !d_t || !d_h1 || !d_h2 || !d_z || !beta || !gamma) return set_err(GMSM_EINVAL, "null vector or challenge");
  const size_t bytes = n * fb;
  for (const void* in : {d_f, d_t, d_h1, d_h2})
    if (overlaps(d_z, bytes, in, bytes)) return set_err(GMSM_EINVAL, "z must not overlap f, t, h1 or h2");
  if (!d_work && gmsm_fr_permutation_workspace_bytes(fr_field, n))
    return set_err(GMSM_EINVAL, "null workspace (gmsm_fr_permutation_workspace_bytes)");
  if (((n - 1) >> PERM_INV_LOG_T) >= 0x7fffffffull) return set_err(GMSM_EINVAL, "vector too large (n = %zu)", n);
  return with_fr(fr_field, [&](auto tag) -> int {
    using P = typename decltype(tag)::type;
    using F = Fp<P>;
    PlookupConsts<P> k;
    if (!read_reduced(beta, &k.beta)) return set_err(GMSM_EINVAL, "beta is not a reduced fr.Element");
    if (!read_reduced(gamma, &k.gamma)) return set_err(GMSM_EINVAL, "gamma is not a reduced fr.Element");
    k.opb = fp_add(F::one(), k.beta);
    k.gopb = fp_mul(k.gamma, k.opb);
    cudaStream_t st = (cudaStream_t)stream;
    F* z = reinterpret_cast<F*>(d_z);
    k_plookup_ratio<P><<<perm_inv_tiles(n), PERM_INV_THREADS, perm_inv_smem_bytes<P>(PERM_INV_LOG_T), st>>>(
        reinterpret_cast<const F*>(d_f), reinterpret_cast<const F*>(d_t), reinterpret_cast<const F*>(d_h1), reinterpret_cast<const F*>(d_h2),
        n, k, PERM_INV_LOG_T, z);
    constexpr int log_l = poly_log_l<P>(), log_b = poly_log_b<P>();
    const size_t smem = poly_smem_bytes<P>(log_l, log_b);
    perm_prefix_schedule<P>(
        z, n, reinterpret_cast<F*>(d_work), log_l, log_b,
        [&](const F* x, uint64_t m, F* heads, uint64_t tiles) {
          k_perm_prod_heads<P><<<(unsigned)tiles, 1u << log_b, smem, st>>>(x, m, log_l, heads);
        },
        [&](F* x, uint64_t m, const F* carry, uint64_t tiles) {
          k_perm_prod_write<P><<<(unsigned)tiles, 1u << log_b, smem, st>>>(x, m, log_l, carry);
        });
    CK(cudaGetLastError());
    return GMSM_OK;
  });
}

extern "C" int gmsm_fft_plookup_numerator_device(gmsm_fft_domain_t* d, const void* d_lz, const void* d_lh1, const void* d_lh2,
                                                 const void* d_lt, const void* d_lf, size_t n, const uint64_t* beta, const uint64_t* gamma,
                                                 const uint64_t* alpha, void* d_out, void* stream) {
  if (!d) return set_err(GMSM_EINVAL, "null domain");
  if (n != d->n) return set_err(GMSM_EINVAL, "len(a) = %zu must equal the domain cardinality %llu", n, (unsigned long long)d->n);
  if (!d_lz || !d_lh1 || !d_lh2 || !d_lt || !d_lf || !d_out || !beta || !gamma || !alpha)
    return set_err(GMSM_EINVAL, "null vector or challenge");
  const size_t bytes = n * 8 * (size_t)d->words;
  for (const void* in : {d_lz, d_lh1, d_lh2, d_lt, d_lf})
    if (overlaps(d_out, bytes, in, bytes)) return set_err(GMSM_EINVAL, "the output must not overlap lz, lh1, lh2, lt or lf");
  std::lock_guard<std::mutex> lk(d->mu);
  CK(cudaSetDevice(d->device));
  return with_fr(d->field, [&](auto tag) -> int {
    using P = typename decltype(tag)::type;
    using F = Fp<P>;
    PlookupNumConsts<P> k;
    if (!read_reduced(beta, &k.c.beta)) return set_err(GMSM_EINVAL, "beta is not a reduced fr.Element");
    if (!read_reduced(gamma, &k.c.gamma)) return set_err(GMSM_EINVAL, "gamma is not a reduced fr.Element");
    if (!read_reduced(alpha, &k.alpha)) return set_err(GMSM_EINVAL, "alpha is not a reduced fr.Element");
    k.c.opb = fp_add(F::one(), k.c.beta);
    k.c.gopb = fp_mul(k.c.gamma, k.c.opb);
    memcpy(k.shift.l, d->consts[3], sizeof(F));
    // gg = (w^2)^(s-1) = w^(n-2) = w^-2 (vector.go:124-126); x^s on the coset is shift^s (-1)^i (vector.go:165-181)
    F winv;
    memcpy(winv.l, d->consts[1], sizeof(F));
    k.gg = fp_sqr(winv);
    const F ss = d->logn ? host_pow2k(k.shift, d->logn - 1) : k.shift;   // shift^(n/2)
    k.xs_inv[0] = fp_inv(fp_sub(ss, F::one()));
    k.xs_inv[1] = fp_inv(fp_neg(fp_add(ss, F::one())));
    k_plookup_numerator<P><<<perm_inv_tiles(n), PERM_INV_THREADS, perm_inv_smem_bytes<P>(PERM_INV_LOG_T), (cudaStream_t)stream>>>(
        reinterpret_cast<const F*>(d_lz), reinterpret_cast<const F*>(d_lh1), reinterpret_cast<const F*>(d_lh2), reinterpret_cast<const F*>(d_lt),
        reinterpret_cast<const F*>(d_lf), n, d->logn, k, reinterpret_cast<const F*>(d->d_tw), PERM_INV_LOG_T, reinterpret_cast<F*>(d_out));
    CK(cudaGetLastError());
    return GMSM_OK;
  });
}

// ---- the O(n) steps of the iop package (ratios.go, polynomial.go:204-241, expressions.go, quotient.go) on device vectors ----

namespace {

int tz64(uint64_t n) {   // bits.TrailingZeros of n > 0
  int t = 0;
  while (!((n >> t) & 1ull)) t++;
  return t;
}

// the iop workspace: the prefix product's carry levels or the tile sums of the Lagrange evaluation, then one u32 flag
template <class P>
size_t iop_flag_offset(uint64_t n) {
  const size_t scan = poly_levels(n, poly_log_l<P>() + poly_log_b<P>()).work * sizeof(Fp<P>);
  const size_t sums = (size_t)perm_inv_tiles(n) * sizeof(Fp<P>);
  return ((scan > sums ? scan : sums) + 15) & ~(size_t)15;
}

template <class P>
void iop_prefix(Fp<P>* z, uint64_t n, Fp<P>* work, cudaStream_t st) {
  constexpr int log_l = poly_log_l<P>(), log_b = poly_log_b<P>();
  const size_t smem = poly_smem_bytes<P>(log_l, log_b);
  perm_prefix_schedule<P>(
      z, n, work, log_l, log_b,
      [&](const Fp<P>* x, uint64_t m, Fp<P>* heads, uint64_t tiles) {
        k_perm_prod_heads<P><<<(unsigned)tiles, 1u << log_b, smem, st>>>(x, m, log_l, heads);
      },
      [&](Fp<P>* x, uint64_t m, const Fp<P>* carry, uint64_t tiles) {
        k_perm_prod_write<P><<<(unsigned)tiles, 1u << log_b, smem, st>>>(x, m, log_l, carry);
      });
}

// the columns of a ratio builder: non-null, not overlapping the output, at most IOP_MAX_COLUMNS
template <class P>
int iop_columns(const void* const* d_cols, const int* bitrev, size_t k, size_t n, const void* d_z, IopColumns<P>* out) {
  if (k == 0 || k > (size_t)IOP_MAX_COLUMNS) return set_err(GMSM_EINVAL, "%zu polynomials per list (1 to %d are supported)", k, IOP_MAX_COLUMNS);
  if (!d_cols || !bitrev) return set_err(GMSM_EINVAL, "null column list");
  const size_t bytes = n * sizeof(Fp<P>);
  out->k = (int)k;
  out->bitrev = 0;
  for (size_t c = 0; c < k; c++) {
    if (!d_cols[c]) return set_err(GMSM_EINVAL, "polynomial %zu is null", c);
    if (overlaps(d_z, bytes, d_cols[c], bytes)) return set_err(GMSM_EINVAL, "the output must not overlap polynomial %zu", c);
    out->p[c] = reinterpret_cast<const Fp<P>*>(d_cols[c]);
    if (bitrev[c]) out->bitrev |= 1u << c;
  }
  return GMSM_OK;
}

}  // namespace

extern "C" size_t gmsm_fr_iop_workspace_bytes(int fr_field, size_t n) {
  if (!gmsm_fft_fr_bytes(fr_field) || n == 0) return 0;
  size_t bytes = 0;
  with_fr(fr_field, [&](auto tag) {
    bytes = iop_flag_offset<typename decltype(tag)::type>(n) + 16;
    return GMSM_OK;
  });
  return bytes;
}

extern "C" int gmsm_fr_iop_ratio_shuffled_device(int fr_field, const void* const* d_num, const int* num_bitrev, const void* const* d_den,
                                                 const int* den_bitrev, size_t k, size_t n, const uint64_t* beta, void* d_z, void* d_work,
                                                 void* stream) {
  if (!gmsm_fft_fr_bytes(fr_field)) return set_err(GMSM_EINVAL, "unknown scalar field %d", fr_field);
  if (n == 0 || (n & (n - 1))) return set_err(GMSM_EINVAL, "n (%zu) must be a power of 2", n);
  if (!d_z || !beta || !d_work) return set_err(GMSM_EINVAL, "null output, beta or workspace (gmsm_fr_iop_workspace_bytes)");
  if (((n - 1) >> PERM_INV_LOG_T) >= 0x7fffffffull) return set_err(GMSM_EINVAL, "vector too large (n = %zu)", n);
  return with_fr(fr_field, [&](auto tag) -> int {
    using P = typename decltype(tag)::type;
    using F = Fp<P>;
    IopColumns<P> num, den;
    if (int rc = iop_columns<P>(d_num, num_bitrev, k, n, d_z, &num)) return rc;
    if (int rc = iop_columns<P>(d_den, den_bitrev, k, n, d_z, &den)) return rc;
    F b;
    if (!read_reduced(beta, &b)) return set_err(GMSM_EINVAL, "beta is not a reduced fr.Element");
    cudaStream_t st = (cudaStream_t)stream;
    F* z = reinterpret_cast<F*>(d_z);
    k_iop_ratio_shuffled<P><<<perm_inv_tiles(n), PERM_INV_THREADS, perm_inv_smem_bytes<P>(PERM_INV_LOG_T), st>>>(num, den, n, tz64(n), b,
                                                                                                                   PERM_INV_LOG_T, z);
    iop_prefix<P>(z, n, reinterpret_cast<F*>(d_work), st);
    CK(cudaGetLastError());
    return GMSM_OK;
  });
}

extern "C" int gmsm_fft_iop_ratio_copy_device(gmsm_fft_domain_t* d, const void* const* d_cols, const int* bitrev, size_t k, size_t n,
                                              const int64_t* d_sigma, const uint64_t* beta, const uint64_t* gamma, void* d_z, void* d_work,
                                              void* stream) {
  if (!d) return set_err(GMSM_EINVAL, "null domain");
  if (n != d->n) return set_err(GMSM_EINVAL, "len(a) = %zu must equal the domain cardinality %llu", n, (unsigned long long)d->n);
  if (!d_z || !beta || !gamma || !d_sigma || !d_work) return set_err(GMSM_EINVAL, "null output, permutation, challenge or workspace");
  if (((n - 1) >> PERM_INV_LOG_T) >= 0x7fffffffull) return set_err(GMSM_EINVAL, "vector too large (n = %zu)", n);
  std::lock_guard<std::mutex> lk(d->mu);
  CK(cudaSetDevice(d->device));
  return with_fr(d->field, [&](auto tag) -> int {
    using P = typename decltype(tag)::type;
    using F = Fp<P>;
    IopColumns<P> cols;
    if (int rc = iop_columns<P>(d_cols, bitrev, k, n, d_z, &cols)) return rc;
    if (overlaps(d_z, n * sizeof(F), d_sigma, k * n * 8)) return set_err(GMSM_EINVAL, "the output must not overlap the permutation");
    IopCopyConsts<P> kc;
    F b, g;
    if (!read_reduced(beta, &b)) return set_err(GMSM_EINVAL, "beta is not a reduced fr.Element");
    if (!read_reduced(gamma, &kc.gamma)) return set_err(GMSM_EINVAL, "gamma is not a reduced fr.Element");
    memcpy(g.l, d->consts[3], sizeof(F));
    for (size_t c = 0; c < k; c++) {
      kc.p[c] = cols.p[c];
      kc.bg[c] = b;
      b = fp_mul(b, g);
    }
    kc.bitrev = cols.bitrev;
    kc.k = (int)k;
    cudaStream_t st = (cudaStream_t)stream;
    // an index outside [0, k n) (a panic in the reference) is refused before the output is written: one flag read back
    uint32_t* flag = reinterpret_cast<uint32_t*>(reinterpret_cast<unsigned char*>(d_work) + iop_flag_offset<P>(n));
    CK(cudaMemsetAsync(flag, 0, 4, st));
    const uint64_t m = (uint64_t)k * n;
    k_iop_check_sigma<<<(unsigned)std::min<uint64_t>((m + 255) / 256, GMSM_NUM_SMS * 32u), 256, 0, st>>>(d_sigma, m, (int64_t)m, flag);
    uint32_t bad = 0;
    CK(cudaMemcpyAsync(&bad, flag, 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (bad) return set_err(GMSM_EINVAL, "the permutation has an entry outside [0, %llu)", (unsigned long long)m);
    F* z = reinterpret_cast<F*>(d_z);
    k_iop_ratio_copy<P><<<perm_inv_tiles(n), PERM_INV_THREADS, perm_inv_smem_bytes<P>(PERM_INV_LOG_T), st>>>(
        kc, d_sigma, n, d->logn, reinterpret_cast<const F*>(d->d_tw), PERM_INV_LOG_T, z);
    iop_prefix<P>(z, n, reinterpret_cast<F*>(d_work), st);
    CK(cudaGetLastError());
    return GMSM_OK;
  });
}

extern "C" int gmsm_fft_iop_lagrange_eval_device(gmsm_fft_domain_t* d, const void* d_c, size_t n, int bitrev, const uint64_t* x,
                                                 void* d_out, void* d_work, void* stream) {
  if (!d) return set_err(GMSM_EINVAL, "null domain");
  if (n != d->n) return set_err(GMSM_EINVAL, "len(a) = %zu must equal the domain cardinality %llu", n, (unsigned long long)d->n);
  if (!d_c || !x || !d_out || !d_work) return set_err(GMSM_EINVAL, "null vector, point, output or workspace");
  if (((n - 1) >> PERM_INV_LOG_T) >= 0x7fffffffull) return set_err(GMSM_EINVAL, "vector too large (n = %zu)", n);
  std::lock_guard<std::mutex> lk(d->mu);
  CK(cudaSetDevice(d->device));
  return with_fr(d->field, [&](auto tag) -> int {
    using P = typename decltype(tag)::type;
    using F = Fp<P>;
    F xv, ci;
    if (!read_reduced(x, &xv)) return set_err(GMSM_EINVAL, "the point is not a reduced fr.Element");
    memcpy(ci.l, d->consts[2], sizeof(F));
    const F scale = fp_mul(fp_sub(host_pow2k(xv, d->logn), F::one()), ci);   // (x^n - 1) / n
    cudaStream_t st = (cudaStream_t)stream;
    F* partial = reinterpret_cast<F*>(d_work);
    const unsigned tiles = perm_inv_tiles(n);
    k_iop_lagrange_terms<P><<<tiles, PERM_INV_THREADS, perm_inv_smem_bytes<P>(PERM_INV_LOG_T), st>>>(
        reinterpret_cast<const F*>(d_c), n, d->logn, bitrev, xv, reinterpret_cast<const F*>(d->d_tw), PERM_INV_LOG_T, partial);
    k_iop_sum<P><<<1, 256, 256 * sizeof(F), st>>>(partial, tiles, scale, reinterpret_cast<F*>(d_out));
    CK(cudaGetLastError());
    return GMSM_OK;
  });
}

extern "C" int gmsm_fr_iop_evaluate_device(int fr_field, const uint32_t* code, size_t len, size_t out_reg, const uint64_t* consts,
                                           size_t nconsts, const void* const* d_inputs, const uint64_t* offsets, const int* bitrev, size_t m,
                                           size_t n, int out_bitrev, void* d_r, void* stream) {
  const size_t fb = gmsm_fft_fr_bytes(fr_field);
  if (!fb) return set_err(GMSM_EINVAL, "unknown scalar field %d", fr_field);
  if (n == 0) return set_err(GMSM_EINVAL, "empty vector (n = 0)");
  if (len == 0 || len > (size_t)IOP_MAX_PROGRAM) return set_err(GMSM_EINVAL, "program of %zu instructions (1 to %d)", len, IOP_MAX_PROGRAM);
  if (out_reg >= (size_t)IOP_MAX_REGISTERS) return set_err(GMSM_EINVAL, "result register %zu (at most %d registers)", out_reg, IOP_MAX_REGISTERS);
  if (nconsts > (size_t)IOP_MAX_CONSTS) return set_err(GMSM_EINVAL, "%zu constants (at most %d)", nconsts, IOP_MAX_CONSTS);
  if (m > (size_t)IOP_MAX_INPUTS) return set_err(GMSM_EINVAL, "%zu inputs (at most %d)", m, IOP_MAX_INPUTS);
  if (!code || !d_r || (nconsts && !consts) || (m && (!d_inputs || !offsets || !bitrev))) return set_err(GMSM_EINVAL, "null argument");
  for (size_t pc = 0; pc < len; pc++) {
    const uint32_t w = code[pc], op = w & 0xff, dst = (w >> 8) & 0xff, a = (w >> 16) & 0xff, b = w >> 24;
    const bool ok = dst < (uint32_t)IOP_MAX_REGISTERS &&
                    (op == IOP_OP_INPUT ? a < m : op == IOP_OP_CONST ? a < nconsts : op == IOP_OP_INDEX ? true
                     : op == IOP_OP_NEG ? a < (uint32_t)IOP_MAX_REGISTERS
                     : op <= IOP_OP_MUL && a < (uint32_t)IOP_MAX_REGISTERS && b < (uint32_t)IOP_MAX_REGISTERS);
    if (!ok) return set_err(GMSM_EINVAL, "invalid instruction %zu (0x%08x)", pc, w);
  }
  IopInputs in{};
  in.m = (int)m;
  for (size_t j = 0; j < m; j++) {
    if (!d_inputs[j]) return set_err(GMSM_EINVAL, "input %zu is null", j);
    if (offsets[j] >= n) return set_err(GMSM_EINVAL, "offset of input %zu is not below n", j);
    if (overlaps(d_r, n * fb, d_inputs[j], n * fb)) return set_err(GMSM_EINVAL, "the result must not overlap input %zu", j);
    in.p[j] = d_inputs[j];
    in.off[j] = offsets[j];
    if (bitrev[j]) in.bitrev |= 1u << j;
  }
  return with_fr(fr_field, [&](auto tag) -> int {
    using P = typename decltype(tag)::type;
    using F = Fp<P>;
    IopProgram<P> prog;
    memcpy(prog.code, code, len * 4);
    prog.len = (int)len;
    prog.out = (int)out_reg;
    for (size_t c = 0; c < nconsts; c++)
      if (!read_reduced(consts + c * (fb / 8), &prog.consts[c])) return set_err(GMSM_EINVAL, "constant %zu is not a reduced fr.Element", c);
    k_iop_evaluate<P><<<(unsigned)std::min<uint64_t>((n + 255) / 256, GMSM_NUM_SMS * 32u), 256, 0, (cudaStream_t)stream>>>(
        prog, in, n, tz64(n), out_bitrev, reinterpret_cast<F*>(d_r));
    CK(cudaGetLastError());
    return GMSM_OK;
  });
}

extern "C" int gmsm_fr_iop_divide_by_xn_minus_one_device(int fr_field, const void* d_a, size_t n, uint64_t offset, int bitrev,
                                                         const uint64_t* inv, size_t rho, void* d_out, void* stream) {
  const size_t fb = gmsm_fft_fr_bytes(fr_field);
  if (!fb) return set_err(GMSM_EINVAL, "unknown scalar field %d", fr_field);
  if (n == 0 || (n & (n - 1))) return set_err(GMSM_EINVAL, "n (%zu) must be a power of 2", n);
  if (rho == 0 || (rho & (rho - 1)) || rho > (size_t)IOP_MAX_RHO) return set_err(GMSM_EINVAL, "rho (%zu) must be a power of 2 up to %d", rho, IOP_MAX_RHO);
  if (!d_a || !d_out || !inv) return set_err(GMSM_EINVAL, "null vector or inverse table");
  if (offset >= n) return set_err(GMSM_EINVAL, "offset is not below n");
  if (overlaps(d_a, n * fb, d_out, n * fb)) return set_err(GMSM_EINVAL, "the output must not overlap the input");
  return with_fr(fr_field, [&](auto tag) -> int {
    using P = typename decltype(tag)::type;
    using F = Fp<P>;
    IopXnInv<P> k;
    k.rho = (uint32_t)rho;
    for (size_t j = 0; j < rho; j++)
      if (!read_reduced(inv + j * (fb / 8), &k.inv[j])) return set_err(GMSM_EINVAL, "inverse %zu is not a reduced fr.Element", j);
    k_iop_div_xn_minus_one<P><<<(unsigned)std::min<uint64_t>((n + 255) / 256, GMSM_NUM_SMS * 32u), 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const F*>(d_a), n, tz64(n), offset, bitrev, k, reinterpret_cast<F*>(d_out));
    CK(cudaGetLastError());
    return GMSM_OK;
  });
}

extern "C" int gmsm_fr_bit_reverse_device(int fr_field, void* d_a, size_t n, void* stream) {
  if (!gmsm_fft_fr_bytes(fr_field)) return set_err(GMSM_EINVAL, "unknown scalar field %d", fr_field);
  if (n == 0 || (n & (n - 1))) return set_err(GMSM_EINVAL, "n (%zu) must be a power of 2", n);
  if (!d_a) return set_err(GMSM_EINVAL, "null vector");
  return with_fr(fr_field, [&](auto tag) -> int {
    using P = typename decltype(tag)::type;
    k_fft_bit_reverse<P><<<(unsigned)std::min<uint64_t>((n + 255) / 256, GMSM_NUM_SMS * 32u), 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<Fp<P>*>(d_a), n, tz64(n));
    CK(cudaGetLastError());
    return GMSM_OK;
  });
}

extern "C" int gmsm_fr_generator(int fr_field, uint64_t m, uint64_t* out) {
  const FrConsts* fcp = fr_consts(fr_field);
  if (!fcp) return set_err(GMSM_EINVAL, "unknown scalar field %d", fr_field);
  if (!out) return set_err(GMSM_EINVAL, "null output");
  int logn = 0;
  if (int rc = domain_log(*fcp, m, &logn)) return rc;
  return with_fr(fr_field, [&](auto tag) -> int {
    using P = typename decltype(tag)::type;
    const Fp<P> g = host_pow2k(host_from_decimal<P>(fcp->root), fcp->max_order - logn);
    memcpy(out, g.l, sizeof(Fp<P>));
    return GMSM_OK;
  });
}
