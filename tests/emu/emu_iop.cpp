// TEST INFRASTRUCTURE ONLY -- the kernels of the iop package (gnark-crypto_b200/csrc/iop_kernels.cuh) on the CPU for every scalar
// field, launched in the order of fft.cu's gmsm_fr_iop_ratio_shuffled_device, gmsm_fft_iop_ratio_copy_device,
// gmsm_fft_iop_lagrange_eval_device, gmsm_fr_iop_evaluate_device and gmsm_fr_iop_divide_by_xn_minus_one_device (the kernels with
// barriers run on the cooperative launcher).  The tile shapes are parameters, so that short vectors reach several scan levels.
#include <cstring>
#include <vector>

#include "iop_kernels.cuh"

namespace {
constexpr size_t EMU_SMEM = 64 * 1024;
thread_local __attribute__((aligned(16))) unsigned char smem_raw[EMU_SMEM];

template <class P>
bool inv_shape_ok(int log_t, unsigned threads) {
  return log_t >= 0 && perm_inv_smem_bytes<P>(log_t) <= EMU_SMEM && (1u << log_t) <= 32 * threads;
}

int tz(uint64_t n) {
  int t = 0;
  while (!((n >> t) & 1ull)) t++;
  return t;
}

template <class P>
IopColumns<P> columns(const uint32_t* const* cols, const int* bitrev, int k) {
  IopColumns<P> c{};
  c.k = k;
  for (int j = 0; j < k; j++) {
    c.p[j] = reinterpret_cast<const Fp<P>*>(cols[j]);
    if (bitrev[j]) c.bitrev |= 1u << j;
  }
  return c;
}

// the exclusive prefix product of fft.cu's iop_prefix at the given scan shape
template <class P>
void prefix(Fp<P>* z, uint64_t n, int log_l, int log_b) {
  using F = Fp<P>;
  std::vector<F> work(poly_levels(n, log_l + log_b).work + 1);
  const unsigned B = 1u << log_b;
  perm_prefix_schedule<P>(
      z, n, work.data(), log_l, log_b,
      [&](const F* x, uint64_t m, F* heads, uint64_t tiles) { emu_launch_coop(k_perm_prod_heads<P>, dim3((unsigned)tiles), B, x, m, log_l, heads); },
      [&](F* x, uint64_t m, const F* carry, uint64_t tiles) { emu_launch_coop(k_perm_prod_write<P>, dim3((unsigned)tiles), B, x, m, log_l, carry); });
}

template <class P>
bool scan_ok(int log_l, int log_b) {
  return log_b >= 0 && log_b <= POLY_MAX_LOG_B && poly_smem_bytes<P>(log_l, log_b) <= EMU_SMEM;
}

template <class P>
int emu_shuffled(const uint32_t* const* num, const int* num_br, const uint32_t* const* den, const int* den_br, int k, uint64_t n,
                 const uint32_t* beta, uint32_t* z, int log_t, unsigned threads, int log_l, int log_b) {
  if (n == 0 || (n & (n - 1)) || k < 1 || k > IOP_MAX_COLUMNS || !inv_shape_ok<P>(log_t, threads) || !scan_ok<P>(log_l, log_b)) return 1;
  Fp<P> b;
  std::memcpy(b.l, beta, sizeof(b));
  emu_launch_coop(k_iop_ratio_shuffled<P>, dim3((unsigned)(((n - 1) >> log_t) + 1)), threads, columns<P>(num, num_br, k),
                  columns<P>(den, den_br, k), n, tz(n), b, log_t, reinterpret_cast<Fp<P>*>(z));
  prefix<P>(reinterpret_cast<Fp<P>*>(z), n, log_l, log_b);
  return 0;
}

// tw: the n / 2 twiddles w^j; consts: beta, gamma, g (FrMultiplicativeGen).  Returns 3 when sigma has an entry outside [0, k n)
// (z is then not written).
template <class P>
int emu_copy(const uint32_t* const* cols, const int* br, int k, uint64_t n, const int64_t* sigma, const uint32_t* tw, const uint32_t* consts,
             uint32_t* z, int log_t, unsigned threads, int log_l, int log_b) {
  using F = Fp<P>;
  if (n == 0 || (n & (n - 1)) || k < 1 || k > IOP_MAX_COLUMNS || !inv_shape_ok<P>(log_t, threads) || !scan_ok<P>(log_l, log_b)) return 1;
  IopCopyConsts<P> kc{};
  F b, g;
  std::memcpy(b.l, consts, sizeof(F));
  std::memcpy(kc.gamma.l, consts + sizeof(F) / 4, sizeof(F));
  std::memcpy(g.l, consts + 2 * sizeof(F) / 4, sizeof(F));
  const IopColumns<P> c = columns<P>(cols, br, k);
  for (int j = 0; j < k; j++) {
    kc.p[j] = c.p[j];
    kc.bg[j] = b;
    b = fp_mul(b, g);
  }
  kc.bitrev = c.bitrev;
  kc.k = k;
  uint32_t bad = 0;
  emu_launch(k_iop_check_sigma, dim3(3), 32u, sigma, (uint64_t)k * n, (int64_t)k * (int64_t)n, &bad);
  if (bad) return 3;
  emu_launch_coop(k_iop_ratio_copy<P>, dim3((unsigned)(((n - 1) >> log_t) + 1)), threads, kc, sigma, n, tz(n),
                  reinterpret_cast<const F*>(tw), log_t, reinterpret_cast<F*>(z));
  prefix<P>(reinterpret_cast<F*>(z), n, log_l, log_b);
  return 0;
}

// consts: x, (x^n - 1) / n; threads of the tile sums and sum_threads of the final sum must be powers of two
template <class P>
int emu_lagrange(const uint32_t* c, uint64_t n, int bitrev, const uint32_t* tw, const uint32_t* consts, uint32_t* out, int log_t,
                 unsigned threads, unsigned sum_threads) {
  using F = Fp<P>;
  if (n == 0 || (n & (n - 1)) || !inv_shape_ok<P>(log_t, threads) || (threads & (threads - 1)) || threads > (2u << log_t) ||
      !sum_threads || (sum_threads & (sum_threads - 1)) || sum_threads * sizeof(F) > EMU_SMEM)
    return 1;
  F x, scale;
  std::memcpy(x.l, consts, sizeof(F));
  std::memcpy(scale.l, consts + sizeof(F) / 4, sizeof(F));
  const unsigned tiles = (unsigned)(((n - 1) >> log_t) + 1);
  std::vector<F> partial(tiles);
  emu_launch_coop(k_iop_lagrange_terms<P>, dim3(tiles), threads, reinterpret_cast<const F*>(c), n, tz(n), bitrev, x,
                  reinterpret_cast<const F*>(tw), log_t, partial.data());
  emu_launch_coop(k_iop_sum<P>, dim3(1), sum_threads, (const F*)partial.data(), (uint64_t)tiles, scale, reinterpret_cast<F*>(out));
  return 0;
}

template <class P>
int emu_evaluate(const uint32_t* code, int len, int out_reg, const uint32_t* consts, int nconsts, const uint32_t* const* inputs,
                 const uint64_t* offsets, const int* bitrev, int m, uint64_t n, int out_bitrev, uint32_t* r) {
  using F = Fp<P>;
  if (n == 0 || len < 1 || len > IOP_MAX_PROGRAM || nconsts > IOP_MAX_CONSTS || m > IOP_MAX_INPUTS || out_reg >= IOP_MAX_REGISTERS) return 1;
  IopProgram<P> prog{};
  std::memcpy(prog.code, code, 4 * (size_t)len);
  prog.len = len;
  prog.out = out_reg;
  for (int j = 0; j < nconsts; j++) std::memcpy(prog.consts[j].l, consts + j * sizeof(F) / 4, sizeof(F));
  IopInputs in{};
  in.m = m;
  for (int j = 0; j < m; j++) {
    in.p[j] = inputs[j];
    in.off[j] = offsets[j];
    if (bitrev[j]) in.bitrev |= 1u << j;
  }
  emu_launch(k_iop_evaluate<P>, dim3(3), 64u, prog, in, n, tz(n), out_bitrev, reinterpret_cast<F*>(r));
  return 0;
}

template <class P>
int emu_divide(const uint32_t* a, uint64_t n, uint64_t offset, int bitrev, const uint32_t* inv, unsigned rho, uint32_t* out) {
  using F = Fp<P>;
  if (n == 0 || (n & (n - 1)) || !rho || (rho & (rho - 1)) || rho > (unsigned)IOP_MAX_RHO || offset >= n) return 1;
  IopXnInv<P> k{};
  k.rho = rho;
  for (unsigned j = 0; j < rho; j++) std::memcpy(k.inv[j].l, inv + j * sizeof(F) / 4, sizeof(F));
  emu_launch(k_iop_div_xn_minus_one<P>, dim3(3), 64u, reinterpret_cast<const F*>(a), n, tz(n), offset, bitrev, k, reinterpret_cast<F*>(out));
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

// field: GMSM_FR_* (0 bn254 ... 6 bw6-761); elements of fr.Limbs u64 Montgomery limbs.  log_t < 0, threads = 0, log_l < 0, log_b < 0:
// the shapes fft.cu uses for the field.  Returns 0, 1 for a refused shape, or 3 for a sigma entry out of range.
extern "C" int emu_iop_ratio_shuffled(int field, const uint32_t* const* num, const int* num_br, const uint32_t* const* den, const int* den_br,
                                      int k, uint64_t n, const uint32_t* beta, uint32_t* z, int log_t, unsigned threads, int log_l, int log_b) {
  return with_field(field, [&](auto p) {
    using P = decltype(p);
    return emu_shuffled<P>(num, num_br, den, den_br, k, n, beta, z, log_t < 0 ? PERM_INV_LOG_T : log_t, threads ? threads : PERM_INV_THREADS,
                           log_l < 0 ? poly_log_l<P>() : log_l, log_b < 0 ? poly_log_b<P>() : log_b);
  });
}

extern "C" int emu_iop_ratio_copy(int field, const uint32_t* const* cols, const int* br, int k, uint64_t n, const int64_t* sigma, const uint32_t* tw,
                                  const uint32_t* consts, uint32_t* z, int log_t, unsigned threads, int log_l, int log_b) {
  return with_field(field, [&](auto p) {
    using P = decltype(p);
    return emu_copy<P>(cols, br, k, n, sigma, tw, consts, z, log_t < 0 ? PERM_INV_LOG_T : log_t, threads ? threads : PERM_INV_THREADS,
                       log_l < 0 ? poly_log_l<P>() : log_l, log_b < 0 ? poly_log_b<P>() : log_b);
  });
}

extern "C" int emu_iop_lagrange_eval(int field, const uint32_t* c, uint64_t n, int bitrev, const uint32_t* tw, const uint32_t* consts,
                                     uint32_t* out, int log_t, unsigned threads, unsigned sum_threads) {
  return with_field(field, [&](auto p) {
    using P = decltype(p);
    return emu_lagrange<P>(c, n, bitrev, tw, consts, out, log_t < 0 ? PERM_INV_LOG_T : log_t, threads ? threads : PERM_INV_THREADS,
                           sum_threads ? sum_threads : 256u);
  });
}

extern "C" int emu_iop_evaluate(int field, const uint32_t* code, int len, int out_reg, const uint32_t* consts, int nconsts,
                                const uint32_t* const* inputs, const uint64_t* offsets, const int* bitrev, int m, uint64_t n, int out_bitrev,
                                uint32_t* r) {
  return with_field(field, [&](auto p) {
    using P = decltype(p);
    return emu_evaluate<P>(code, len, out_reg, consts, nconsts, inputs, offsets, bitrev, m, n, out_bitrev, r);
  });
}

extern "C" int emu_iop_divide(int field, const uint32_t* a, uint64_t n, uint64_t offset, int bitrev, const uint32_t* inv, unsigned rho,
                              uint32_t* out) {
  return with_field(field, [&](auto p) {
    using P = decltype(p);
    return emu_divide<P>(a, n, offset, bitrev, inv, rho, out);
  });
}
