// TEST INFRASTRUCTURE ONLY -- runs the product's kernels (gnark-crypto_b200/csrc/kernels.cuh, unmodified) on the CPU, one
// emulated thread at a time, in the order gnark-crypto_b200/csrc/engine_impl.cuh launches them (run_accumulate,
// run_bucket_reduce, run_finalize), so that the kernel-level logic -- digit recoding + histogram, the two scatters,
// the chunked segmented reduction with its owner / carry rule and the two-part launch, the carry levels, the
// segment reduction, the finalize, the window-table level -- is checked against the oracle WITHOUT a GPU
// (tests/test_emu_kernels.py).  Chunk length, carry run lengths, segment length, scatter passes and the launch
// split are parameters here, so the tests also visit shapes the engine's own heuristics would not pick.
// Never linked into libgmsm.so: the product has no CPU path.
#include <algorithm>
#include <cstring>
#include <vector>

#include "affine_kernels.cuh"

using namespace gmsm;

namespace {

struct Opts {
  int c;
  int tables;         // 1: window-table mode (one shared bucket set over W table rows)
  uint32_t K;         // entries per accumulate chunk
  uint32_t K2_first;  // items per thread, first carry level
  uint32_t K2;        // ... later levels
  uint32_t L;         // buckets per reduction segment
  int passes;         // bucket-range passes of the shared scatter
  int split;          // > 0: two-part accumulate, split after `split` windows / passes
  int batches;        // > 1: pipelined batches (scratch buckets + k_merge_buckets)
  void* partials_out; // non-null: write the W (or 1) window partials there and skip the finalize
  int mode;           // bit 0: the real K1b scan kernels (block scans with warp shuffles) instead of a host scan
                      // bit 1: batch-affine bucket accumulation (affine_kernels.cuh, GMSM_AFFINE=1) instead of k_accumulate
                      // bit 2: every launch through the cooperative (fiber) launcher
                      // bit 4: force K1's warp-aggregated atomics (as if the sampling pass had found a hot value)
                      // bit 3: the lane-parallel (quad) form of the tail kernels -- carry levels, segment reduction, group sums
};

static bool g_coop_all = false;
// launch through the sequential launcher, or the cooperative one when asked for (kernels with barriers / shuffles
// always name emu_launch_coop directly)
template <class Kn, class... A>
static void LAUNCH(Kn kernel, dim3 grid, unsigned block, A... args) {
  if (g_coop_all) emu_launch_coop(kernel, grid, block, args...);
  else emu_launch(kernel, grid, block, args...);
}

// K1b as engine_impl.cuh's scan_u32: per-block totals, one-block scan of the totals, per-block scan + prefix
static void real_scan(const uint32_t* in, uint32_t nbp, uint32_t* out) {
  const unsigned nb_blocks = (unsigned)((nbp + SCAN_TILE - 1) / SCAN_TILE);
  std::vector<uint32_t> block_sums(2 * (size_t)nb_blocks + 16, 0);
  emu_launch_coop(k_scan_block_sums, dim3(nb_blocks), (unsigned)SCAN_THREADS, in, nbp, block_sums.data());
  emu_launch_coop(k_scan_top, dim3(1), 1024u, block_sums.data(), (uint32_t)nb_blocks, block_sums.data() + nb_blocks);
  emu_launch_coop(k_scan_final, dim3(nb_blocks), (unsigned)SCAN_THREADS, in, nbp, (const uint32_t*)block_sums.data(), out);
}


static unsigned nblk(size_t n, unsigned t) { return (unsigned)((n + t - 1) / t); }

// stages K1..K2b of engine_impl.cuh's run_accumulate on one batch: afterwards `buckets` holds the batch's bucket sums
template <class G>
int emu_accumulate(const Affine<typename G::F>* points, uint32_t row_stride, const typename G::Fr* scalars, size_t n, const WindowPlan& p,
                   bool shared, const Opts& o, std::vector<XYZZ<typename G::F>>& buckets) {
  using F = typename G::F;
  using X = XYZZ<F>;
  if (n == 0) return 0;
  const uint32_t n32 = (uint32_t)n;
  const size_t nbp = (size_t)p.nb_total + 1;
    // K1: digits + histogram
    std::vector<uint32_t> hist(nbp + 8, 0), offsets(nbp + 8, 0), digits(n * (size_t)p.nwin + 16, 0), ranks(n * (size_t)p.nwin + 16, 0xFFFFFFFFu),
        entries(n * (size_t)p.nwin + 16, 0);
    // (warp collectives -- __match_any_sync / __shfl_sync -- inside: always the cooperative launcher)
    emu_launch_coop(k_skew_probe<G>, dim3(PROBE_BLOCKS), 256u, scalars, n32, p.c, p.nwin, hist.data() + nbp + 4);
    if (o.mode & 16) hist[nbp + 4] = 1;    // force the rank mode (as if the sampling pass had found skewed scalars)
    if (o.mode & 32) hist[nbp + 4] = 0;    // force the plain mode
    emu_launch_coop(k_digits_hist<G>, dim3(std::min<unsigned>(nblk(n, 256), GMSM_NUM_SMS * 16u)), 256u, scalars, n32, p.c, p.nwin,
                    shared ? 0u : p.nb, digits.data(), ranks.data(), hist.data(), (const uint32_t*)(hist.data() + nbp + 4));
    // K1b: exclusive scan -- the three scan kernels (cooperative launch) or a host scan
    auto scan_u32 = [&](const uint32_t* in, uint32_t* out) {
      if (o.mode & 1) { real_scan(in, (uint32_t)nbp, out); return; }
      uint32_t run = 0;
      for (size_t i = 0; i < nbp; i++) { out[i] = run; run += in[i]; }
    };
    scan_u32(hist.data(), offsets.data());
    // K1c: scatter
    int NPASS = p.nwin;
    if (shared) NPASS = std::max(1, o.passes);
    const uint32_t range_sz = shared ? (p.nb_total + (uint32_t)NPASS - 1) / (uint32_t)NPASS : p.nb;
    if (shared) {
      for (int r = 0; r < NPASS; r++) {
        const uint32_t blo = (uint32_t)std::min<uint64_t>((uint64_t)r * range_sz, p.nb_total);
        const uint32_t bhi = (uint32_t)std::min<uint64_t>((uint64_t)(r + 1) * range_sz, p.nb_total);
        if (blo >= bhi) continue;
        LAUNCH(k_scatter_shared, dim3(std::min<unsigned>(nblk(n, 1024), 296u), (unsigned)p.nwin), 256, (const uint32_t*)digits.data(),
                   (const uint32_t*)ranks.data(), n32, row_stride, hist.data(), (const uint32_t*)offsets.data(), entries.data(), blo, bhi,
                   (const uint32_t*)(hist.data() + nbp + 4));
      }
    } else {
      for (int j = 0; j < p.nwin; j++)
        LAUNCH(k_scatter_window, dim3(std::min<unsigned>(nblk(n, 1024), GMSM_NUM_SMS * 8u)), 256, (const uint32_t*)(digits.data() + (size_t)j * n),
                   (const uint32_t*)(ranks.data() + (size_t)j * n), n32, hist.data() + (size_t)j * p.nb,
                   (const uint32_t*)(offsets.data() + (size_t)j * p.nb), entries.data(), (const uint32_t*)(hist.data() + nbp + 4));
    }
    if (hist[nbp + 4]) {
      // rank mode: the ranks K1 handed out number every bucket's entries 0 .. count-1 exactly once
      std::vector<uint32_t> seen(offsets[p.nb_total], 0);
      for (int j = 0; j < p.nwin; j++)
        for (size_t i = 0; i < n; i++) {
          const uint32_t code = digits[(size_t)j * n + i];
          if (!code) continue;
          const uint32_t b = (shared ? 0u : (uint32_t)j * p.nb) + code_bucket(code);
          const uint32_t pos = offsets[b] + ranks[(size_t)j * n + i];
          if (pos >= offsets[b + 1] || seen[pos]++) return 10;
        }
      for (uint32_t v : seen) if (v != 1) return 10;
    } else {
      for (size_t i = 0; i < nbp; i++)
        if (hist[i] != 0) return 10;   // plain mode: every counter must have been consumed exactly by the scatter
    }
    if (o.mode & 2) {
      // K2 (batch-affine, engine_impl.cuh's affine branch): balanced tree over the bucket-ordered entries, one shared
      // inversion per level through the hierarchical product scans
      using A = Affine<F>;
      const uint32_t nbt = p.nb_total;
      uint32_t maxlen = 0;
      emu_launch_coop(k_aff_max_len, dim3(4), 256u, (const uint32_t*)offsets.data(), nbt, &maxlen);
      int nlevels = 0;
      while (((uint64_t)1 << nlevels) < maxlen) nlevels++;
      const size_t ent = n * (size_t)p.nwin;
      const size_t m1 = (ent + std::min(nbp, ent)) / 2 + 2, m2 = (m1 + std::min(nbp, m1)) / 2 + 2;
      std::vector<A> buf0(m1), buf1(m2);
      std::vector<F> pref(m1);
      std::vector<uint32_t> off_a(nbp + 8, 0), off_b(nbp + 8, 0), counts(nbp + 8, 0);
      const uint32_t* off_cur = offsets.data();
      const A* src_cur = nullptr;
      size_t m_up = ent;
      for (int l = 0; l < nlevels; l++) {
        uint32_t* off_next = (l & 1) ? off_b.data() : off_a.data();
        LAUNCH(k_aff_level_counts, dim3(std::min<unsigned>(nblk(nbp, 256), 8u)), 256u, (const uint32_t*)offsets.data(), nbt, l + 1, counts.data());
        scan_u32(counts.data(), off_next);
        const size_t m_next = std::min(m_up, (m_up + std::min<size_t>(nbt, m_up)) / 2 + 1);
        const uint32_t B = o.K ? std::min<uint32_t>(o.K, 128u) : 8u;      // slots per lane: the chunk-length knob
        const size_t T = ((m_next + 32 * (size_t)B - 1) / (32 * (size_t)B)) * 32;
        if (m_next > ((l & 1) ? m2 : m1)) return 11;
        A* dst = (l & 1) ? buf1.data() : buf0.data();
        std::vector<F> totals(T), ps(T);
        const unsigned NB = nblk(T, PSCAN_TILE);
        std::vector<F> bp(3 * ((size_t)NB + 8));
        const size_t bp_stride = (size_t)NB + 8;
        if (l == 0)
          LAUNCH(k_aff_forward<G, true>, dim3(nblk(T, 128)), 128u, points, (const uint32_t*)entries.data(), src_cur, off_cur, (const uint32_t*)off_next,
                 nbt, B, (uint32_t)T, pref.data(), totals.data());
        else
          LAUNCH(k_aff_forward<G, false>, dim3(nblk(T, 128)), 128u, points, (const uint32_t*)entries.data(), src_cur, off_cur, (const uint32_t*)off_next,
                 nbt, B, (uint32_t)T, pref.data(), totals.data());
        emu_launch_coop(k_aff_scan_tiles<G>, dim3(NB), (unsigned)PSCAN_THREADS, (const F*)totals.data(), (uint32_t)T, ps.data(), bp.data());
        emu_launch_coop(k_aff_scan_top<G>, dim3(1), (unsigned)PSCAN_THREADS, (const F*)bp.data(), (uint32_t)NB, bp.data() + bp_stride,
                        bp.data() + 2 * bp_stride);
        if (l == 0)
          LAUNCH(k_aff_backward<G, true>, dim3(nblk(T, 128)), 128u, points, (const uint32_t*)entries.data(), src_cur, off_cur, (const uint32_t*)off_next,
                 nbt, B, (uint32_t)T, (const F*)pref.data(), (const F*)ps.data(), (const F*)(bp.data() + 2 * bp_stride), dst);
        else
          LAUNCH(k_aff_backward<G, false>, dim3(nblk(T, 128)), 128u, points, (const uint32_t*)entries.data(), src_cur, off_cur, (const uint32_t*)off_next,
                 nbt, B, (uint32_t)T, (const F*)pref.data(), (const F*)ps.data(), (const F*)(bp.data() + 2 * bp_stride), dst);
        src_cur = dst;
        off_cur = off_next;
        m_up = m_next;
      }
      if (nlevels == 0)
        LAUNCH(k_aff_to_buckets<G, true>, dim3(std::min<unsigned>(nblk(nbt, 256), 8u)), 256u, points, (const uint32_t*)entries.data(), src_cur, off_cur, nbt,
               buckets.data());
      else
        LAUNCH(k_aff_to_buckets<G, false>, dim3(std::min<unsigned>(nblk(nbt, 256), 8u)), 256u, points, (const uint32_t*)entries.data(), src_cur, off_cur, nbt,
               buckets.data());
      return 0;
    }
    // K2: accumulate
    const uint32_t K = o.K;
    const size_t nchunks = (n * (size_t)p.nwin + K - 1) / K;
    std::vector<X> carr0(nchunks), carr1((nchunks + 1) / 2 + 1);
    std::vector<uint32_t> ids0(nchunks + 8, 0), ids1((nchunks + 1) / 2 + 8, 0);
    const int split = std::min(o.split, NPASS);
    if (split > 0 && split < NPASS) {
      const uint32_t split_bucket = (uint32_t)std::min<uint64_t>((uint64_t)split * range_sz, p.nb_total);
      for (int part = 1; part <= 2; part++)
        LAUNCH(k_accumulate<G>, dim3(nblk(nchunks, 128)), 128, points, (const uint32_t*)entries.data(), (const uint32_t*)offsets.data(),
                   p.nb_total, K, (uint32_t)nchunks, buckets.data(), carr0.data(), ids0.data(), part, split_bucket);
    } else {
      LAUNCH(k_accumulate<G>, dim3(nblk(nchunks, 128)), 128, points, (const uint32_t*)entries.data(), (const uint32_t*)offsets.data(),
                 p.nb_total, K, (uint32_t)nchunks, buckets.data(), carr0.data(), ids0.data(), 0, 0u);
    }
    // K2b: carry levels
    {
      size_t n_in = nchunks;
      bool first = true;
      X* cp[2] = {carr0.data(), carr1.data()};
      uint32_t* ip[2] = {ids0.data(), ids1.data()};
      std::vector<X> big1;
      std::vector<uint32_t> bigi;
      int cur = 0;
      while (n_in > 1) {
        const uint32_t k2 = first ? o.K2_first : o.K2;
        first = false;
        const size_t n_out = (n_in + k2 - 1) / k2;
        if ((o.mode & 8) && !(getenv("EMU_NOQ") && strchr(getenv("EMU_NOQ"), 'c')))
          emu_launch_coop(k_carry_level<G, true>, dim3(nblk(n_out * 4, 128)), 128u, (const X*)cp[cur], (const uint32_t*)ip[cur], (uint32_t)n_in, k2,
                          buckets.data(), cp[cur ^ 1], ip[cur ^ 1]);
        else
          LAUNCH(k_carry_level<G, false>, dim3(nblk(n_out, 128)), 128, (const X*)cp[cur], (const uint32_t*)ip[cur], (uint32_t)n_in, k2, buckets.data(),
                     cp[cur ^ 1], ip[cur ^ 1]);
        n_in = n_out;
        cur ^= 1;
      }
    }
  return 0;
}

template <class G>
int emu_msm(const void* points_v, const void* scalars_v, size_t n, const Opts& o, void* out_jac) {
  using F = typename G::F;
  using X = XYZZ<F>;
  using A = Affine<F>;
  WindowPlan p = make_plan(G::FrParams::BITS, o.c);
  const bool shared = o.tables != 0;
  if (shared) p.nb_total = std::max(p.nb, p.nb_last);
  const int red_windows = shared ? 1 : p.nwin;
  const uint32_t n32 = (uint32_t)n;
  const auto* scalars = reinterpret_cast<const typename G::Fr*>(scalars_v);
  const A* points = reinterpret_cast<const A*>(points_v);

  // window tables: row j = 2^c * row j-1 (gmsm_tables_build_device)
  std::vector<A> table;
  if (shared) {
    table.resize((size_t)p.nwin * std::max<size_t>(n, 1));
    if (n) std::memcpy(table.data(), points, n * sizeof(A));
    for (int j = 1; j < p.nwin && n; j++)
      LAUNCH(k_table_level<G>, dim3(nblk((n + TAB_M - 1) / TAB_M, 128)), 128, (const A*)(table.data() + (size_t)(j - 1) * n), n32, o.c,
                 table.data() + (size_t)j * n);
    points = table.data();
  }

  std::vector<X> buckets(p.nb_total, X::inf());
  std::vector<X> partials(red_windows, X::inf());
  // pipelined host calls (pipeline_run in gmsm.cu): contiguous batches, the first into the bucket array, every later
  // one into scratch buckets that k_merge_buckets adds on top
  const int nbatch = std::max(1, std::min<int>(o.batches, (int)std::max<size_t>(n, 1)));
  for (int bi = 0; bi < nbatch; bi++) {
    const size_t lo = n * bi / nbatch, hi = n * (bi + 1) / nbatch;
    if (bi == 0) {
      if (int rc = emu_accumulate<G>(points + lo, (uint32_t)n, scalars + lo, hi - lo, p, shared, o, buckets)) return rc;
    } else {
      std::vector<X> scratch_b(p.nb_total, X::inf());
      if (int rc = emu_accumulate<G>(points + lo, (uint32_t)n, scalars + lo, hi - lo, p, shared, o, scratch_b)) return rc;
      LAUNCH(k_merge_buckets<G>, dim3(nblk(p.nb_total, 128)), 128, buckets.data(), (const X*)scratch_b.data(), p.nb_total);
    }
  }
  // K3: bucket reduction
  {
    const uint32_t nbmax = shared ? p.nb_total : std::max(p.nb, p.nb_last);
    const uint32_t L = o.L, S = (nbmax + L - 1) / L;
    const uint32_t nb_reg = shared ? p.nb_total : p.nb, nb_last = shared ? p.nb_total : p.nb_last;
    std::vector<X> seg0((size_t)red_windows * S), seg1((size_t)red_windows * ((S + 15) / 16) + 1);
    if ((o.mode & 8) && !(getenv("EMU_NOQ") && strchr(getenv("EMU_NOQ"), 's')))
      emu_launch_coop(k_bucket_segments<G, true>, dim3(nblk((size_t)red_windows * S * 4, 128)), 128u, (const X*)buckets.data(), red_windows, nb_reg,
                      nb_last, L, S, seg0.data());
    else
      LAUNCH(k_bucket_segments<G, false>, dim3(nblk((size_t)red_windows * S, 128)), 128, (const X*)buckets.data(), red_windows, nb_reg, nb_last, L, S,
                 seg0.data());
    uint32_t per = S;
    X* sp[2] = {seg0.data(), seg1.data()};
    int cur = 0;
    while (per > 1) {
      const bool quad = (o.mode & 8) && !(getenv("EMU_NOQ") && strchr(getenv("EMU_NOQ"), 'g'));
      const uint32_t R = quad ? 16u : 2u * TREE_THREADS, outp = (per + R - 1) / R;
      X* dst = (outp == 1) ? partials.data() : sp[cur ^ 1];
      if (quad)
        emu_launch_coop(k_sum_groups<G, true>, dim3(nblk((size_t)red_windows * outp * 4, 128)), 128u, (const X*)sp[cur], per, R, outp, red_windows, dst);
      else     // block tree with barriers: cooperative launcher
        emu_launch_coop(k_sum_tree<G>, dim3(outp, (unsigned)red_windows), (unsigned)TREE_THREADS, (const X*)sp[cur], per, outp, dst);
      per = outp;
      cur ^= 1;
    }
    if (S == 1) std::memcpy(partials.data(), seg0.data(), (size_t)red_windows * sizeof(X));
  }
  if (o.partials_out) {   // one rank of a sharded MSM: stop after the bucket reduction (gmsm_ctx_window_sums_device)
    std::memcpy(o.partials_out, partials.data(), (size_t)red_windows * sizeof(X));
    return 0;
  }
  // K4: finalize
  std::vector<X> scratch(red_windows);
  Jac<F> out;
  if (o.mode & 8) emu_launch_coop(k_finalize<G, true>, dim3(1), (unsigned)FIN_THREADS, (const X*)partials.data(), 1, red_windows, p.c, scratch.data(), &out);
  else emu_launch_coop(k_finalize<G, false>, dim3(1), (unsigned)FIN_THREADS, (const X*)partials.data(), 1, red_windows, p.c, scratch.data(), &out);
  std::memcpy(out_jac, &out, sizeof(out));
  return 0;
}

// gmsm_ctx_finalize_device: nranks x W gathered partials (rank-major) -> per-window sum over the ranks, Horner, normal form
template <class G>
int emu_finalize(const void* partials, int nranks, int c, int tables, void* out_jac) {
  using F = typename G::F;
  using X = XYZZ<F>;
  const WindowPlan p = make_plan(G::FrParams::BITS, c);
  const int red_windows = tables ? 1 : p.nwin;
  std::vector<X> scratch(red_windows);
  Jac<F> out;
  emu_launch_coop(k_finalize<G, false>, dim3(1), (unsigned)FIN_THREADS, (const X*)partials, nranks, red_windows, p.c, scratch.data(), &out);
  std::memcpy(out_jac, &out, sizeof(out));
  return 0;
}

}  // namespace

#ifndef EMU_GROUP
#error "compile with -DEMU_GROUP=0..12"
#endif
#if EMU_GROUP == 0
using EmuG = bn254_g1;
#elif EMU_GROUP == 1
using EmuG = bn254_g2;
#elif EMU_GROUP == 2
using EmuG = bls12381_g1;
#elif EMU_GROUP == 3
using EmuG = bls12381_g2;
#elif EMU_GROUP == 4
using EmuG = bls12377_g1;
#elif EMU_GROUP == 5
using EmuG = bls12377_g2;
#elif EMU_GROUP == 6
using EmuG = secp256k1_g1;
#elif EMU_GROUP == 7
using EmuG = bw6761_g1;
#elif EMU_GROUP == 8
using EmuG = bw6761_g2;
#elif EMU_GROUP == 9
using EmuG = bls24315_g1;
#elif EMU_GROUP == 10
using EmuG = bls24317_g1;
#elif EMU_GROUP == 11
using EmuG = bw6633_g1;
#else
using EmuG = bw6633_g2;
#endif
#define EMU_CAT2(a, b) a##b
#define EMU_CAT(a, b) EMU_CAT2(a, b)
extern "C" int EMU_CAT(emu_msm_, EMU_GROUP)(const void* points, const void* scalars, size_t n, int c, int tables, uint32_t K, uint32_t K2_first,
                                             uint32_t K2, uint32_t L, int passes, int split, int batches, int mode, void* out_jac) {
  if (c < 2 || c > 24 || K < 1 || K2_first < 2 || K2 < 2 || L < 1) return 1;
  Opts o{c, tables, K, K2_first, K2, L, passes, split, batches, nullptr, mode};
  g_coop_all = (mode & 4) != 0;
  if ((mode & 2) && (tables || batches > 1)) return 2;   // as in the engine: the batch-affine pass is plain, single-batch only
  return emu_msm<EmuG>(points, scalars, n, o, out_jac);
}

// fixed-base helpers: k_generate_multiples (out[i] = [start + i] * base) and k_batch_scalar_mul (N1,
// BatchScalarMultiplicationG1/G2, g1.go:1039-1118) as gmsm_batch_scalar_mul launches them
extern "C" int EMU_CAT(emu_generate_, EMU_GROUP)(const void* base, uint64_t start, size_t n, void* out) {
  using A = Affine<typename EmuG::F>;
  if (n == 0) return 0;
  LAUNCH(k_generate_multiples<EmuG>, dim3(nblk((n + GEN_M - 1) / GEN_M, 128)), 128, (const A*)base, start, (uint64_t)n, (A*)out);
  return 0;
}
extern "C" int EMU_CAT(emu_batch_scalar_mul_, EMU_GROUP)(const void* base, const void* scalars, size_t n, int c, void* out) {
  using A = Affine<typename EmuG::F>;
  if (n == 0) return 0;
  const WindowPlan p = make_plan(EmuG::FrParams::BITS, c);
  const size_t tbl = (size_t)1 << (std::max(p.c, p.last_c) - 1);
  std::vector<A> table(tbl);
  LAUNCH(k_generate_multiples<EmuG>, dim3(nblk((tbl + GEN_M - 1) / GEN_M, 128)), 128, (const A*)base, (uint64_t)1, (uint64_t)tbl, table.data());
  LAUNCH(k_batch_scalar_mul<EmuG>, dim3(nblk(n, 128)), 128, (const A*)table.data(), (const typename EmuG::Fr*)scalars, (uint32_t)n, p.c, p.nwin,
             (A*)out);
  return 0;
}

extern "C" void EMU_CAT(emu_set_block_order_, EMU_GROUP)(unsigned order) { emu_block_order = order; }

// K1 alone: the digits k_digits_hist writes for the scalars (digits[j*n + i], W = ceil(fr.Bits / c) rows), in the plain
// (rank_mode = 0) or the rank mode (1, warp collectives: cooperative launcher).  Returns 10 if the histogram does not
// count exactly the non-zero digits.
extern "C" int EMU_CAT(emu_digits_, EMU_GROUP)(const void* scalars, size_t n, int c, int rank_mode, uint32_t* digits_out) {
  if (c < 2 || c > 24) return 1;
  if (n == 0) return 0;
  const WindowPlan p = make_plan(EmuG::FrParams::BITS, c);
  const size_t nbp = (size_t)p.nb_total + 1;
  std::vector<uint32_t> hist(nbp + 8, 0), ranks(n * (size_t)p.nwin + 16, 0xFFFFFFFFu);
  hist[nbp + 4] = rank_mode ? 1u : 0u;
  const auto* s = reinterpret_cast<const typename EmuG::Fr*>(scalars);
  const dim3 grid(std::min<unsigned>(nblk(n, 256), GMSM_NUM_SMS * 16u));
  if (rank_mode)
    emu_launch_coop(k_digits_hist<EmuG>, grid, 256u, s, (uint32_t)n, p.c, p.nwin, p.nb, digits_out, ranks.data(), hist.data(),
                    (const uint32_t*)(hist.data() + nbp + 4));
  else
    emu_launch(k_digits_hist<EmuG>, grid, 256u, s, (uint32_t)n, p.c, p.nwin, p.nb, digits_out, ranks.data(), hist.data(),
               (const uint32_t*)(hist.data() + nbp + 4));
  std::vector<uint32_t> want(nbp, 0);
  for (int j = 0; j < p.nwin; j++)
    for (size_t i = 0; i < n; i++)
      if (const uint32_t code = digits_out[(size_t)j * n + i]) want[(size_t)j * p.nb + code_bucket(code)]++;
  for (size_t b = 0; b < nbp; b++)
    if (hist[b] != want[b]) return 10;
  return 0;
}

// one rank's window partials (W x xyzz, or 1 in window-table mode), and the combine over ranks
extern "C" int EMU_CAT(emu_window_sums_, EMU_GROUP)(const void* points, const void* scalars, size_t n, int c, int tables, uint32_t K, void* out_partials) {
  Opts o{c, tables, K, 4, 16, 32, 3, 1, 1, out_partials, 0};
  g_coop_all = false;
  return emu_msm<EmuG>(points, scalars, n, o, nullptr);
}
extern "C" int EMU_CAT(emu_finalize_, EMU_GROUP)(const void* partials, int nranks, int c, int tables, void* out_jac) {
  return emu_finalize<EmuG>(partials, nranks, c, tables, out_jac);
}
