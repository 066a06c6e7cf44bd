// TEST INFRASTRUCTURE ONLY -- runs the counting sort of the bucket pass as engine_impl.cuh launches it (K1 k_digits_hist,
// K1b with k_scan_final_ends, K1c k_scatter_window / k_scatter_window_aux / k_scatter_shared without an offsets array: the counters are bucket end
// pointers) on the CPU over the stand-in tests/emu/cuda_runtime.h, and hands back what the accumulate would read: offsets,
// entries, and the counters after the scatter (tests/test_emu_scatter_ends_cpu.py).  Never linked into libgmsm.so.
#include <algorithm>
#include <cstring>
#include <vector>

#include "kernels.cuh"

using namespace gmsm;

namespace {
unsigned nblk(size_t n, unsigned t) { return (unsigned)((n + t - 1) / t); }
}

// bn254 G1 scalars (4 u64 Montgomery limbs each).  tables = 0: one bucket range per window, W scatter launches;
// tables = 1: one shared bucket set, `passes` bucket-range launches.  rank = 1 forces the rank mode, 0 the plain mode.
// offsets / counters: nb_total + 1 words, entries: n * W words, digits: n * W words (window-major).  Returns 0, or 1 on a
// bad shape.
extern "C" int emu_sort_entries(const uint64_t* scalars, size_t n, int c, int tables, int passes, int rank, uint32_t* offsets_out,
                                uint32_t* counters_out, uint32_t* entries_out, uint32_t* digits_out, uint32_t* nb_total_out) {
  using G = bn254_g1;
  WindowPlan p = make_plan(G::FrParams::BITS, c);
  if (tables) p.nb_total = std::max(p.nb, p.nb_last);
  const uint32_t n32 = (uint32_t)n;
  const size_t nbp = (size_t)p.nb_total + 1;
  std::vector<uint32_t> hist(nbp + 8, 0), offsets(nbp + 8, 0), digits(n * (size_t)p.nwin + 16, 0),
      ranks(n * (size_t)p.nwin + 16, 0xFFFFFFFFu), entries(n * (size_t)p.nwin + 16, 0xFFFFFFFFu);
  const auto* s = reinterpret_cast<const typename G::Fr*>(scalars);
  hist[nbp + 4] = rank ? 1u : 0u;
  emu_launch_coop(k_digits_hist<G>, dim3(std::min<unsigned>(nblk(n, 256), 64u)), 256u, s, n32, p.c, p.nwin, tables ? 0u : p.nb,
                  digits.data(), ranks.data(), hist.data(), (const uint32_t*)(hist.data() + nbp + 4));
  const unsigned nb_blocks = nblk(nbp, SCAN_TILE);
  std::vector<uint32_t> block_sums(2 * (size_t)nb_blocks + 16, 0);
  emu_launch_coop(k_scan_block_sums, dim3(nb_blocks), (unsigned)SCAN_THREADS, (const uint32_t*)hist.data(), (uint32_t)nbp,
                  block_sums.data());
  emu_launch_coop(k_scan_top, dim3(1), 1024u, block_sums.data(), (uint32_t)nb_blocks, block_sums.data() + nb_blocks);
  emu_launch_coop(k_scan_final_ends, dim3(nb_blocks), (unsigned)SCAN_THREADS, hist.data(), (uint32_t)nbp,
                  (const uint32_t*)block_sums.data(), offsets.data());
  const uint32_t* flag = hist.data() + nbp + 4;
  if (tables) {
    if (passes < 1) return 1;
    const uint32_t range_sz = (p.nb_total + (uint32_t)passes - 1) / (uint32_t)passes;
    for (int r = 0; r < passes; r++) {
      const uint32_t blo = (uint32_t)std::min<uint64_t>((uint64_t)r * range_sz, p.nb_total);
      const uint32_t bhi = (uint32_t)std::min<uint64_t>((uint64_t)(r + 1) * range_sz, p.nb_total);
      if (blo >= bhi) continue;
      emu_launch(k_scatter_shared, dim3(std::min<unsigned>(nblk(n, 1024), 7u), (unsigned)p.nwin), 256u, (const uint32_t*)digits.data(),
                 (const uint32_t*)ranks.data(), n32, n32, hist.data(), (const uint32_t*)nullptr, entries.data(), blo, bhi, flag);
    }
  } else {
    // even windows as on the call's stream, odd ones as on the auxiliary stream (the slim form)
    for (int j = 0; j < p.nwin; j++) {
      const uint32_t* dw = digits.data() + (size_t)j * n;
      const uint32_t* rw = ranks.data() + (size_t)j * n;
      uint32_t* ends = hist.data() + (size_t)j * p.nb;
      if (j % 2 == 0)
        emu_launch(k_scatter_window, dim3(std::min<unsigned>(nblk(n, 256u * SCATTER_U), 5u)), 256u, dw, rw, n32, ends,
                   (const uint32_t*)nullptr, entries.data(), flag);
      else
        emu_launch(k_scatter_window_aux, dim3(std::min<unsigned>(nblk(n, 256u * SCATTER_AUX_U), 2u)), 256u, dw, rw, n32, ends,
                   (const uint32_t*)nullptr, entries.data(), flag);
    }
  }
  const size_t m = offsets[p.nb_total];
  std::memcpy(offsets_out, offsets.data(), nbp * 4);
  std::memcpy(counters_out, hist.data(), nbp * 4);
  std::memcpy(entries_out, entries.data(), m * 4);
  std::memcpy(digits_out, digits.data(), n * (size_t)p.nwin * 4);
  *nb_total_out = p.nb_total;
  return 0;
}
