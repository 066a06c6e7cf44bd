// Template orchestration of the kernels for one (curve, group); included by inst_*.cu.
#pragma once
#include <cstring>

#include "engine.h"
#include "kernels.cuh"
#include "affine_kernels.cuh"
#include "lagrange_kernels.cuh"
#include "mpc_kernels.cuh"

namespace gmsm {

#define LAUNCH_CHECK() CK(cudaGetLastError())

// stages K1..K2b on one batch of (points, scalars): afterwards c->buckets holds the bucket sums.
// rmw = 0: buckets are (re)initialised by this batch; rmw = 1: the batch is accumulated on top of the
// buckets of the previous batches (pipelined one-shot call: H2D of batch k+1 overlaps K1..K2 of batch k).
template <class G>
static int run_accumulate(gmsm_ctx* c, const void* d_points, const void* d_scalars, size_t n, int rmw, cudaStream_t st) {
  using F = typename G::F;
  using X = XYZZ<F>;
  const WindowPlan& p = c->plan;
  int launches = 0;
  const bool prof = c->profiling;
  auto mark = [&](int i) { if (prof) cudaEventRecord(c->ev[i], st); };
  mark(0);
  // a follow-up batch (rmw) is accumulated into the scratch bucket array and merged at the end, so the
  // hot loop never carries a read-modify-write (a divergent full add per bucket boundary otherwise)
  X* buckets = reinterpret_cast<X*>(rmw ? c->buckets2 : c->buckets);
  if (n == 0) {
    if (!rmw) CK(cudaMemsetAsync(buckets, 0, (size_t)p.nb_total * sizeof(X), st));
    for (int i = 1; i <= 5; i++) mark(i);
    c->tl_npass = c->tl_parts = 0;
    c->last_launches = 0;
    return GMSM_OK;
  }
  const uint32_t n32 = (uint32_t)n;
  const size_t nbp = (size_t)p.nb_total + 1;
  const auto* scalars = reinterpret_cast<const typename G::Fr*>(d_scalars);
  const auto* points = reinterpret_cast<const Affine<F>*>(d_points);

  // K1: digits + histogram
  CK(cudaMemsetAsync(c->hist, 0, (nbp + 8) * 4, st));
  {
    unsigned blocks = std::min<unsigned>(nblk(n, 256), GMSM_NUM_SMS * 16u);
    // the mode flag lives in the pad of hist[] (just cleared: plain); GMSM_K1_MODE forces it instead of sampling the scalars
    if (c->k1_mode < 0) {
      k_skew_probe<G><<<PROBE_BLOCKS, 256, 0, st>>>(scalars, n32, p.c, p.nwin, c->hist + nbp + 4);
      launches++;
    } else if (c->k1_mode == 1) {
      CK(cudaMemsetAsync(c->hist + nbp + 4, 1, 1, st));   // little-endian word 1
    }
    k_digits_hist<G><<<blocks, 256, 0, st>>>(scalars, n32, p.c, p.nwin, c->shared ? 0u : p.nb, c->digits, c->ranks, c->hist, c->hist + nbp + 4);
    launches++;
    LAUNCH_CHECK();
  }
  mark(1);
  // K1b: scan
  // ends: the counters `in` become bucket end pointers as well (the histogram, for the scatter)
  auto scan_u32 = [&](uint32_t* in, uint32_t* out, bool ends) -> int {
    unsigned nb_blocks = nblk(nbp, SCAN_TILE);
    k_scan_block_sums<<<nb_blocks, SCAN_THREADS, 0, st>>>(in, (uint32_t)nbp, c->block_sums);
    k_scan_top<<<1, 1024, 0, st>>>(c->block_sums, nb_blocks, c->block_sums + nb_blocks);
    if (ends)
      k_scan_final_ends<<<nb_blocks, SCAN_THREADS, 0, st>>>(in, (uint32_t)nbp, c->block_sums, out);
    else
      k_scan_final<<<nb_blocks, SCAN_THREADS, 0, st>>>(in, (uint32_t)nbp, c->block_sums, out);
    launches += 3;
    LAUNCH_CHECK();
    return GMSM_OK;
  };
  if (int rc = scan_u32(c->hist, c->offsets, true)) return rc;
  mark(2);
  // K1c: scatter, one launch per window (L2-resident write set).  In the extended-Jacobian mode only the
  // first SPLIT_W windows are scattered on the call's stream; the rest go to the context's auxiliary stream
  // and run underneath the first part of the accumulate kernel (multiplier-bound, L2 idle) -- see K2.
  // (faster for the G1 groups; slower for G2, whose 255-register accumulate blocks leave no room for co-resident
  // scatter blocks -> G1 groups only.)  SPLIT_W = 4 by default: at bn254 G1 n = 2^24 (15 windows) part 1 then lasts long
  // enough for the other 11 windows to be scattered underneath it, and part 2 hardly waits (DESIGN.md section 5).
  // Window-table mode: one pass per bucket range instead of one per window (k_scatter_shared); the ranges play
  // the role of the windows for the overlap with the accumulate.
  // (timed at bn254 G1 n = 2^24, c = 22: every pass streams all n*W digits, so few passes win even though a pass's
  // slice -- ~200 MB -- exceeds L2: 4 passes with one of them ahead of the accumulate beat both 12 passes and 1 pass)
  int NPASS = p.nwin;
  if (c->shared) {
    const double slice = (double)n * p.nwin * 4.0 / 200e6;
    NPASS = c->table_passes > 0 ? c->table_passes : (int)std::min(16.0, std::max(4.0, slice + 0.5));
  }
  const uint32_t range_sz = c->shared ? (p.nb_total + (uint32_t)NPASS - 1) / (uint32_t)NPASS : p.nb;
  const int SPLIT_W = (!c->affine && sizeof(F) <= 48 && p.nwin >= 6 && n >= (1u << 16)) ? std::min(c->shared ? c->split_tab : c->split_w, NPASS) : NPASS;
  // The counters in hist are bucket end pointers (k_scan_final_ends): the scatters take their positions from them and get no
  // offsets.  On the auxiliary stream the slim form (k_scatter_window_aux, one block per SM) so that it shares the SMs with
  // the accumulate; that stream has the highest priority (gmsm.cu, ctx_alloc).
  const unsigned scatter_blocks = std::min<unsigned>(nblk(n, 256 * SCATTER_U), GMSM_NUM_SMS * (unsigned)SCATTER_BLOCKS_PER_SM);
  const unsigned scatter_blocks_aux = std::min<unsigned>(nblk(n, 256 * SCATTER_AUX_U), GMSM_NUM_SMS * (unsigned)SCATTER_AUX_BLOCKS_PER_SM);
  const unsigned shared_blocks = std::min<unsigned>(nblk(n, 256 * 4), GMSM_NUM_SMS * 2u);
  // profiling level 2: events around every scatter pass and the accumulate parts (gmsm_ctx_last_timeline_ms)
  const bool timeline = c->profiling >= 2;
  if (timeline) {
    while (c->tl_ev.size() < (size_t)NPASS * 2 + 4) {
      cudaEvent_t e;
      CK(cudaEventCreate(&e));
      c->tl_ev.push_back(e);
    }
    c->tl_npass = NPASS;
    c->tl_split = std::min(SPLIT_W, NPASS);
    c->tl_parts = 0;
  }
  auto tl = [&](size_t i, cudaStream_t s) { if (timeline) cudaEventRecord(c->tl_ev[i], s); };
  auto scatter = [&](int r, cudaStream_t s) {   // pass r: bucket range r (window-table mode) or window r
    tl(2 * (size_t)r, s);
    if (c->shared) {
      const uint32_t blo = std::min<uint64_t>((uint64_t)r * range_sz, p.nb_total);
      const uint32_t bhi = std::min<uint64_t>((uint64_t)(r + 1) * range_sz, p.nb_total);
      if (blo < bhi) {
        k_scatter_shared<<<dim3(shared_blocks, (unsigned)p.nwin), 256, 0, s>>>(c->digits, c->ranks, n32, c->tab_stride, c->hist,
                                                                              nullptr, c->entries, blo, bhi, c->hist + nbp + 4);
        launches++;
      }
    } else {
      const uint32_t* dw = c->digits + (size_t)r * n;
      const uint32_t* rw = c->ranks + (size_t)r * n;
      uint32_t* ends = c->hist + (size_t)r * p.nb;
      if (s == st)
        k_scatter_window<<<scatter_blocks, 256, 0, s>>>(dw, rw, n32, ends, nullptr, c->entries, c->hist + nbp + 4);
      else
        k_scatter_window_aux<<<scatter_blocks_aux, 256, 0, s>>>(dw, rw, n32, ends, nullptr, c->entries, c->hist + nbp + 4);
      launches++;
    }
    tl(2 * (size_t)r + 1, s);
  };
  if (SPLIT_W < NPASS) {
    CK(cudaEventRecord(c->ev_split[0], st));           // scan done: offsets, digits, hist are ready
    CK(cudaStreamWaitEvent(c->aux, c->ev_split[0], 0));
    for (int r = SPLIT_W; r < NPASS; r++) scatter(r, c->aux);
    CK(cudaEventRecord(c->ev_split[1], c->aux));
  }
  for (int r = 0; r < SPLIT_W; r++) scatter(r, st);
  LAUNCH_CHECK();
  mark(3);
  if (c->affine && c->shared) return set_err(GMSM_EINVAL, "internal: window tables need the default accumulation mode");
  if (c->affine && rmw) return set_err(GMSM_EINVAL, "internal: batch-affine accumulation cannot extend existing buckets");
  if (c->affine) {
    // K2 (batch-affine): balanced tree over the bucket-ordered entries, one shared inversion per level
    using A = Affine<F>;
    const uint32_t nbt = p.nb_total;
    CK(cudaMemsetAsync(c->aff_maxlen, 0, 4, st));
    k_aff_max_len<<<GMSM_NUM_SMS * 4, 256, 0, st>>>(c->offsets, nbt, c->aff_maxlen);
    launches++;
    LAUNCH_CHECK();
    CK(cudaMemcpyAsync(c->aff_maxlen_host, c->aff_maxlen, 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    const uint32_t maxlen = *c->aff_maxlen_host;
    int nlevels = 0;
    while (((uint64_t)1 << nlevels) < maxlen) nlevels++;
    const uint32_t* off_cur = c->offsets;
    const A* src_cur = nullptr;
    size_t m_up = n * (size_t)p.nwin;
    F* bp = reinterpret_cast<F*>(c->aff_bp);
    const size_t bp_stride = c->aff_tcap / 1024 + 8;
    for (int l = 0; l < nlevels; l++) {
      uint32_t* off_next = c->aff_off[l & 1];
      k_aff_level_counts<<<std::min<unsigned>(nblk(nbp, 256), GMSM_NUM_SMS * 8u), 256, 0, st>>>(c->offsets, nbt, l + 1, c->aff_counts);
      launches++;
      if (int rc = scan_u32(c->aff_counts, off_next, false)) return rc;
      // sum_b ceil(len_b/2) <= (m + #nonempty)/2 and #nonempty <= min(nb, m): non-increasing bound
      const size_t m_next = std::min(m_up, (m_up + std::min<size_t>(nbt, m_up)) / 2 + 1);
      uint32_t B = 8;
      while (B < 128 && (double)B < (double)m_next / ((double)GMSM_NUM_SMS * 512.0 * 4.0)) B <<= 1;
      // warp-interleaved slots: a warp owns 32*B consecutive slots; T = threads = thread totals
      const size_t T = ((m_next + 32 * (size_t)B - 1) / (32 * (size_t)B)) * 32;
      if (T > c->aff_tcap || m_next > ((l & 1) ? c->aff_cap2 : c->aff_cap1))
        return set_err(GMSM_EINVAL, "internal: affine level bound exceeded (level %d, T=%zu, m=%zu)", l, T, m_next);
      A* dst = reinterpret_cast<A*>(c->aff_buf[l & 1]);
      F* pref = reinterpret_cast<F*>(c->aff_pref);
      F* totals = reinterpret_cast<F*>(c->aff_totals);
      F* ps = reinterpret_cast<F*>(c->aff_ps);
      const unsigned NB = nblk(T, PSCAN_TILE);
      if (l == 0)
        k_aff_forward<G, true><<<nblk(T, 128), 128, 0, st>>>(points, c->entries, src_cur, off_cur, off_next, nbt, B, (uint32_t)T, pref, totals);
      else
        k_aff_forward<G, false><<<nblk(T, 128), 128, 0, st>>>(points, c->entries, src_cur, off_cur, off_next, nbt, B, (uint32_t)T, pref, totals);
      k_aff_scan_tiles<G><<<NB, PSCAN_THREADS, 0, st>>>(totals, (uint32_t)T, ps, bp);
      k_aff_scan_top<G><<<1, PSCAN_THREADS, 0, st>>>(bp, NB, bp + bp_stride, bp + 2 * bp_stride);
      if (l == 0)
        k_aff_backward<G, true><<<nblk(T, 128), 128, 0, st>>>(points, c->entries, src_cur, off_cur, off_next, nbt, B, (uint32_t)T, pref, ps, bp + 2 * bp_stride, dst);
      else
        k_aff_backward<G, false><<<nblk(T, 128), 128, 0, st>>>(points, c->entries, src_cur, off_cur, off_next, nbt, B, (uint32_t)T, pref, ps, bp + 2 * bp_stride, dst);
      launches += 4;
      LAUNCH_CHECK();
      src_cur = dst;
      off_cur = off_next;
      m_up = m_next;
    }
    if (nlevels == 0)
      k_aff_to_buckets<G, true><<<std::min<unsigned>(nblk(nbt, 256), GMSM_NUM_SMS * 8u), 256, 0, st>>>(points, c->entries, src_cur, off_cur, nbt, buckets);
    else
      k_aff_to_buckets<G, false><<<std::min<unsigned>(nblk(nbt, 256), GMSM_NUM_SMS * 8u), 256, 0, st>>>(points, c->entries, src_cur, off_cur, nbt, buckets);
    launches++;
    LAUNCH_CHECK();
    mark(4);
  } else {
  // K2: accumulate
    const uint32_t K = c->acc_K ? c->acc_K : pick_K(n, p.nwin);
    const size_t nchunks = (n * (size_t)p.nwin + K - 1) / K;
    if (nchunks > c->max_chunks) return set_err(GMSM_EINVAL, "internal: chunk bound exceeded (%zu > %zu)", nchunks, c->max_chunks);
    CK(cudaMemsetAsync(buckets, 0, (size_t)p.nb_total * sizeof(X), st));
    {
      X* carr = reinterpret_cast<X*>(c->carries[0]);
      const size_t t0 = 2 * (size_t)NPASS;   // timeline slots of the accumulate parts
      tl(t0, st);
      if (SPLIT_W < NPASS) {
        const uint32_t split_bucket = (uint32_t)std::min<uint64_t>((uint64_t)SPLIT_W * range_sz, p.nb_total);
        k_accumulate<G><<<nblk(nchunks, 128), 128, 0, st>>>(points, c->entries, c->offsets, p.nb_total, K, (uint32_t)nchunks,
                                                            buckets, carr, c->carry_ids[0], 1, split_bucket);
        tl(t0 + 1, st);
        CK(cudaStreamWaitEvent(st, c->ev_split[1], 0));   // the remaining windows are scattered
        tl(t0 + 2, st);
        k_accumulate<G><<<nblk(nchunks, 128), 128, 0, st>>>(points, c->entries, c->offsets, p.nb_total, K, (uint32_t)nchunks,
                                                            buckets, carr, c->carry_ids[0], 2, split_bucket);
        tl(t0 + 3, st);
        launches += 2;
        if (timeline) c->tl_parts = 2;
      } else {
        k_accumulate<G><<<nblk(nchunks, 128), 128, 0, st>>>(points, c->entries, c->offsets, p.nb_total, K, (uint32_t)nchunks,
                                                            buckets, carr, c->carry_ids[0], 0, 0);
        tl(t0 + 1, st);
        launches++;
        if (timeline) c->tl_parts = 1;
      }
      LAUNCH_CHECK();
    }
    mark(4);
    // K2b: carry join levels
    {
      size_t n_in = nchunks;
      int cur = 0;
      while (n_in > 1) {
        // the first level carries nearly all the additions (one carry per chunk): a short run length there
        // means more threads for the same work; the later levels see mostly empty slots
        const uint32_t k2 = (cur == 0 && n_in == nchunks) ? c->K2_first : c->K2;
        size_t n_out = (n_in + k2 - 1) / k2;
        if (c->use_quad(n_out))
          k_carry_level<G, true><<<nblk(n_out * 4, 128), 128, 0, st>>>(reinterpret_cast<const X*>(c->carries[cur]), c->carry_ids[cur],
                                                                    (uint32_t)n_in, k2, buckets,
                                                                    reinterpret_cast<X*>(c->carries[cur ^ 1]), c->carry_ids[cur ^ 1]);
        else
          k_carry_level<G, false><<<nblk(n_out, 128), 128, 0, st>>>(reinterpret_cast<const X*>(c->carries[cur]), c->carry_ids[cur],
                                                                   (uint32_t)n_in, k2, buckets,
                                                                   reinterpret_cast<X*>(c->carries[cur ^ 1]), c->carry_ids[cur ^ 1]);
        launches++;
        LAUNCH_CHECK();
        n_in = n_out;
        cur ^= 1;
      }
    }
  }
  if (rmw) {
    k_merge_buckets<G><<<nblk(p.nb_total, 128), 128, 0, st>>>(reinterpret_cast<X*>(c->buckets), buckets, p.nb_total);
    launches++;
    LAUNCH_CHECK();
  }
  mark(5);
  c->last_launches = launches;
  return GMSM_OK;
}

// stage K3: bucket reduction of c->buckets -> W window partials
template <class G>
static int run_bucket_reduce(gmsm_ctx* c, void* d_partials, cudaStream_t st) {
  using F = typename G::F;
  using X = XYZZ<F>;
  const WindowPlan& p = c->plan;
  int launches = 0;
  const bool prof = c->profiling;
  auto mark = [&](int i) { if (prof) cudaEventRecord(c->ev[i], st); };
  X* buckets = reinterpret_cast<X*>(c->buckets);
  {
    const uint32_t S = c->seg_S, L = c->seg_L;
    // window-table mode: one window of nb_total shared buckets
    const int nwin = c->red_windows();
    const uint32_t nb_reg = c->shared ? p.nb_total : p.nb, nb_last = c->shared ? p.nb_total : p.nb_last;
    if (c->use_quad((size_t)nwin * S))
      k_bucket_segments<G, true><<<nblk((size_t)nwin * S * 4, 128), 128, 0, st>>>(buckets, nwin, nb_reg, nb_last, L, S,
                                                                             reinterpret_cast<X*>(c->seg[0]));
    else
      k_bucket_segments<G, false><<<nblk((size_t)nwin * S, 128), 128, 0, st>>>(buckets, nwin, nb_reg, nb_last, L, S,
                                                                          reinterpret_cast<X*>(c->seg[0]));
    launches++;
    LAUNCH_CHECK();
    uint32_t per = S;
    int cur = 0;
    while (per > 1) {
      const bool quad = c->use_quad((size_t)nwin * per);
      const uint32_t R = quad ? 16u : 2u * TREE_THREADS;
      uint32_t outp = (per + R - 1) / R;
      X* dst = (outp == 1) ? reinterpret_cast<X*>(d_partials) : reinterpret_cast<X*>(c->seg[cur ^ 1]);
      if (quad)
        k_sum_groups<G, true><<<nblk((size_t)nwin * outp * 4, 128), 128, 0, st>>>(reinterpret_cast<const X*>(c->seg[cur]), per, R, outp,
                                                                             nwin, dst);
      else
        k_sum_tree<G><<<dim3(outp, (unsigned)nwin), TREE_THREADS, 0, st>>>(reinterpret_cast<const X*>(c->seg[cur]), per, outp, dst);
      launches++;
      LAUNCH_CHECK();
      per = outp;
      cur ^= 1;
    }
    if (S == 1) {
      CK(cudaMemcpyAsync(d_partials, c->seg[0], (size_t)nwin * sizeof(X), cudaMemcpyDeviceToDevice, st));
    }
  }
  mark(6);
  c->last_launches += launches;
  return GMSM_OK;
}

// per-window partial sums of one batch -> d_partials (W xyzz)
template <class G>
static int run_window_sums(gmsm_ctx* c, const void* d_points, const void* d_scalars, size_t n, void* d_partials,
                           cudaStream_t st) {
  if (int rc = run_accumulate<G>(c, d_points, d_scalars, n, 0, st)) return rc;
  return run_bucket_reduce<G>(c, d_partials, st);
}

template <class G>
static int run_finalize(gmsm_ctx* c, const void* d_partials, int nranks, void* d_out, cudaStream_t st) {
  using F = typename G::F;
  if (c->quad_mode > 0)
    k_finalize<G, true><<<1, FIN_THREADS, 0, st>>>(reinterpret_cast<const XYZZ<F>*>(d_partials), nranks, c->red_windows(), c->plan.c,
                                                   reinterpret_cast<XYZZ<F>*>(c->fin_scratch), reinterpret_cast<Jac<F>*>(d_out));
  else
    k_finalize<G, false><<<1, FIN_THREADS, 0, st>>>(reinterpret_cast<const XYZZ<F>*>(d_partials), nranks, c->red_windows(), c->plan.c,
                                                    reinterpret_cast<XYZZ<F>*>(c->fin_scratch), reinterpret_cast<Jac<F>*>(d_out));
  LAUNCH_CHECK();
  return GMSM_OK;
}


template <class G>
static int run_generate(const void* d_base, uint64_t start, size_t n, void* d_out, cudaStream_t st) {
  size_t threads = (n + GEN_M - 1) / GEN_M;
  k_generate_multiples<G><<<nblk(threads, 128), 128, 0, st>>>(reinterpret_cast<const Affine<typename G::F>*>(d_base), start,
                                                             (uint64_t)n, reinterpret_cast<Affine<typename G::F>*>(d_out));
  LAUNCH_CHECK();
  return GMSM_OK;
}

template <class G>
static int run_test_op(int op, const uint32_t* da, const uint32_t* db, uint32_t* dout, size_t n) {
  k_test_op<G><<<nblk(n, 64), 64>>>(op, da, db, dout, (uint32_t)n);
  LAUNCH_CHECK();
  return GMSM_OK;
}

template <class G>
static int run_digits_dump(const void* d_scalars, size_t n, int c, int nwin, uint32_t* dout) {
  k_digits_dump<G><<<nblk(n, 128), 128>>>(reinterpret_cast<const typename G::Fr*>(d_scalars), (uint32_t)n, c, nwin, dout);
  LAUNCH_CHECK();
  return GMSM_OK;
}

template <class G>
static int run_batch_scalar_mul(const void* d_table, const void* d_scalars, size_t n, int c, int nwin, void* d_out, cudaStream_t st) {
  using F = typename G::F;
  k_batch_scalar_mul<G><<<nblk(n, 128), 128, 0, st>>>(reinterpret_cast<const Affine<F>*>(d_table),
                                                    reinterpret_cast<const typename G::Fr*>(d_scalars), (uint32_t)n, c, nwin,
                                                    reinterpret_cast<Affine<F>*>(d_out));
  LAUNCH_CHECK();
  return GMSM_OK;
}

template <class G>
static int run_table_level(const void* d_in, size_t n, int c, void* d_out, cudaStream_t st) {
  using A = Affine<typename G::F>;
  k_table_level<G><<<nblk((n + TAB_M - 1) / TAB_M, 128), 128, 0, st>>>(reinterpret_cast<const A*>(d_in), (uint32_t)n, c,
                                                                       reinterpret_cast<A*>(d_out));
  LAUNCH_CHECK();
  return GMSM_OK;
}

// kzg.ToLagrangeG1 (lagrange_kernels.cuh): logn stage launches, then the finish launch, all on st
template <class G>
static int run_to_lagrange(const void* d_points, size_t n, const uint64_t* w_inv, const uint64_t* n_inv, void* d_out, void* d_work,
                           cudaStream_t st) {
  using F = typename G::F;
  using Fr = typename G::Fr;
  int logn = 0;
  while (((size_t)1 << logn) < n) logn++;
  Fr wi, ni;
  memcpy(wi.l, w_inv, sizeof(Fr));
  memcpy(ni.l, n_inv, sizeof(Fr));
  const LagPowers<G> pw = lag_powers<G>(wi, logn);
  const auto* in = reinterpret_cast<const Affine<F>*>(d_points);
  auto* ws = reinterpret_cast<XYZZ<F>*>(d_work);
  lagrange_schedule(
      n, logn,
      [&](int s, uint64_t threads) {
        if (s == 0)
          k_lag_stage<G, true><<<nblk(threads, 128), 128, 0, st>>>(in, ws, (uint32_t)threads, logn, s, pw);
        else
          k_lag_stage<G, false><<<nblk(threads, 128), 128, 0, st>>>(in, ws, (uint32_t)threads, logn, s, pw);
      },
      [&](uint64_t threads) {
        k_lag_finish<G><<<nblk(threads, 128), 128, 0, st>>>(ws, (uint32_t)n, logn, ni, reinterpret_cast<Affine<F>*>(d_out));
      });
  LAUNCH_CHECK();
  return GMSM_OK;
}

// out[i] = [c r^(start + i)] points[i], 1 <= n < 2^32 (mpc_kernels.cuh): one launch on st
template <class G>
static int run_scale_powers(const void* d_points, size_t n, const uint64_t* c, const uint64_t* r, uint64_t start, void* d_out,
                            cudaStream_t st) {
  using A = Affine<typename G::F>;
  const ScalePowers<G> pw = scale_powers_args<G>(c, r, start);
  scale_powers_schedule(n, [&](uint64_t threads) {
    k_scale_powers<G><<<nblk(threads, 128), 128, 0, st>>>(reinterpret_cast<const A*>(d_points), (uint32_t)n, pw, reinterpret_cast<A*>(d_out));
  });
  LAUNCH_CHECK();
  return GMSM_OK;
}

template <class G>
static bool fr_reduced(const uint64_t* limbs) {
  typename G::Fr x;
  memcpy(x.l, limbs, sizeof(x));
  return fp_is_reduced(x);
}

#define GMSM_CURVE_INFO(G) {G::F::N, G::FrParams::BITS, 4 * G::FrParams::N}
#define GMSM_INSTANTIATE(G, NAME)                                                                  \
  const GroupVTable NAME = {GMSM_CURVE_INFO(G), &run_window_sums<G>, &run_accumulate<G>, &run_bucket_reduce<G>, &run_finalize<G>, &run_generate<G>, \
                            &test_op_sizes<G>, &run_test_op<G>, &run_digits_dump<G>, &run_batch_scalar_mul<G>, &run_table_level<G>, &fr_reduced<G>, &run_scale_powers<G>};
// the G1 groups of the seven pairing curves: also kzg.ToLagrangeG1
#define GMSM_INSTANTIATE_PAIRING_G1(G, NAME)                                                       \
  const GroupVTable NAME = {GMSM_CURVE_INFO(G), &run_window_sums<G>, &run_accumulate<G>, &run_bucket_reduce<G>, &run_finalize<G>, &run_generate<G>, \
                            &test_op_sizes<G>, &run_test_op<G>, &run_digits_dump<G>, &run_batch_scalar_mul<G>, &run_table_level<G>, &fr_reduced<G>, &run_scale_powers<G>, \
                            &run_to_lagrange<G>};

}  // namespace gmsm
