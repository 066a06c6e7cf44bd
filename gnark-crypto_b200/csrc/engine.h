// Shared host-side declarations of the engine: context, error plumbing, per-group function table.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/gmsm.h"
#include "groups.cuh"

namespace gmsm {

int set_err(int code, const char* fmt, ...);

#define CK(call)                                                                                   \
  do {                                                                                             \
    cudaError_t e_ = (call);                                                                       \
    if (e_ != cudaSuccess) {                                                                       \
      return ::gmsm::set_err(e_ == cudaErrorMemoryAllocation ? GMSM_ENOMEM                          \
                     : (e_ == cudaErrorNoDevice || e_ == cudaErrorInsufficientDriver) ? GMSM_ENODEV \
                                                                                       : GMSM_ECUDA, \
                     "%s:%d %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_));            \
    }                                                                                              \
  } while (0)

struct CurveInfo {
  int coord_words;  // u32 words of one coordinate-field element
  int fr_bits;
  int scalar_bytes; // one fr.Element: 32 (4 x uint64), 48 for bw6-761 (6 x uint64)
};

// GMSM_ENODEV when the process sees no CUDA device; GMSM_EINVAL with range_fmt (given the id and the device count) when
// `device` is not one of them; otherwise `device` is made current (gmsm.cu)
int use_device(int device, const char* range_fmt = "device %d out of range (%d devices)");
// the device of the entry points that take none: GMSM_DEVICE, default 0
int default_device();

struct DevBuf {   // a device allocation freed on every exit path (the CK macro returns early on errors)
  void* p = nullptr;
  ~DevBuf() { if (p) cudaFree(p); }
  template <class T> T* as() { return reinterpret_cast<T*>(p); }
};

}  // namespace gmsm

struct gmsm_ctx {
  int curve = 0;
  int device = 0;
  size_t max_n = 0;
  gmsm::CurveInfo ci{};
  gmsm::WindowPlan plan{};
  // window-table mode (gmsm_ctx_create_tables): the point operand is a table of W rows, row j = 2^(c*j) * bases,
  // all windows share one bucket set of plan.nb_total = max(nb, nb_last) buckets, the bucket reduction and the
  // finalize see a single window.  tab_stride = points per table row (set by the caller before each accumulate).
  bool shared = false;
  uint32_t tab_stride = 0;
  int table_passes = 0;   // bucket-range passes of the shared scatter (0 = from the entry count; GMSM_TABLE_PASSES)
  int red_windows() const { return shared ? 1 : plan.nwin; }   // partials per call
  // chunking
  uint32_t acc_K = 0;       // accumulate chunk length forced by GMSM_ACC_K (0 = pick_K)
  uint32_t K2 = 16;         // items per thread of the later carry levels (GMSM_K2)
  uint32_t K2_first = 4;    // items per thread of the first carry level (GMSM_K2_FIRST): 4x the threads for the level that
                            // holds nearly all the carry additions (faster at bn254 G1 2^24)
  int k1_mode = -1;         // counting-sort mode forced by GMSM_K1_MODE: 0 plain, 1 rank, -1 = chosen per call by k_skew_probe
  // the GMSM_* experiment knobs this context was built under (knob_signature() in gmsm.cu): the host entry points keep a
  // context between calls and build a new one when the environment no longer matches
  std::string knobs;
  uint32_t seg_L = 32, seg_S = 0;
  // lane-parallel tail (quad.cuh): one QUAD of lanes per chain instead of one thread.  Slower than the serial form for the
  // 8- and 12-limb groups, so it is OFF unless GMSM_QUAD=1 asks for it
  // (GMSM_QUAD_MAX then bounds the number of chains a stage may have to use it).
  int quad_mode = 0;
  size_t quad_max_items = (size_t)1 << 40;
  bool use_quad(size_t items) const { return quad_mode > 0 && items <= quad_max_items; }
  // device workspace
  uint32_t* hist = nullptr;      // nb_total + 1 (+pad)
  uint32_t* offsets = nullptr;   // nb_total + 1
  uint32_t* block_sums = nullptr;
  uint32_t* entries = nullptr;   // max_n * W (+pad)
  uint32_t* digits = nullptr;    // max_n * W, chunk-major (digits[j*n + i])
  uint32_t* ranks = nullptr;     // max_n * W, same layout: position of the entry inside its bucket (numbered by K1's atomics)
  void* buckets = nullptr;       // nb_total xyzz
  void* buckets2 = nullptr;      // scratch buckets of a follow-up batch (pipelined calls), allocated on demand
  void* carries[2] = {nullptr, nullptr};
  uint32_t* carry_ids[2] = {nullptr, nullptr};
  void* seg[2] = {nullptr, nullptr};
  // batch-affine accumulation variant (affine_kernels.cuh); selected per context with GMSM_AFFINE=1 (default off)
  bool affine = false;
  void* aff_buf[2] = {nullptr, nullptr};   // level outputs, ping-pong (affine points)
  void* aff_pref = nullptr;                // running products before each denominator
  void* aff_totals = nullptr;              // per-thread total products
  void* aff_ps = nullptr;                  // per-thread prefix*suffix products inside a scan tile
  void* aff_bp = nullptr;                  // per-tile products, their exclusive prefixes, their inverses (3 arrays)
  uint32_t* aff_off[2] = {nullptr, nullptr};
  uint32_t* aff_counts = nullptr;
  uint32_t* aff_maxlen = nullptr;          // device
  uint32_t* aff_maxlen_host = nullptr;     // pinned
  size_t aff_cap1 = 0, aff_cap2 = 0, aff_tcap = 0;
  void* win_partials = nullptr;  // W xyzz (own result for single-rank msm)
  void* fin_scratch = nullptr;   // W xyzz
  size_t max_chunks = 0;
  size_t ws_bytes = 0;
  int last_launches = 0;
  int profiling = 0;                   // 1: stage events (ev); 2: also the scatter / accumulate timeline (tl_ev)
  cudaEvent_t ev[9] = {};
  // timeline of the last profiled call at level 2: events before and after every scatter pass (2 per pass, on the stream it
  // ran on), then before / after accumulate part 1 (or the only part) and part 2 -- part 2's "before" is recorded after the
  // wait for the auxiliary stream.  Created on first use.
  std::vector<cudaEvent_t> tl_ev;
  int tl_npass = 0, tl_split = 0, tl_parts = 0;
  int split_w = 4;                     // windows scattered before the accumulate starts (GMSM_SPLIT_W)
  int split_tab = 1;                   // the same for the bucket-range passes of the window-table mode
  cudaStream_t aux = nullptr;          // auxiliary stream: scatter of the later windows under the accumulate
  cudaEvent_t ev_split[2] = {};
  // completion of the last call enqueued on this context: every device-level entry point makes its stream wait for it
  // before touching the shared workspace, so calls from different streams / threads queue up instead of overlapping
  cudaEvent_t ev_done = nullptr;
  bool have_stage = false;
  std::mutex mu;
};

template <class T>
static inline cudaError_t dmalloc(T** p, size_t bytes, size_t* acc) {
  *acc += bytes;
  return cudaMalloc((void**)p, bytes ? bytes : 16);
}

static inline uint32_t pick_K(size_t n, int nwin) {
  // chunk length of the accumulate kernel: long enough to amortise the per-chunk bucket search and
  // flush, short enough to fill the SMs x 512 threads several times over
  double total = (double)n * nwin;
  double k = total / ((double)GMSM_NUM_SMS * 512.0 * 8.0);
  uint32_t K = 4;
  while (K < 256 && (double)K < k) K <<= 1;
  return K;
}


namespace gmsm {

static inline unsigned nblk(size_t n, unsigned t) { return (unsigned)((n + t - 1) / t); }

// one table per (curve, group); each lives in its own translation unit (inst_*.cu) so the four
// heavy template instantiations compile in parallel
struct GroupVTable {
  CurveInfo ci;   // the sizes of the group's types (GMSM_INSTANTIATE)
  int (*window_sums)(gmsm_ctx*, const void* d_points, const void* d_scalars, size_t n, void* d_partials, cudaStream_t);
  int (*accumulate)(gmsm_ctx*, const void* d_points, const void* d_scalars, size_t n, int rmw, cudaStream_t);
  int (*bucket_reduce)(gmsm_ctx*, void* d_partials, cudaStream_t);
  int (*finalize)(gmsm_ctx*, const void* d_partials, int nranks, void* d_out, cudaStream_t);
  int (*generate)(const void* d_base, uint64_t start, size_t n, void* d_out, cudaStream_t);
  void (*test_op_sizes)(int op, int* wa, int* wb, int* wo);
  int (*test_op)(int op, const uint32_t* da, const uint32_t* db, uint32_t* dout, size_t n);
  int (*digits_dump)(const void* d_scalars, size_t n, int c, int nwin, uint32_t* dout);
  int (*batch_scalar_mul)(const void* d_table, const void* d_scalars, size_t n, int c, int nwin, void* d_out, cudaStream_t);
  int (*table_level)(const void* d_in, size_t n, int c, void* d_out, cudaStream_t);   // out[i] = 2^c * in[i]
  bool (*fr_reduced)(const uint64_t* limbs);   // an fr.Element (Montgomery u64 limbs) below the scalar field's modulus
  // out[i] = [c r^(start + i)] points[i] for 1 <= n < 2^32 affine points (mpc_kernels.cuh), affine normal form; c, r reduced
  // Montgomery fr limbs; d_out may equal d_points
  int (*scale_powers)(const void* d_points, size_t n, const uint64_t* c, const uint64_t* r, uint64_t start, void* d_out, cudaStream_t);
  // kzg.ToLagrangeG1 (lagrange_kernels.cuh) on n = 2^k >= 2 affine points: w_inv = fr.Generator(n)^-1 and n_inv = 1/n as
  // Montgomery fr limbs, d_work holds n extended-Jacobian points.  Null except for the G1 groups of the pairing curves.
  int (*to_lagrange)(const void* d_points, size_t n, const uint64_t* w_inv, const uint64_t* n_inv, void* d_out, void* d_work,
                     cudaStream_t);
};
// fr.Generator(n)^-1 and 1/n of the scalar field fr_field (GMSM_FR_*) as Montgomery u64 limbs, n a power of two (fft.cu); the
// error of fr.Generator past maxOrderRoot
int fr_domain_inverses(int fr_field, uint64_t n, uint64_t* w_inv, uint64_t* n_inv);
extern const GroupVTable vt_bn254_g1, vt_bn254_g2, vt_bls12381_g1, vt_bls12381_g2, vt_bls12377_g1, vt_bls12377_g2, vt_secp256k1_g1,
    vt_bw6761_g1, vt_bw6761_g2, vt_bls24315_g1, vt_bls24317_g1, vt_bw6633_g1, vt_bw6633_g2;

}  // namespace gmsm
