// Device side of the Fr FFT (next-row N3): the kernels of fft.cu, in a header of their own so that the CPU kernel
// emulation of tests/emu/ can compile and run them too (tests/test_emu_kernels.py); fft.cu includes this file verbatim.
// See fft.cu for the reference citations (ecc/bn254/fr/fft/fft.go:31-190, 195+, 262+, bitreverse.go:17-42).
#pragma once
#include <cuda_runtime.h>

#include "field.cuh"
#include "vec_io.cuh"

using namespace gmsm;

namespace {

// stages fused in shared memory: 2^10 elements per block, 32 KB for the 4-limb fields, 40 KB for bw6-633 and 48 KB for bw6-761
// (48 KB is the default dynamic shared-memory limit, so no cudaFuncSetAttribute opt-in is needed).  Elements move through
// load_vec / store_vec: 16-byte accesses for 32- and 48-byte elements, 8-byte ones for the 40-byte bw6-633 element.
constexpr int TILE_LOG = 10;
constexpr int TILE = 1 << TILE_LOG;

// tw[t] = w^t for t < count, from pw[k] = w^(2^k)
template <class P>
__global__ void k_fft_powers(Fp<P>* __restrict__ tw, uint64_t count, const Fp<P>* __restrict__ pw, int nbits) {
  for (uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; t < count; t += (uint64_t)gridDim.x * blockDim.x) {
    Fp<P> acc = Fp<P>::one();
    for (int k = 0; k < nbits; k++)
      if ((t >> k) & 1ull) acc = fp_mul(acc, load_vec(pw + k));
    store_vec(tw + t, acc);
  }
}

// one DIF stage with half-size h >= TILE: (x, y) -> (x + y, (x - y) * w^(j * stride))
template <class P>
__global__ void k_fft_dif_stage(Fp<P>* __restrict__ a, const Fp<P>* __restrict__ tw, uint64_t half_n, uint64_t h, uint64_t stride) {
  for (uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; t < half_n; t += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t j = t & (h - 1), blk = t / h;
    const uint64_t i0 = blk * 2 * h + j, i1 = i0 + h;
    Fp<P> x = load_vec(a + i0), y = load_vec(a + i1);
    store_vec(a + i0, fp_add(x, y));
    Fp<P> d = fp_sub(x, y);
    store_vec(a + i1, j ? fp_mul(d, load_vec(tw + j * stride)) : d);
  }
}
// one DIT stage with half-size h >= TILE: (x, y) -> (x + y w, x - y w)
template <class P>
__global__ void k_fft_dit_stage(Fp<P>* __restrict__ a, const Fp<P>* __restrict__ tw, uint64_t half_n, uint64_t h, uint64_t stride) {
  for (uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; t < half_n; t += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t j = t & (h - 1), blk = t / h;
    const uint64_t i0 = blk * 2 * h + j, i1 = i0 + h;
    Fp<P> x = load_vec(a + i0), y = load_vec(a + i1);
    if (j) y = fp_mul(y, load_vec(tw + j * stride));
    store_vec(a + i0, fp_add(x, y));
    store_vec(a + i1, fp_sub(x, y));
  }
}

// the stages with half-size < tile (tile = min(n, TILE)) on one tile per block, in shared memory.
// DIF: the LAST log2(tile) stages; DIT: the FIRST log2(tile) stages.  blockDim.x = tile / 2.
template <class P, bool IS_DIF>
__global__ void k_fft_tile(Fp<P>* __restrict__ a, const Fp<P>* __restrict__ tw, uint64_t n, uint32_t tile) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Fp<P>* s = reinterpret_cast<Fp<P>*>(smem_raw);
  const uint64_t base = (uint64_t)blockIdx.x * tile;
  const uint32_t tid = threadIdx.x, half = tile >> 1;
  store_vec(s + tid, load_vec(a + base + tid));
  store_vec(s + tid + half, load_vec(a + base + tid + half));
  __syncthreads();
  if (IS_DIF) {
    for (uint32_t h = half; h >= 1; h >>= 1) {
      const uint32_t j = tid & (h - 1), blk = tid / h;
      const uint32_t i0 = blk * 2 * h + j, i1 = i0 + h;
      Fp<P> x = load_vec(s + i0), y = load_vec(s + i1);
      Fp<P> d = fp_sub(x, y);
      if (j) d = fp_mul(d, load_vec(tw + (uint64_t)j * ((n >> 1) / h)));
      store_vec(s + i0, fp_add(x, y));
      store_vec(s + i1, d);
      __syncthreads();
    }
  } else {
    for (uint32_t h = 1; h <= half; h <<= 1) {
      const uint32_t j = tid & (h - 1), blk = tid / h;
      const uint32_t i0 = blk * 2 * h + j, i1 = i0 + h;
      Fp<P> x = load_vec(s + i0), y = load_vec(s + i1);
      if (j) y = fp_mul(y, load_vec(tw + (uint64_t)j * ((n >> 1) / h)));
      store_vec(s + i0, fp_add(x, y));
      store_vec(s + i1, fp_sub(x, y));
      __syncthreads();
    }
  }
  store_vec(a + base + tid, load_vec(s + tid));
  store_vec(a + base + tid + half, load_vec(s + tid + half));
}

// a[i] *= scalar * u^(e(i)), e(i) = i or bitrev(i); pw[k] = u^(2^k) (nbits entries); use_shift = 0: scalar only
template <class P>
__global__ void k_fft_scale(Fp<P>* __restrict__ a, uint64_t n, int logn, const Fp<P>* __restrict__ pw, int use_shift, int bitrev,
                            Fp<P> scalar, int use_scalar) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    Fp<P> v = load_vec(a + i);
    if (use_scalar) v = fp_mul(v, scalar);
    if (use_shift) {
      const uint64_t e = bitrev ? (logn ? (__brevll(i) >> (64 - logn)) : 0ull) : i;
      for (int k = 0; k < logn; k++)
        if ((e >> k) & 1ull) v = fp_mul(v, load_vec(pw + k));
    }
    store_vec(a + i, v);
  }
}

template <class P>
__global__ void k_fft_bit_reverse(Fp<P>* __restrict__ a, uint64_t n, int logn) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t r = logn ? (__brevll(i) >> (64 - logn)) : 0;
    if (r > i) {
      Fp<P> x = load_vec(a + i), y = load_vec(a + r);
      store_vec(a + i, y);
      store_vec(a + r, x);
    }
  }
}

}  // namespace
