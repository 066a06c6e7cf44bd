// Vector load / store of PODs made of uint32 limbs, shared by the MSM kernels (kernels.cuh) and the Fr FFT kernels
// (fft_kernels.cuh): 16-byte granules where the size allows it (16 B aligned in memory), 8-byte granules otherwise (the
// 10-limb fields of bls24-315 / bls24-317 / bw6-633: 40-byte elements and scalars, 120-byte Jacobian triples -- a multiple
// of 8 and 8-byte aligned like every u64-limb object of the reference).  The choice is made at compile time on sizeof(T).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "hd.cuh"

namespace gmsm {

template <class T>
GMSM_D T load_vec(const T* p) {
  static_assert(sizeof(T) % 8 == 0, "8-byte granules");
  T r;
  uint32_t* w = reinterpret_cast<uint32_t*>(&r);
  if constexpr (sizeof(T) % 16 == 0) {
    const uint4* s = reinterpret_cast<const uint4*>(p);
#pragma unroll
    for (int i = 0; i < (int)(sizeof(T) / 16); i++) {
      uint4 v = s[i];
      w[4 * i + 0] = v.x;
      w[4 * i + 1] = v.y;
      w[4 * i + 2] = v.z;
      w[4 * i + 3] = v.w;
    }
  } else {
    const uint2* s = reinterpret_cast<const uint2*>(p);
#pragma unroll
    for (int i = 0; i < (int)(sizeof(T) / 8); i++) {
      uint2 v = s[i];
      w[2 * i + 0] = v.x;
      w[2 * i + 1] = v.y;
    }
  }
  return r;
}
// read-only path (points and scalars are never written during an MSM): non-coherent loads through the texture
// path, 128 bits wide (LDG.E.128.CONSTANT, the widest global load sm_90a has) where the size allows it.
template <class T>
GMSM_D T load_vec_ro(const T* p) {
  static_assert(sizeof(T) % 8 == 0, "8-byte granules");
  T r;
  uint32_t* w = reinterpret_cast<uint32_t*>(&r);
  if constexpr (sizeof(T) % 16 == 0) {
    const uint4* s = reinterpret_cast<const uint4*>(p);
#pragma unroll
    for (int i = 0; i < (int)(sizeof(T) / 16); i++) {
      uint4 v = __ldg(s + i);
      w[4 * i + 0] = v.x;
      w[4 * i + 1] = v.y;
      w[4 * i + 2] = v.z;
      w[4 * i + 3] = v.w;
    }
  } else {
    const uint2* s = reinterpret_cast<const uint2*>(p);
#pragma unroll
    for (int i = 0; i < (int)(sizeof(T) / 8); i++) {
      uint2 v = __ldg(s + i);
      w[2 * i + 0] = v.x;
      w[2 * i + 1] = v.y;
    }
  }
  return r;
}
template <class T>
GMSM_D void store_vec(T* p, const T& r) {
  static_assert(sizeof(T) % 8 == 0, "8-byte granules");
  const uint32_t* w = reinterpret_cast<const uint32_t*>(&r);
  if constexpr (sizeof(T) % 16 == 0) {
    uint4* d = reinterpret_cast<uint4*>(p);
#pragma unroll
    for (int i = 0; i < (int)(sizeof(T) / 16); i++) d[i] = make_uint4(w[4 * i], w[4 * i + 1], w[4 * i + 2], w[4 * i + 3]);
  } else {
    uint2* d = reinterpret_cast<uint2*>(p);
#pragma unroll
    for (int i = 0; i < (int)(sizeof(T) / 8); i++) d[i] = make_uint2(w[2 * i], w[2 * i + 1]);
  }
}

}  // namespace gmsm
