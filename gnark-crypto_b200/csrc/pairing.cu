// Pairings of bn254 and bls12-381 on the device: MillerLoop, FinalExponentiation and Pair (ecc/bn254/pairing.go,
// ecc/bls12-381/pairing.go).  Kernels and launch order: pairing_kernels.cuh.  The other pairing curves need other towers or line
// shapes (bls12-377: v^3 = u; bw6: Fp6 over Fp3; bls24: Fp24) and are refused with GMSM_EINVAL.
#include <cuda_runtime.h>

#include <cstdint>

#include "engine.h"

#include "pairing_kernels.cuh"
#include "tower_testops.cuh"

using namespace gmsm;

template <class F>
static int with_pairing_field(gmsm_curve_t curve, F f) {
  if (curve == GMSM_BN254_G1) return f(bn254_fp{});
  if (curve == GMSM_BLS12381_G1) return f(bls12381_fp{});
  return set_err(GMSM_EINVAL, "pairing: bn254 and bls12-381 only (curve id %d; pass the curve's G1 id)", (int)curve);
}

static size_t gt_bytes(gmsm_curve_t curve) {
  return curve == GMSM_BN254_G1 ? 12 * 32 : curve == GMSM_BLS12381_G1 ? 12 * 48 : 0;
}

extern "C" size_t gmsm_pairing_workspace_bytes(gmsm_curve_t curve, size_t n) {
  return gt_bytes(curve) * (n ? pairing_work_elems(n, PAIRING_CHUNK) : 0);
}

template <class P>
static int run_miller(const void* d_P, const void* d_Q, size_t n, void* d_work, cudaStream_t st) {
  using G = Fp12<P>;
  G* w = reinterpret_cast<G*>(d_work);
  const auto* pts = reinterpret_cast<const Affine<Fp<P>>*>(d_P);
  const auto* qs = reinterpret_cast<const Affine<Fp2<P>>*>(d_Q);
  const size_t acc = pairing_acc_index(n, PAIRING_CHUNK);
  cudaError_t ce = cudaSuccess;
  pairing_schedule(
      n, PAIRING_CHUNK,
      [&](size_t off, size_t m, size_t dst) {
        k_miller_loop<P><<<nblk(m, PAIRING_THREADS), PAIRING_THREADS, 0, st>>>(pts + off, qs + off, (uint32_t)m, w + dst);
        if (ce == cudaSuccess) ce = cudaGetLastError();
      },
      [&](size_t src, size_t m, size_t dst) {
        k_gt_reduce<P><<<nblk((m + 1) / 2, PAIRING_THREADS), PAIRING_THREADS, 0, st>>>(w + src, (uint32_t)m, w + dst);
        if (ce == cudaSuccess) ce = cudaGetLastError();
      },
      [&](size_t src, bool first) {
        k_gt_accumulate<P><<<1, 1, 0, st>>>(w + acc, w + src, (int)first);
        if (ce == cudaSuccess) ce = cudaGetLastError();
      });
  CK(ce);
  return GMSM_OK;
}

static int check_args(const char* name, gmsm_curve_t curve, const void* a, const void* b, const void* c, size_t n) {
  if (!gt_bytes(curve))
    return set_err(GMSM_EINVAL, "%s: bn254 and bls12-381 only (curve id %d; pass the curve's G1 id)", name, (int)curve);
  if (n == 0) return set_err(GMSM_EINVAL, "%s: invalid inputs sizes", name);
  if (n > 0xFFFFFFFFull) return set_err(GMSM_EINVAL, "%s: n too large", name);
  if (!a || !b || !c) return set_err(GMSM_EINVAL, "%s: null pointer", name);
  return GMSM_OK;
}

// d_out (one GT element) = MillerLoop(P, Q); d_work holds gmsm_pairing_workspace_bytes(curve, n) bytes
extern "C" int gmsm_pairing_miller_loop_device(gmsm_curve_t curve, const void* d_P, const void* d_Q, size_t n, void* d_out, void* d_work,
                                               void* stream) {
  if (int rc = check_args("gmsm_pairing_miller_loop", curve, d_P, d_Q, d_out, n)) return rc;
  if (!d_work || ((uintptr_t)d_P & 15) || ((uintptr_t)d_Q & 15) || ((uintptr_t)d_out & 15) || ((uintptr_t)d_work & 15))
    return set_err(GMSM_EINVAL, "gmsm_pairing_miller_loop: points, output and workspace must be 16-byte aligned device buffers");
  cudaStream_t st = (cudaStream_t)stream;
  return with_pairing_field(curve, [&](auto p) {
    using P = decltype(p);
    if (int rc = run_miller<P>(d_P, d_Q, n, d_work, st)) return rc;
    CK(cudaMemcpyAsync(d_out, reinterpret_cast<Fp12<P>*>(d_work) + pairing_acc_index(n, PAIRING_CHUNK), sizeof(Fp12<P>),
                       cudaMemcpyDeviceToDevice, st));
    return (int)GMSM_OK;
  });
}

// d_out = FinalExponentiation(d_z[0], d_z[1..k)); nothing is allocated
extern "C" int gmsm_pairing_final_exp_device(gmsm_curve_t curve, const void* d_z, size_t k, void* d_out, void* stream) {
  if (int rc = check_args("gmsm_pairing_final_exp", curve, d_z, d_out, d_out, k)) return rc;
  if (((uintptr_t)d_z & 15) || ((uintptr_t)d_out & 15))
    return set_err(GMSM_EINVAL, "gmsm_pairing_final_exp: elements must be 16-byte aligned device buffers");
  cudaStream_t st = (cudaStream_t)stream;
  return with_pairing_field(curve, [&](auto p) {
    using P = decltype(p);
    k_final_exp<P><<<1, 1, 0, st>>>(reinterpret_cast<const Fp12<P>*>(d_z), (uint32_t)k, reinterpret_cast<Fp12<P>*>(d_out));
    CK(cudaGetLastError());
    return (int)GMSM_OK;
  });
}

// d_out = Pair(P, Q) = FinalExponentiation(MillerLoop(P, Q)); d_work as for the Miller loop
extern "C" int gmsm_pair_device(gmsm_curve_t curve, const void* d_P, const void* d_Q, size_t n, void* d_out, void* d_work, void* stream) {
  if (int rc = check_args("gmsm_pair", curve, d_P, d_Q, d_out, n)) return rc;
  if (!d_work || ((uintptr_t)d_P & 15) || ((uintptr_t)d_Q & 15) || ((uintptr_t)d_out & 15) || ((uintptr_t)d_work & 15))
    return set_err(GMSM_EINVAL, "gmsm_pair: points, output and workspace must be 16-byte aligned device buffers");
  cudaStream_t st = (cudaStream_t)stream;
  return with_pairing_field(curve, [&](auto p) {
    using P = decltype(p);
    if (int rc = run_miller<P>(d_P, d_Q, n, d_work, st)) return rc;
    const auto* acc = reinterpret_cast<const Fp12<P>*>(d_work) + pairing_acc_index(n, PAIRING_CHUNK);
    k_final_exp<P><<<1, 1, 0, st>>>(acc, 1u, reinterpret_cast<Fp12<P>*>(d_out));
    CK(cudaGetLastError());
    return (int)GMSM_OK;
  });
}

// host entries: one upload, the device entry on the default stream, one download
extern "C" int gmsm_pairing_miller_loop(gmsm_curve_t curve, const uint64_t* P, const uint64_t* Q, size_t n, uint64_t* out) {
  if (int rc = check_args("gmsm_pairing_miller_loop", curve, P, Q, out, n)) return rc;
  if (int rc = use_device(default_device())) return rc;
  const size_t ab = gmsm_affine_bytes(curve), gb = gt_bytes(curve);
  DevBuf dP, dQ, dW, dO;
  if (cudaMalloc(&dP.p, n * ab) != cudaSuccess || cudaMalloc(&dQ.p, 2 * n * ab) != cudaSuccess ||
      cudaMalloc(&dW.p, gmsm_pairing_workspace_bytes(curve, n)) != cudaSuccess || cudaMalloc(&dO.p, gb) != cudaSuccess)
    return set_err(GMSM_ENOMEM, "gmsm_pairing_miller_loop: device allocation failed");
  CK(cudaMemcpy(dP.p, P, n * ab, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(dQ.p, Q, 2 * n * ab, cudaMemcpyHostToDevice));
  if (int rc = gmsm_pairing_miller_loop_device(curve, dP.p, dQ.p, n, dO.p, dW.p, nullptr)) return rc;
  CK(cudaMemcpy(out, dO.p, gb, cudaMemcpyDeviceToHost));
  return GMSM_OK;
}

extern "C" int gmsm_pairing_final_exp(gmsm_curve_t curve, const uint64_t* z, size_t k, uint64_t* out) {
  if (int rc = check_args("gmsm_pairing_final_exp", curve, z, out, out, k)) return rc;
  if (int rc = use_device(default_device())) return rc;
  const size_t gb = gt_bytes(curve);
  DevBuf dZ, dO;
  if (cudaMalloc(&dZ.p, k * gb) != cudaSuccess || cudaMalloc(&dO.p, gb) != cudaSuccess)
    return set_err(GMSM_ENOMEM, "gmsm_pairing_final_exp: device allocation failed");
  CK(cudaMemcpy(dZ.p, z, k * gb, cudaMemcpyHostToDevice));
  if (int rc = gmsm_pairing_final_exp_device(curve, dZ.p, k, dO.p, nullptr)) return rc;
  CK(cudaMemcpy(out, dO.p, gb, cudaMemcpyDeviceToHost));
  return GMSM_OK;
}

extern "C" int gmsm_pair(gmsm_curve_t curve, const uint64_t* P, const uint64_t* Q, size_t n, uint64_t* out) {
  if (int rc = check_args("gmsm_pair", curve, P, Q, out, n)) return rc;
  if (int rc = use_device(default_device())) return rc;
  const size_t ab = gmsm_affine_bytes(curve), gb = gt_bytes(curve);
  DevBuf dP, dQ, dW, dO;
  if (cudaMalloc(&dP.p, n * ab) != cudaSuccess || cudaMalloc(&dQ.p, 2 * n * ab) != cudaSuccess ||
      cudaMalloc(&dW.p, gmsm_pairing_workspace_bytes(curve, n)) != cudaSuccess || cudaMalloc(&dO.p, gb) != cudaSuccess)
    return set_err(GMSM_ENOMEM, "gmsm_pair: device allocation failed");
  CK(cudaMemcpy(dP.p, P, n * ab, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(dQ.p, Q, 2 * n * ab, cudaMemcpyHostToDevice));
  if (int rc = gmsm_pair_device(curve, dP.p, dQ.p, n, dO.p, dW.p, nullptr)) return rc;
  CK(cudaMemcpy(out, dO.p, gb, cudaMemcpyDeviceToHost));
  return GMSM_OK;
}

// test hook: k_tower_op (tower_testops.cuh) over n host elements
extern "C" int gmsm_test_tower_op(gmsm_curve_t curve, int op, const uint64_t* a, const uint64_t* b, uint64_t* out, size_t n) {
  return with_pairing_field(curve, [&](auto p) {
    using P = decltype(p);
    int wa, wb, wo;
    tower_op_sizes<P>(op, &wa, &wb, &wo);
    if (wo == 0) return set_err(GMSM_EINVAL, "gmsm_test_tower_op: op %d is not an op of curve id %d", op, (int)curve);
    if (n == 0) return (int)GMSM_OK;
    if (n > 0xFFFFFFFFull || !a || (wb && !b) || !out) return set_err(GMSM_EINVAL, "gmsm_test_tower_op: invalid arguments");
    if (int rc = use_device(default_device())) return rc;
    const size_t e = sizeof(Fp2<P>);
    DevBuf da, db, dout;
    if (cudaMalloc(&da.p, n * wa * e) != cudaSuccess || cudaMalloc(&db.p, n * (wb ? wb : 1) * e) != cudaSuccess ||
        cudaMalloc(&dout.p, n * wo * e) != cudaSuccess)
      return set_err(GMSM_ENOMEM, "gmsm_test_tower_op: device allocation failed");
    CK(cudaMemcpy(da.p, a, n * wa * e, cudaMemcpyHostToDevice));
    if (wb) CK(cudaMemcpy(db.p, b, n * wb * e, cudaMemcpyHostToDevice));
    k_tower_op<P><<<nblk(n, PAIRING_THREADS), PAIRING_THREADS>>>(op, da.as<Fp2<P>>(), db.as<Fp2<P>>(), dout.as<Fp2<P>>(), (uint32_t)n);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(out, dout.p, n * wo * e, cudaMemcpyDeviceToHost));
    return (int)GMSM_OK;
  });
}
