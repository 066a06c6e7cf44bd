// Next-row N2 (SURVEY.md section 8f): bulk decoding of serialised G1 points on the device -- what stands between an SRS in
// gnark-crypto's standard WriteTo format and the resident bases of the MSM engine.
//
// Replaces (reference): G1Affine.SetBytes / setBytes without the subgroup check (ecc/bn254/marshal.go:858-950,
// ecc/bls12-381/marshal.go:886-1000, and the same code of bls12-377, bls24-315, bls24-317, bw6-633 and bw6-761; the Decoder's
// NoSubgroupChecks path, marshal.go:52-60, which also splits the work in "read X" and "unsafeComputeY", :952-990),
// fp.Element.SetBytesCanonical (fp/element.go:905-925), fp.Sqrt (fp/element.go:1142-1153 for q = 3 mod 4: y = x^((q+1)/4);
// here Tonelli-Shanks for every q, which is that same power when q = 3 mod 4; checked by squaring), LexicographicallyLargest
// (fp/element.go:282-296).
// Wire format: big-endian X (|| Y), canonical (non-Montgomery) values, flag bits in the most significant byte:
//   bn254 (two spare bits, marshal.go:25-31):      00 uncompressed | 10 compressed, smallest y | 11 largest y | 01 infinity
//   bls12-381 / bls12-377 / bls24-315 / bls24-317 / bw6-633 / bw6-761 (three bits, :27-34):
//                                                 000 uncompressed | 010 uncompressed infinity | 100 / 101 compressed | 110 infinity
// A stream is homogeneous (raw: RawBytes points of 2 * fp.Bytes, else Bytes points of fp.Bytes), so each point is read at a
// fixed stride and is infinity only under its own kind's flag: 110 in a compressed stream, 010 in a raw one (bn254: none; its
// RawBytes infinity is the all-zero point, decoded as (0, 0)).  Any other pattern, 010 among compressed points or 110 among
// raw ones included, is "invalid point encoding": the reference would read such a point at the other kind's length.
// One thread per point (decode_kernels.cuh); results are the reference's in-memory G1Affine (Montgomery limbs, infinity = zeroes).
#include <cuda_runtime.h>

#include <cstdint>
#include <cstring>

#include "engine.h"

#include "decode_kernels.cuh"

using namespace gmsm;

static const char* dec_message(int code) {
  switch (code) {
    case DEC_BAD_INFINITY: return "invalid infinity point encoding";                                   // marshal.go:41
    case DEC_BAD_ELEMENT: return "invalid fp.Element encoding";                                        // fp/element.go:920
    case DEC_NO_SQRT: return "invalid compressed coordinate: square root doesn't exist";               // marshal.go:929
    case DEC_NOT_ON_CURVE: return "invalid point: subgroup check failed";                              // marshal.go:946 (on-curve part)
    case DEC_BAD_FLAGS: return "invalid point encoding";                                               // marshal.go:42
  }
  return "decode error";
}

template <class P>
static int run_decode(const void* d_bytes, size_t n, int raw, int check, const DecodeConsts<P>& kc, void* d_out, unsigned long long* d_err,
                      cudaStream_t st) {
  k_g1_decode<P><<<nblk(n, 128), 128, 0, st>>>(reinterpret_cast<const uint8_t*>(d_bytes), (uint32_t)n, raw, check, kc,
                                              reinterpret_cast<Affine<Fp<P>>*>(d_out), d_err);
  CK(cudaGetLastError());
  return GMSM_OK;
}

// bytes (device) -> affine points (device).  *d_first_error (device, 8 bytes) receives (index << 8 | code) of the first bad
// point, or stays all-ones.
extern "C" int gmsm_g1_decode_device(gmsm_curve_t curve, const void* d_bytes, size_t n, int raw, int check_on_curve, void* d_points,
                                     void* d_first_error, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (n > 0xFFFFFF00ull) return set_err(GMSM_EINVAL, "n too large");
  CK(cudaMemsetAsync(d_first_error, 0xFF, 8, st));
  if (n == 0) return GMSM_OK;
  const int rc = with_g1_decode_consts(curve, [&](const auto& kc) {
    return run_decode(d_bytes, n, raw, check_on_curve, kc, d_points, (unsigned long long*)d_first_error, st);
  });
  if (rc < 0) return set_err(GMSM_EINVAL, "gmsm_g1_decode: G1 groups of the pairing curves only (curve id %d)", (int)curve);
  return rc;
}

// host bytes -> host points (Go memory layout), n points of a homogeneous stream (raw = 1: RawBytes, 0: Bytes)
extern "C" int gmsm_g1_decode(gmsm_curve_t curve, const uint8_t* bytes, size_t n, int raw, int check_on_curve, uint64_t* out_points) {
  size_t ab = gmsm_affine_bytes(curve);
  if (!ab) return set_err(GMSM_EINVAL, "unknown curve id %d", (int)curve);
  if (int rc = use_device(default_device())) return rc;
  if (n == 0) return GMSM_OK;
  const size_t in_bytes = n * (raw ? ab : ab / 2);
  DevBuf d_in, d_out, d_err;
  if (cudaMalloc(&d_in.p, in_bytes) != cudaSuccess || cudaMalloc(&d_out.p, n * ab) != cudaSuccess || cudaMalloc(&d_err.p, 8) != cudaSuccess)
    return set_err(GMSM_ENOMEM, "gmsm_g1_decode: device allocation failed");
  int rc = GMSM_OK;
  unsigned long long first = ~0ull;
  cudaError_t ce = cudaMemcpy(d_in.p, bytes, in_bytes, cudaMemcpyHostToDevice);
  if (ce == cudaSuccess) rc = gmsm_g1_decode_device(curve, d_in.p, n, raw, check_on_curve, d_out.p, d_err.p, nullptr);
  if (ce == cudaSuccess && rc == GMSM_OK) ce = cudaMemcpy(out_points, d_out.p, n * ab, cudaMemcpyDeviceToHost);
  if (ce == cudaSuccess && rc == GMSM_OK) ce = cudaMemcpy(&first, d_err.p, 8, cudaMemcpyDeviceToHost);
  if (ce != cudaSuccess) return set_err(GMSM_ECUDA, "gmsm_g1_decode: %s", cudaGetErrorString(ce));
  if (rc != GMSM_OK) return rc;
  if (first != ~0ull) return set_err(GMSM_EINVAL, "point %llu: %s", first >> 8, dec_message((int)(first & 0xFF)));
  return GMSM_OK;
}
