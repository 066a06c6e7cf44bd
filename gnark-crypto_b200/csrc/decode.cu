// Next-row N2 (SURVEY.md section 8f): bulk (de)serialisation of points on the device -- what stands between an SRS or a
// powers-of-tau transcript in gnark-crypto's standard WriteTo format and the resident points of the MSM engine and of mpcsetup.
//
// Replaces (reference): G1Affine.SetBytes / setBytes without the subgroup check (ecc/bn254/marshal.go:858-950,
// ecc/bls12-381/marshal.go:886-1000, and the same code of bls12-377, bls24-315, bls24-317, bw6-633 and bw6-761; the Decoder's
// NoSubgroupChecks path, marshal.go:52-60, which also splits the work in "read X" and "unsafeComputeY", :952-990),
// fp.Element.SetBytesCanonical (fp/element.go:905-925), fp.Sqrt (fp/element.go:1142-1153 for q = 3 mod 4: y = x^((q+1)/4);
// here Tonelli-Shanks for every q, which is that same power when q = 3 mod 4; checked by squaring), LexicographicallyLargest
// (fp/element.go:282-296).
// G2Affine.setBytes without the subgroup check (bn254 marshal.go:1116-1216, bls12-381 :1160+, bls12-377 the same) over Fp2 for
// bn254, bls12-381 and bls12-377: y^2 = x^3 + b' with the twist's bTwistCurveCoeff (bn254.go:109, bls12-381.go:104,
// bls12-377.go:105); "no root" decided by the norm as E2.Legendre does, the root by the complex method over Tonelli-Shanks
// (any root serves: the sign is then fixed by E2.LexicographicallyLargest, A1 or A0 when A1 = 0; internal/fptower/e2.go).  The
// G2 groups of bw6-761 and bw6-633 are curves over Fp (b' = 4 and 8, bw6-761.go:95, bw6-633.go:84) and go through the G1 kernel.
// G1Affine / G2Affine Bytes and RawBytes (marshal.go:801-846, :1051-1100) for the twelve G1 and G2 groups of the seven pairing
// curves: canonical big-endian X (|| Y), coordinates over Fp2 as A1 || A0; Bytes sets the smallest / largest / infinity flag,
// RawBytes writes infinity as mUncompressedInfinity and zeroes (bn254: all zeroes).
// Wire format: big-endian X (|| Y), canonical (non-Montgomery) values, flag bits in the most significant byte (of X.A1 for Fp2):
//   bn254 (two spare bits, marshal.go:25-31):      00 uncompressed | 10 compressed, smallest y | 11 largest y | 01 infinity
//   bls12-381 / bls12-377 / bls24-315 / bls24-317 / bw6-633 / bw6-761 (three bits, :27-34):
//                                                 000 uncompressed | 010 uncompressed infinity | 100 / 101 compressed | 110 infinity
// A stream is homogeneous (raw: RawBytes points of 2 * the coordinate's bytes, else Bytes points of one coordinate), so each
// point is read at a fixed stride and is infinity only under its own kind's flag: 110 in a compressed stream, 010 in a raw one
// (bn254: none; its RawBytes infinity is the all-zero point, decoded as (0, 0)).  Any other pattern, 010 among compressed points
// or 110 among raw ones included, is "invalid point encoding": the reference would read such a point at the other kind's length.
// One thread per point (decode_kernels.cuh, marshal_kernels.cuh); decoded points are the reference's in-memory G1Affine /
// G2Affine (Montgomery limbs, {A0, A1} per Fp2 coordinate, infinity = zeroes).  Encoding stages each block's output in shared
// memory so that the global writes are coalesced.
#include <cuda_runtime.h>

#include <cstdint>
#include <cstring>

#include "engine.h"

#include "decode_kernels.cuh"
#include "marshal_kernels.cuh"

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
template <class P>
static int run_decode(const void* d_bytes, size_t n, int raw, int check, const G2DecodeConsts<P>& kc, void* d_out, unsigned long long* d_err,
                      cudaStream_t st) {
  k_g2_decode<P><<<nblk(n, 128), 128, 0, st>>>(reinterpret_cast<const uint8_t*>(d_bytes), (uint32_t)n, raw, check, kc,
                                              reinterpret_cast<Affine<Fp2<P>>*>(d_out), d_err);
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

// the G2 twin of gmsm_g1_decode_device
extern "C" int gmsm_g2_decode_device(gmsm_curve_t curve, const void* d_bytes, size_t n, int raw, int check_on_curve, void* d_points,
                                     void* d_first_error, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (!is_g2_decode_group(curve))
    return set_err(GMSM_EINVAL, "gmsm_g2_decode: G2 groups of bn254, bls12-381, bls12-377, bw6-761 and bw6-633 only (curve id %d)", (int)curve);
  if (n > 0xFFFFFF00ull) return set_err(GMSM_EINVAL, "n too large");
  // the kernel stores each point with 16-byte stores and folds the first error with a 64-bit atomic
  if (((uintptr_t)d_points & 15) || ((uintptr_t)d_first_error & 7))
    return set_err(GMSM_EINVAL, "gmsm_g2_decode: points must be 16-byte and the error word 8-byte aligned device buffers");
  CK(cudaMemsetAsync(d_first_error, 0xFF, 8, st));
  if (n == 0) return GMSM_OK;
  return with_g2_decode_consts(curve, [&](const auto& kc) {
    return run_decode(d_bytes, n, raw, check_on_curve, kc, d_points, (unsigned long long*)d_first_error, st);
  });
}

using DecodeDeviceFn = int (*)(gmsm_curve_t, const void*, size_t, int, int, void*, void*, void*);

// host bytes -> host points through a device decoder: one upload, one launch, one download, and the first error as the reference's
// message prefixed by the point's index
static int host_decode(const char* name, DecodeDeviceFn decode, gmsm_curve_t curve, const uint8_t* bytes, size_t n, int raw,
                       int check_on_curve, uint64_t* out_points) {
  size_t ab = gmsm_affine_bytes(curve);
  if (!ab) return set_err(GMSM_EINVAL, "unknown curve id %d", (int)curve);
  if (int rc = use_device(default_device())) return rc;
  if (n == 0) return GMSM_OK;
  const size_t in_bytes = n * (raw ? ab : ab / 2);
  DevBuf d_in, d_out, d_err;
  if (cudaMalloc(&d_in.p, in_bytes) != cudaSuccess || cudaMalloc(&d_out.p, n * ab) != cudaSuccess || cudaMalloc(&d_err.p, 8) != cudaSuccess)
    return set_err(GMSM_ENOMEM, "%s: device allocation failed", name);
  int rc = GMSM_OK;
  unsigned long long first = ~0ull;
  cudaError_t ce = cudaMemcpy(d_in.p, bytes, in_bytes, cudaMemcpyHostToDevice);
  if (ce == cudaSuccess) rc = decode(curve, d_in.p, n, raw, check_on_curve, d_out.p, d_err.p, nullptr);
  if (ce == cudaSuccess && rc == GMSM_OK) ce = cudaMemcpy(out_points, d_out.p, n * ab, cudaMemcpyDeviceToHost);
  if (ce == cudaSuccess && rc == GMSM_OK) ce = cudaMemcpy(&first, d_err.p, 8, cudaMemcpyDeviceToHost);
  if (ce != cudaSuccess) return set_err(GMSM_ECUDA, "%s: %s", name, cudaGetErrorString(ce));
  if (rc != GMSM_OK) return rc;
  if (first != ~0ull) return set_err(GMSM_EINVAL, "point %llu: %s", first >> 8, dec_message((int)(first & 0xFF)));
  return GMSM_OK;
}

// host bytes -> host points (Go memory layout), n points of a homogeneous stream (raw = 1: RawBytes, 0: Bytes)
extern "C" int gmsm_g1_decode(gmsm_curve_t curve, const uint8_t* bytes, size_t n, int raw, int check_on_curve, uint64_t* out_points) {
  return host_decode("gmsm_g1_decode", gmsm_g1_decode_device, curve, bytes, n, raw, check_on_curve, out_points);
}

extern "C" int gmsm_g2_decode(gmsm_curve_t curve, const uint8_t* bytes, size_t n, int raw, int check_on_curve, uint64_t* out_points) {
  if (!is_g2_decode_group(curve))
    return set_err(GMSM_EINVAL, "gmsm_g2_decode: G2 groups of bn254, bls12-381, bls12-377, bw6-761 and bw6-633 only (curve id %d)", (int)curve);
  return host_decode("gmsm_g2_decode", gmsm_g2_decode_device, curve, bytes, n, raw, check_on_curve, out_points);
}

// bytes of one encoded point of a pairing group (0 for any other id)
static size_t encoded_bytes(gmsm_curve_t curve, int raw) {
  const size_t ab = gmsm_affine_bytes(curve);
  if (with_encode_group(curve, [](auto) { return 0; }) < 0) return 0;
  return raw ? ab : ab / 2;                // RawBytes: X || Y, as many bytes as the in-memory point; Bytes: X
}

extern "C" int gmsm_points_encode_device(gmsm_curve_t curve, const void* d_points, size_t n, int raw, void* d_bytes, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (!encoded_bytes(curve, raw))
    return set_err(GMSM_EINVAL, "gmsm_points_encode: G1 and G2 groups of the pairing curves only (curve id %d)", (int)curve);
  if (n > 0xFFFFFF00ull) return set_err(GMSM_EINVAL, "n too large");
  if (n == 0) return GMSM_OK;
  // the kernel reads each point with 16-byte loads (every affine point is a multiple of 16 bytes) and writes 32-bit words
  if (!d_points || !d_bytes || ((uintptr_t)d_points & 15) || ((uintptr_t)d_bytes & 3))
    return set_err(GMSM_EINVAL, "gmsm_points_encode: points must be 16-byte and bytes 4-byte aligned device buffers");
  return with_encode_group(curve, [&](auto g) {
    using G = decltype(g);
    using P = typename G::Params;
    using C = std::conditional_t<G::degree == 1, Fp<P>, Fp2<P>>;
    const auto* pts = reinterpret_cast<const Affine<C>*>(d_points);
    auto* out = reinterpret_cast<uint32_t*>(d_bytes);
    if (raw) k_points_encode<P, G::degree, 1><<<nblk(n, ENC_THREADS), ENC_THREADS, 0, st>>>(pts, (uint32_t)n, out);
    else k_points_encode<P, G::degree, 0><<<nblk(n, ENC_THREADS), ENC_THREADS, 0, st>>>(pts, (uint32_t)n, out);
    CK(cudaGetLastError());
    return (int)GMSM_OK;
  });
}

extern "C" int gmsm_points_encode(gmsm_curve_t curve, const uint64_t* points, size_t n, int raw, uint8_t* out) {
  const size_t ab = gmsm_affine_bytes(curve), eb = encoded_bytes(curve, raw);
  if (!eb) return set_err(GMSM_EINVAL, "gmsm_points_encode: G1 and G2 groups of the pairing curves only (curve id %d)", (int)curve);
  if (int rc = use_device(default_device())) return rc;
  if (n == 0) return GMSM_OK;
  DevBuf d_in, d_out;
  if (cudaMalloc(&d_in.p, n * ab) != cudaSuccess || cudaMalloc(&d_out.p, n * eb) != cudaSuccess)
    return set_err(GMSM_ENOMEM, "gmsm_points_encode: device allocation failed");
  cudaError_t ce = cudaMemcpy(d_in.p, points, n * ab, cudaMemcpyHostToDevice);
  int rc = GMSM_OK;
  if (ce == cudaSuccess) rc = gmsm_points_encode_device(curve, d_in.p, n, raw, d_out.p, nullptr);
  if (ce == cudaSuccess && rc == GMSM_OK) ce = cudaMemcpy(out, d_out.p, n * eb, cudaMemcpyDeviceToHost);
  if (ce != cudaSuccess) return set_err(GMSM_ECUDA, "gmsm_points_encode: %s", cudaGetErrorString(ce));
  return rc;
}
