/* gmsm.h -- C ABI of the H100-native multi-scalar-multiplication engine.
 *
 * Drop-in boundary for ConsenSys/gnark-crypto's MultiExp (all citations relative to the
 * reference tree):
 *
 *   (*G1Jac).MultiExp(points []G1Affine, scalars []fr.Element, config ecc.MultiExpConfig)
 *       ecc/bn254/multiexp.go:32        ecc/bls12-381/multiexp.go:32
 *   (*G2Jac).MultiExp                   ecc/bn254/multiexp.go:357       ecc/bls12-381/multiexp.go:355
 *   (*G1Affine).MultiExp / (*G2Affine).MultiExp  (:20, :345) keep calling the Jac version.
 *   ecc.MultiExpConfig{NbTasks int}     ecc/ecc.go:107-110
 *
 * The reference has no FFI; a cgo shim (INTEGRATION.md) binds these symbols from a build-tagged
 * sibling of the generated multiexp.go.  Buffers are passed exactly as Go holds them:
 *
 *   points  : n x {X, Y}; each coordinate L little-endian uint64 limbs in Montgomery form
 *             (L = 4 bn254 / secp256k1, 5 bls24-315 / bls24-317, 6 bls12-381 / bls12-377, 10 bw6-633, 12 bw6-761; G2 coordinates are {A0, A1} pairs, except on
 *             bw6-761 / bw6-633 whose G2 is over Fp); infinity = all zero (g1.go:41-47,178-180).  64 / 96 / 128 / 192 bytes per point.
 *   scalars : n x fr.Limbs uint64 (4; 5 for bw6-633, 6 for bw6-761 -- gmsm_scalar_bytes), Montgomery form, reduced (fr/element.go:36).
 *   out     : Jacobian {X, Y, Z}, 3 x L (G2: 3 x 2L) uint64, Montgomery form.  The engine writes the
 *             affine-normalised representative (X, Y, One), or (0, 0, 0) for infinity.  It is
 *             G1Jac.Equal to what the Go path returns and FromJacobian of it is limb-identical.
 *   Only 8-byte alignment of host pointers is assumed.  All functions are thread-safe.
 *
 * Return value: 0 on success, otherwise a GMSM_E* code; gmsm_last_error() gives the text for the
 * calling thread (the shim turns it into the Go `error`; the two reference error strings,
 * multiexp.go:61-71, are reproduced verbatim).
 */
#ifndef GMSM_H
#define GMSM_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  GMSM_BN254_G1 = 0,
  GMSM_BN254_G2 = 1,
  GMSM_BLS12381_G1 = 2,
  GMSM_BLS12381_G2 = 3,
  GMSM_BLS12377_G1 = 4,  /* next-row N4: ecc/bls12-377 */
  GMSM_BLS12377_G2 = 5,  /* its Fp2 tower has u^2 = -5 (e2_bls377.go) */
  GMSM_SECP256K1_G1 = 6, /* N4: ecc/secp256k1/multiexp.go:32 -- fp and fr fill all 256 bits */
  GMSM_BW6761_G1 = 7,    /* N4: ecc/bw6-761/multiexp.go:32  -- 12-word Fp, scalars are 6 x uint64 (fr.Bits = 377) */
  GMSM_BW6761_G2 = 8,    /* N4: ecc/bw6-761/multiexp.go:306 -- G2 is also over Fp */
  GMSM_BLS24315_G1 = 9,  /* N4: ecc/bls24-315/multiexp.go:32 -- 5-word Fp (G2 of the bls24 curves is over Fp4: not provided) */
  GMSM_BLS24317_G1 = 10, /* N4: ecc/bls24-317/multiexp.go:32 */
  GMSM_BW6633_G1 = 11,   /* N4: ecc/bw6-633/multiexp.go:32  -- 10-word Fp, scalars are 5 x uint64 (fr.Bits = 315) */
  GMSM_BW6633_G2 = 12    /* N4: ecc/bw6-633/multiexp.go:304 -- G2 over Fp */
} gmsm_curve_t;

enum {
  GMSM_OK = 0,
  GMSM_EINVAL = 1,   /* bad argument (incl. the reference's "invalid config: config.NbTasks > 1024") */
  GMSM_ECUDA = 2,    /* CUDA runtime error */
  GMSM_ENOMEM = 3,   /* device allocation failed */
  GMSM_ENODEV = 4    /* no CUDA device: the engine has NO CPU fallback */
};

const char* gmsm_last_error(void);
const char* gmsm_version(void);

/* sizes in bytes for a curve: affine point, scalar, Jacobian output, one extended-Jacobian partial */
size_t gmsm_affine_bytes(gmsm_curve_t curve);
size_t gmsm_scalar_bytes(gmsm_curve_t curve);
size_t gmsm_jac_bytes(gmsm_curve_t curve);
size_t gmsm_xyzz_bytes(gmsm_curve_t curve);

/* ---- 1. one-shot drop-ins: host buffers in, host Jacobian out (replaces multiexp.go:32 / :357) ----
 * nb_tasks mirrors config.NbTasks: <= 0 means "default", > 1024 is the reference's error; it does
 * not otherwise influence the GPU schedule.  */
int gmsm_bn254_g1_multiexp(const uint64_t* points, const uint64_t* scalars, size_t n, int nb_tasks,
                           uint64_t out_jac[12]);
int gmsm_bn254_g2_multiexp(const uint64_t* points, const uint64_t* scalars, size_t n, int nb_tasks,
                           uint64_t out_jac[24]);
int gmsm_bls12381_g1_multiexp(const uint64_t* points, const uint64_t* scalars, size_t n, int nb_tasks,
                              uint64_t out_jac[18]);
int gmsm_bls12381_g2_multiexp(const uint64_t* points, const uint64_t* scalars, size_t n, int nb_tasks,
                              uint64_t out_jac[36]);
int gmsm_bls12377_g1_multiexp(const uint64_t* points, const uint64_t* scalars, size_t n, int nb_tasks,
                              uint64_t out_jac[18]);   /* ecc/bls12-377/multiexp.go:32 */
int gmsm_bls12377_g2_multiexp(const uint64_t* points, const uint64_t* scalars, size_t n, int nb_tasks,
                              uint64_t out_jac[36]);
int gmsm_secp256k1_g1_multiexp(const uint64_t* points, const uint64_t* scalars, size_t n, int nb_tasks,
                               uint64_t out_jac[12]);  /* ecc/secp256k1/multiexp.go:32 */
int gmsm_bw6761_g1_multiexp(const uint64_t* points, const uint64_t* scalars /* n x 6 */, size_t n, int nb_tasks,
                            uint64_t out_jac[36]);     /* ecc/bw6-761/multiexp.go:32 */
int gmsm_bw6761_g2_multiexp(const uint64_t* points, const uint64_t* scalars /* n x 6 */, size_t n, int nb_tasks,
                            uint64_t out_jac[36]);     /* ecc/bw6-761/multiexp.go:306 (G2 is over Fp as well) */
int gmsm_bls24315_g1_multiexp(const uint64_t* points, const uint64_t* scalars, size_t n, int nb_tasks,
                              uint64_t out_jac[15]);   /* ecc/bls24-315/multiexp.go:32 */
int gmsm_bls24317_g1_multiexp(const uint64_t* points, const uint64_t* scalars, size_t n, int nb_tasks,
                              uint64_t out_jac[15]);   /* ecc/bls24-317/multiexp.go:32 */
int gmsm_bw6633_g1_multiexp(const uint64_t* points, const uint64_t* scalars /* n x 5 */, size_t n, int nb_tasks,
                            uint64_t out_jac[30]);     /* ecc/bw6-633/multiexp.go:32 */
int gmsm_bw6633_g2_multiexp(const uint64_t* points, const uint64_t* scalars /* n x 5 */, size_t n, int nb_tasks,
                            uint64_t out_jac[30]);     /* ecc/bw6-633/multiexp.go:304 */
int gmsm_multiexp(gmsm_curve_t curve, const uint64_t* points, const uint64_t* scalars, size_t n,
                  int nb_tasks, uint64_t* out_jac);
/* sharded calls with one process per GPU: every process runs its shard through the pipelined engine and gets the W
 * window partials back (host memory, W * gmsm_xyzz_bytes); the partials of all shards are then joined with
 * gmsm_ctx_finalize_device.  All shards must pass the same window width (gmsm_choose_window_bits of the TOTAL size). */
int gmsm_choose_window_bits(gmsm_curve_t curve, size_t n_total);
int gmsm_multiexp_window_sums(gmsm_curve_t curve, const uint64_t* points, const uint64_t* scalars, size_t n, int c,
                              int device, void* out_partials);
/* kernels launched by the last one-shot call in this process (bench.py's gpu_launches) */
int gmsm_last_oneshot_launches(void);

/* ---- 2. resident bases (the prover flow: SRS / proving-key points are static, kzg.Commit
 * ecc/bn254/kzg/kzg.go:159-176 passes pk.G1[:len(p)]) ---- */
typedef struct gmsm_bases gmsm_bases_t;
/* device >= 0: all bases on that GPU; device == -1: sharded contiguously over the GPUs listed in GMSM_DEVICES
 * (every call then runs one host thread per shard and joins the window partials on the first one) */
gmsm_bases_t* gmsm_bases_upload(gmsm_curve_t curve, const uint64_t* points, size_t n, int device);
/* MSM over bases[offset, offset+n) with host scalars */
int gmsm_bases_multiexp(gmsm_bases_t* bases, size_t offset, const uint64_t* scalars, size_t n,
                        int nb_tasks, uint64_t* out_jac);
void gmsm_bases_free(gmsm_bases_t* bases);
/* the same with scalars that are already in device memory (e.g. the output of gmsm_fft_device: iFFT -> fromMont -> digits
 * without a PCIe crossing, SURVEY.md section 8(f) N3); d_scalars lives on the device of the (single-shard) bases, the work is
 * ordered after `stream`'s earlier work, the result comes back to the host */
int gmsm_bases_multiexp_device(gmsm_bases_t* bases, size_t offset, const void* d_scalars, size_t n, int nb_tasks,
                               uint64_t* out_jac, void* stream);
/* Window tables for resident bases (no reference counterpart: the reference re-reads its bases on every call; this
 * serves the static-SRS flow of kzg.Commit, kzg/kzg.go:159-176).  Replaces the device copy of the bases by a table of
 * W rows, row j = 2^(c*j) * bases (W x the device memory, built once on the GPU).  Afterwards gmsm_bases_multiexp
 * runs ONE bucket set over the n*W table points with the signed digits of partitionScalars (multiexp.go:709-803):
 * no per-window bucket reduction, no Horner (msmReduceChunk), wider windows (c = 22, W = 12 at n = 2^24 instead of
 * c = 17, W = 15).  Results are bit-identical.  c = 0: width from the cost model. */
int gmsm_bases_precompute(gmsm_bases_t* bases, int c);
int gmsm_bases_table_bits(const gmsm_bases_t* bases);   /* c of the tables, 0 if none */

/* ---- 3. device-level engine (device pointers; what bench.py times with inputs resident in HBM and
 * what the multi-GPU path composes).  `stream` is a cudaStream_t (NULL = default stream). ---- */
typedef struct gmsm_ctx gmsm_ctx_t;
/* c = 0: window width from the cost model; otherwise 2 <= c <= 24 (the reference's c in 2..16 are a
 * subset: tests sweep them like multiexp_test.go:95-126) */
gmsm_ctx_t* gmsm_ctx_create(gmsm_curve_t curve, size_t max_n, int c, int device);
void gmsm_ctx_destroy(gmsm_ctx_t* ctx);
int gmsm_ctx_window_bits(const gmsm_ctx_t* ctx);
int gmsm_ctx_num_windows(const gmsm_ctx_t* ctx);
size_t gmsm_ctx_workspace_bytes(const gmsm_ctx_t* ctx);
/* number of kernels launched by the last msm call on this ctx (bench.py's gpu_launches) */
int gmsm_ctx_last_launches(const gmsm_ctx_t* ctx);
/* full MSM: d_out_jac receives the Jacobian triple (device memory, gmsm_jac_bytes) */
int gmsm_ctx_msm_device(gmsm_ctx_t* ctx, const void* d_points, const void* d_scalars, size_t n,
                        void* d_out_jac, void* stream);
/* per-window partial sums only (W extended-Jacobian points, W * gmsm_xyzz_bytes): the per-rank
 * result that ranks exchange over NCCL (reference analogue: the halves joined by AddAssign,
 * multiexp.go:128-140) */
int gmsm_ctx_window_sums_device(gmsm_ctx_t* ctx, const void* d_points, const void* d_scalars, size_t n,
                                void* d_partials, void* stream);
/* combine nranks x W gathered partials: per-window sum over ranks, Horner over windows
 * (msmReduceChunk, multiexp.go:302-315), normalise; d_out_jac as above */
int gmsm_ctx_finalize_device(gmsm_ctx_t* ctx, const void* d_partials, int nranks, void* d_out_jac,
                             void* stream);
/* window-table mode at device level (what gmsm_bases_precompute composes): the context shares one bucket set
 * between all windows; d_table holds gmsm_ctx_num_windows(ctx) rows of row_stride affine points, row j =
 * 2^(c*j) * row 0, built by gmsm_tables_build_device (current device; d_table may alias d_points for row 0).
 * gmsm_ctx_msm_tables_device computes the MSM of scalars[0, n) with the bases row0[offset, offset + n). */
gmsm_ctx_t* gmsm_ctx_create_tables(gmsm_curve_t curve, size_t max_n, int c, int device);
int gmsm_tables_build_device(gmsm_curve_t curve, int c, const void* d_points, size_t n, void* d_table,
                             size_t row_stride, void* stream);
int gmsm_ctx_msm_tables_device(gmsm_ctx_t* ctx, const void* d_table, size_t row_stride, size_t offset,
                               const void* d_scalars, size_t n, void* d_out_jac, void* stream);
/* timings of the last msm call's stages in milliseconds (CUDA events on the call's stream), filled only
 * when enabled with gmsm_ctx_set_profiling(ctx, 1): [digits+hist, scan, scatter, accumulate,
 * carries, bucket-reduce, finalize, total] */
void gmsm_ctx_set_profiling(gmsm_ctx_t* ctx, int on);
int gmsm_ctx_last_stage_ms(gmsm_ctx_t* ctx, float out_ms[8]);
/* with gmsm_ctx_set_profiling(ctx, 2), the last call's scatter / accumulate timeline (CUDA events on the call's stream and on
 * the context's auxiliary stream), in milliseconds from the start of the call: out_ms[0] = P scatter passes, [1] = passes
 * scattered on the call's stream ahead of the accumulate (the others ran on the auxiliary stream), [2] = accumulate parts (1
 * or 2); then start, end of pass 0 .. P-1; then start, end of accumulate part 1 (or of the only part) and of part 2 (-1 when
 * there is none), part 2's start being the end of its wait for the auxiliary stream.  *count = 3 + 2P + 4 values; GMSM_EINVAL
 * when cap is smaller or no timeline was recorded (the batch-affine mode records none). */
int gmsm_ctx_last_timeline_ms(gmsm_ctx_t* ctx, float* out_ms, int cap, int* count);

/* ---- 4. base generation (fixed-base helper, SURVEY.md N1/K6): out[i] = [start + i] * base, affine,
 * device pointers; used to build on-curve benchmark inputs without the Go toolchain ---- */
int gmsm_generate_multiples_device(gmsm_curve_t curve, const uint64_t* base_affine_host, uint64_t start,
                                   size_t n, void* d_out_points, void* stream);

/* fixed-base batch scalar multiplication (next-row N1): out[i] = [scalars[i]] * base, affine normal form.
 * Replaces BatchScalarMultiplicationG1 / G2 (ecc/bn254/g1.go:1039-1118, g2.go:1001+), the step before MSM
 * in kzg.NewSRS (kzg/kzg.go:129).  Host buffers; scalars in Montgomery form like everywhere else. */
int gmsm_batch_scalar_mul(gmsm_curve_t curve, const uint64_t* base_affine, const uint64_t* scalars, size_t n,
                          uint64_t* out_points);

/* ---- next-row N2: bulk decoding of serialised G1 points (an SRS in the standard WriteTo format -> resident bases).
 * Replaces G1Affine.SetBytes without the subgroup check -- the Decoder's NoSubgroupChecks path -- ecc/bn254/marshal.go:858-950
 * (:52-60, :952-990), ecc/bls12-381/marshal.go:886-1000: big-endian canonical X (|| Y) with the flag bits of marshal.go:25-31 in
 * the top byte (two bits for bn254, three for the others); compressed points take a square root of x^3 + b (Tonelli-Shanks, which
 * is fp.Sqrt's (x^3 + b)^((q+1)/4) when q = 3 mod 4) with the sign chosen by LexicographicallyLargest (fp/element.go:282-296).  `bytes` is a homogeneous stream of n points: raw = 1, RawBytes
 * (2 x fp.Bytes each); raw = 0, Bytes (compressed, fp.Bytes each).  check_on_curve != 0 also verifies y^2 = x^3 + b of
 * uncompressed points (for bn254 G1, cofactor 1, that IS the reference's subgroup check).  Output: the reference's in-memory
 * G1Affine (Montgomery limbs, infinity = zeroes).  Errors are the reference's, prefixed by the index of the first bad point.
 * Curves: the G1 groups of bn254, bls12-381, bls12-377, bls24-315, bls24-317, bw6-633 and bw6-761, both forms. ---- */
int gmsm_g1_decode(gmsm_curve_t curve, const uint8_t* bytes, size_t n, int raw, int check_on_curve, uint64_t* out_points);
/* device buffers; *d_first_error (8 bytes, device) = (index << 8 | code) of the first bad point, all-ones if none */
int gmsm_g1_decode_device(gmsm_curve_t curve, const void* d_bytes, size_t n, int raw, int check_on_curve, void* d_points,
                          void* d_first_error, void* stream);
/* G2Affine.setBytes without the subgroup check (ecc/bn254/marshal.go:1116-1216, ecc/bls12-381/marshal.go:1160+), the same shape
 * as the G1 pair: wire order X.A1 || X.A0 (|| Y.A1 || Y.A0), flags in the top byte of X.A1, compressed points take a square root
 * of X^3 + b' in Fp2 (b' = bTwistCurveCoeff; "no root" decided by the norm, as E2.Legendre does) with the sign of
 * E2.LexicographicallyLargest.  Output: the reference's in-memory G2Affine ({A0, A1} Montgomery limbs per coordinate, infinity =
 * zeroes).  Groups: GMSM_BN254_G2, GMSM_BLS12381_G2, GMSM_BLS12377_G2, and GMSM_BW6761_G2 / GMSM_BW6633_G2 (curves over Fp, b' =
 * 4 and 8: decoded by the G1 kernel); any other id is GMSM_EINVAL.  The device entry wants d_points 16-byte and d_first_error
 * 8-byte aligned (GMSM_EINVAL otherwise). */
int gmsm_g2_decode(gmsm_curve_t curve, const uint8_t* bytes, size_t n, int raw, int check_on_curve, uint64_t* out_points);
int gmsm_g2_decode_device(gmsm_curve_t curve, const void* d_bytes, size_t n, int raw, int check_on_curve, void* d_points,
                          void* d_first_error, void* stream);
/* G1Affine / G2Affine Bytes (raw = 0: X with the smallest / largest / infinity flag, one coordinate's bytes per point) and
 * RawBytes (raw = 1: X || Y; infinity is mUncompressedInfinity and zeroes, all zeroes on bn254), marshal.go:801-846 and
 * :1051-1100, for the G1 and G2 groups of the seven pairing curves (secp256k1 and unknown ids: GMSM_EINVAL).  Points are the
 * reference's in-memory affine points with reduced Montgomery limbs; n < 2^32.  The device entry is ordered on `stream` and
 * allocates nothing; d_points must be 16-byte and d_bytes 4-byte aligned (GMSM_EINVAL otherwise). */
int gmsm_points_encode(gmsm_curve_t curve, const uint64_t* points, size_t n, int raw, uint8_t* out);
int gmsm_points_encode_device(gmsm_curve_t curve, const void* d_points, size_t n, int raw, void* d_bytes, void* stream);

/* ---- next-row N3: Fr FFT behind gnark-crypto's fft.Domain (ecc/bn254/fr/fft/domain.go:24-110, fft.go:31-190,
 * bitreverse.go:17-42; the fr/fft packages of bls12-381, bls12-377, bls24-315, bls24-317, bw6-633 and bw6-761 are the same
 * generated code with their own constants).  `a` is the []fr.Element image (n x words u64, Montgomery; words = fr.Limbs =
 * gmsm_fft_fr_bytes / 8: 4, or 5 for bw6-633, 6 for bw6-761), transformed in place; len(a) must equal the domain cardinality.  decimation: GMSM_DIT = 0 (input bit-reversed,
 * output natural), GMSM_DIF = 1 (input natural, output bit-reversed) -- fft.Decimation, fft.go:18-23.  coset != 0
 * = fft.OnCoset().  FFTInverse includes the scaling by CardinalityInv. ---- */
typedef struct gmsm_fft_domain gmsm_fft_domain_t;
enum {
  GMSM_FR_BN254 = 0, GMSM_FR_BLS12381 = 1, GMSM_FR_BLS12377 = 2,
  GMSM_FR_BLS24315 = 3,  /* maxOrderRoot 22 */
  GMSM_FR_BLS24317 = 4,  /* maxOrderRoot 60 */
  GMSM_FR_BW6633 = 5,    /* maxOrderRoot 20: domains stop at 2^20; 5-word elements */
  GMSM_FR_BW6761 = 6     /* maxOrderRoot 46; 6-word elements */
};
enum { GMSM_DIT = 0, GMSM_DIF = 1 };
/* fr.Bytes of a scalar field id (32, 40 for bw6-633, 48 for bw6-761); 0 for an unknown id */
size_t gmsm_fft_fr_bytes(int fr_field);
/* NewDomain(m) / NewDomain(m, WithShift(shift)): cardinality = next power of two >= m (past 2^maxOrderRoot: the reference's
 * "too big" error); shift = NULL selects GeneratorFullMultiplicativeGroup() (bn254 5, bls12-381 7, bls12-377 22, bls24-315 7,
 * bls24-317 7, bw6-633 13, bw6-761 15), otherwise `words` u64 Montgomery limbs */
gmsm_fft_domain_t* gmsm_fft_domain_create(int fr_field, uint64_t m, const uint64_t* shift, int device);
void gmsm_fft_domain_free(gmsm_fft_domain_t* domain);
uint64_t gmsm_fft_domain_cardinality(const gmsm_fft_domain_t* domain);
/* Generator, GeneratorInv, CardinalityInv, FrMultiplicativeGen, FrMultiplicativeGenInv (5 x words u64, Montgomery) */
int gmsm_fft_domain_constants(const gmsm_fft_domain_t* domain, uint64_t* out);
int gmsm_fft(gmsm_fft_domain_t* domain, uint64_t* a, size_t n, int decimation, int coset);           /* host buffer */
int gmsm_fft_inverse(gmsm_fft_domain_t* domain, uint64_t* a, size_t n, int decimation, int coset);   /* host buffer */
int gmsm_fft_device(gmsm_fft_domain_t* domain, void* d_a, size_t n, int inverse, int decimation, int coset, void* stream);
int gmsm_fft_bit_reverse_device(gmsm_fft_domain_t* domain, void* d_a, size_t n, void* stream);        /* fft.BitReverse */

/* ---- the Fr polynomial steps of kzg.Open / kzg.BatchOpenSinglePoint on device vectors: eval (ecc/bn254/kzg/kzg.go:55-63),
 * dividePolyByXminusA (:567-582) and the gamma-fold (:302-319); the same for the other six scalar fields.  Vectors are device
 * []fr.Element images (n x fr.Limbs u64, Montgomery, reduced) on the current device; the work is ordered on `stream` (a
 * cudaStream_t, NULL = default stream) and nothing is allocated inside a call.  Host scalars (a, gamma) are fr.Limbs u64
 * Montgomery limbs and must be reduced.  Results are the reference's limbs. ---- */
/* bytes of device workspace gmsm_fr_poly_div_x_minus_a_device needs for n coefficients (0: none; 0 for an unknown field) */
size_t gmsm_fr_poly_workspace_bytes(int fr_field, size_t n);
/* *d_fa = f(a) (one element) and, when d_h != NULL, d_h[0, n-1) = (f - f(a)) / (X - a); d_h must not overlap d_f, which is
 * left unchanged (the reference divides a copy).  d_h = NULL: evaluation only.  n = 0 is GMSM_EINVAL. */
int gmsm_fr_poly_div_x_minus_a_device(int fr_field, const void* d_f, size_t n, const uint64_t* a, void* d_h, void* d_fa,
                                      void* d_work, void* stream);
/* d_out[j] = sum_i gamma^i f_i[j] for j < out_len, f_i zero past lens[i] (gamma^0 = 1); d_polys: host array of k device
 * pointers, each input read once */
int gmsm_fr_poly_fold_device(int fr_field, const void* const* d_polys, const size_t* lens, size_t k, const uint64_t* gamma,
                             void* d_out, size_t out_len, void* stream);
/* linear combination of the SHPLONK / FFLONK batch openings (ecc/bn254/shplonk, ecc/bn254/fflonk):
 * d_out[m * strides[i] + offsets[i]] (+)= scalars[i] * f_i[m] for m < lens[i], summed over i, for the indices below out_len; every
 * other index of d_out[0, out_len) is set to 0 (accumulate = 0) or left as it is (accumulate != 0).  scalars: k x fr.Limbs u64,
 * reduced.  The gamma-fold is scalars gamma^i, strides 1, offsets 0; stride t with offsets 0..t-1 interleaves t polynomials
 * (fflonk.Fold).  GMSM_EINVAL: unknown field, k = 0, out_len = 0, a zero stride, an unreduced scalar, an input overlapping
 * d_out. */
int gmsm_fr_poly_lincomb_device(int fr_field, const void* const* d_polys, const size_t* lens, const uint64_t* scalars,
                                const size_t* strides, const size_t* offsets, size_t k, void* d_out, size_t out_len, int accumulate,
                                void* stream);

/* ---- the Fr steps of permutation.Prove (ecc/bn254/fr/permutation/permutation.go; the same for the other six scalar fields)
 * and fr.BatchInvert on device vectors, with the conventions of the gmsm_fr_poly_* block above (vectors on the current device,
 * ordered on `stream`, nothing allocated inside a call, reduced Montgomery host scalars).  GMSM_EINVAL: unknown field, n = 0, an
 * unreduced scalar, a null vector, buffers that overlap where this is not allowed. ---- */
/* d_out[i] = d_a[i]^-1 for i < n, zero -> zero (fr.BatchInvert, fr/element.go:658-687); d_out may equal d_a (in place) but
 * must not overlap it otherwise */
int gmsm_fr_batch_invert_device(int fr_field, const void* d_a, size_t n, void* d_out, void* stream);
/* bytes of device workspace gmsm_fr_permutation_accumulate_device needs for n elements (0: none; 0 for an unknown field) */
size_t gmsm_fr_permutation_workspace_bytes(int fr_field, size_t n);
/* evaluateAccumulationPolynomialBitReversed (permutation.go:52-75): d_z[rev(k)] = prod_{j<k} (eps - t1[j]) (eps - t2[j])^-1
 * with zero -> zero inversion (the reference's entries past the first eps = t2[k-1] are zero), d_z[0] = 1; n a power of two.
 * d_z must not overlap d_t1 or d_t2, which are left unchanged. */
int gmsm_fr_permutation_accumulate_device(int fr_field, const void* d_t1, const void* d_t2, size_t n, const uint64_t* epsilon,
                                          void* d_z, void* d_work, void* stream);
/* the quotient numerator of permutation.Prove (evaluateFirstPartNumReverse, evaluateSecondPartNumReverse and the omega-fold,
 * permutation.go:78-121, 206-214) from the bit-reversed coset DIF outputs lt1, lt2, lz: with i = rev(p), w the domain's generator
 * and g its FrMultiplicativeGen, d_out[p] = (omega (lz[p] - 1) (g^n - 1) / (g w^i - 1) + (eps - lt2[p]) lz[rev(i + 1 mod n)] -
 * (eps - lt1[p]) lz[p]) / (g^n - 1).  n must equal the domain cardinality; d_out must not overlap the inputs, which are left
 * unchanged. */
int gmsm_fft_permutation_numerator_device(gmsm_fft_domain_t* domain, const void* d_lt1, const void* d_lt2, const void* d_lz, size_t n,
                                          const uint64_t* epsilon, const uint64_t* omega, void* d_out, void* stream);

/* ---- sort.Sort(fr.Vector) and the Fr steps of plookup.ProveLookupVector (ecc/bn254/fr/plookup/vector.go; the same for the
 * other six scalar fields), with the conventions of the block above ---- */
/* bytes of device workspace gmsm_fr_sort_device needs for n elements (0 for n = 0 or an unknown field) */
size_t gmsm_fr_sort_workspace_bytes(int fr_field, size_t n);
/* d_out = d_in sorted ascending by canonical value (fr.Element.Cmp, fr/element.go:254), in Montgomery form; equal keys are
 * bit-identical, so the result is unique.  An exact LSD radix sort over the canonical bytes that skips every byte position at
 * which all keys agree: the call reads which positions vary back to the host, so it returns once the kernels before that copy on
 * `stream` have run.  d_out may equal d_in (in place) but must not overlap it otherwise; n < 2^31; the workspace must not overlap
 * d_in or d_out. */
int gmsm_fr_sort_device(int fr_field, const void* d_in, size_t n, void* d_out, void* d_work, void* stream);
/* evaluateAccumulationPolynomial (vector.go:52-95), in natural order: d_z[0] = 1, d_z[i+1] = d_z[i] (1+beta)(gamma+f[i])
 * (gamma(1+beta)+t[i]+beta t[i+1]) / ((gamma(1+beta)+h1[i]+beta h1[i+1])(gamma(1+beta)+h2[i]+beta h2[i+1])), zero -> zero
 * inversion as fr.BatchInvert.  The workspace is gmsm_fr_permutation_workspace_bytes(fr_field, n) bytes (the same scan).  d_z must
 * not overlap the four inputs, which are left unchanged. */
int gmsm_fr_plookup_accumulate_device(int fr_field, const void* d_f, const void* d_t, const void* d_h1, const void* d_h2, size_t n,
                                      const uint64_t* beta, const uint64_t* gamma, void* d_z, void* d_work, void* stream);
/* the quotient of plookup.ProveLookupVector before its inverse FFT (evaluateNumBitReversed, evaluateZStartsByOneBitReversed,
 * evaluateZEndsByOneBitReversed, evaluateOverlapH1h2BitReversed and computeQuotientCanonical, vector.go:97-335) from the
 * bit-reversed coset DIF outputs lz, lh1, lh2, lt, lf on `domain` (the big domain, of size 2s): the four constraint terms folded
 * with alpha and divided by x^s - 1.  n must equal the domain cardinality; d_out must not overlap the inputs, which are left
 * unchanged. */
int gmsm_fft_plookup_numerator_device(gmsm_fft_domain_t* domain, const void* d_lz, const void* d_lh1, const void* d_lh2, const void* d_lt,
                                      const void* d_lf, size_t n, const uint64_t* beta, const uint64_t* gamma, const uint64_t* alpha,
                                      void* d_out, void* stream);

/* ---- the O(n) steps of the iop package (ecc/bn254/fr/iop: ratios.go, polynomial.go, expressions.go, quotient.go; the same for
 * the other six scalar fields), with the conventions of the blocks above.  Limits, refused with GMSM_EINVAL: at most 32
 * polynomials per list of a ratio builder; an Evaluate program of at most 256 instructions over at most 16 registers (live
 * values), 32 constants and 32 inputs; a DivideByXMinusOne ratio rho = len / size that is a power of two up to 64. ---- */
/* bytes of device workspace every gmsm_*_iop_* call with a workspace needs for n elements (0 for n = 0 or an unknown field) */
size_t gmsm_fr_iop_workspace_bytes(int fr_field, size_t n);
/* BuildRatioShuffledVectors after ToLagrange (ratios.go:78-119): d_z[k] = prod_{i<k} prod_c (beta - num_c[i]) / prod_c (beta -
 * den_c[i]) in natural order (Lagrange, Regular), d_z[0] = 1, zero -> zero inversion (every d_z[k] past the first zero denominator
 * is zero, as in the reference).  k columns per list; column c is read at i, or at its bit reversal when *_bitrev[c] != 0.  n a
 * power of two; d_z must not overlap a column, which are left unchanged. */
int gmsm_fr_iop_ratio_shuffled_device(int fr_field, const void* const* d_num, const int* num_bitrev, const void* const* d_den,
                                      const int* den_bitrev, size_t k, size_t n, const uint64_t* beta, void* d_z, void* d_work,
                                      void* stream);
/* BuildRatioCopyConstraint after ToLagrange (ratios.go:165-238): d_z[k] = prod_{i<k} prod_c (P_c[i] + beta g^c w^i + gamma) /
 * prod_c (P_c[i] + beta ID[sigma[c n + i]] + gamma), ID[s] = g^(s / n) w^(s mod n), w and g = FrMultiplicativeGen of `domain`, in
 * natural order, d_z[0] = 1, zero -> zero inversion.  d_sigma: k n int64 entries on the device.  An entry outside [0, k n) is
 * refused before d_z is written: the call reads one flag back, so it returns once the work before it on `stream` has run.  n must
 * equal the domain cardinality; d_z must not overlap a column or sigma. */
int gmsm_fft_iop_ratio_copy_device(gmsm_fft_domain_t* domain, const void* const* d_cols, const int* bitrev, size_t k, size_t n,
                                   const int64_t* d_sigma, const uint64_t* beta, const uint64_t* gamma, void* d_z, void* d_work,
                                   void* stream);
/* evalLagrange (polynomial.go:204-241): *d_out = (x^n - 1) / n sum_i w^i / (x - w^i) c[idx(i)], idx(i) = i or its bit reversal
 * (bitrev != 0), w the generator of `domain`; zero for x on the domain, as in the reference.  n must equal the domain cardinality. */
int gmsm_fft_iop_lagrange_eval_device(gmsm_fft_domain_t* domain, const void* d_c, size_t n, int bitrev, const uint64_t* x, void* d_out,
                                      void* d_work, void* stream);
/* Evaluate (expressions.go:26-73) of a straight-line program: d_r[idx(i)] = f(i, x_0.GetCoeff(i), ...) for i < n, idx(i) = i or
 * Reverse64(i) >> (64 - TrailingZeros(n)) (out_bitrev != 0).  Input j is read at (i + offsets[j]) mod n, bit-reversed the same way
 * when bitrev[j] != 0 (offsets[j] = (len / size) shift mod n).  Instruction word: op | dst << 8 | a << 16 | b << 24, op 0 input a,
 * 1 constant a, 2 the index i, 3 add, 4 sub, 5 mul (registers a, b), 6 negate (register a); register out_reg holds f.  Constants:
 * nconsts reduced Montgomery elements.  d_r must not overlap an input. */
int gmsm_fr_iop_evaluate_device(int fr_field, const uint32_t* code, size_t len, size_t out_reg, const uint64_t* consts, size_t nconsts,
                                const void* const* d_inputs, const uint64_t* offsets, const int* bitrev, size_t m, size_t n, int out_bitrev,
                                void* d_r, void* stream);
/* the elementwise step of DivideByXMinusOne (quotient.go:40-47): d_out[rev(i)] = a[(i + offset) mod n, bit-reversed when bitrev !=
 * 0] inv[i mod rho] for i < n, n a power of two; inv: rho reduced Montgomery elements.  d_out must not overlap d_a. */
int gmsm_fr_iop_divide_by_xn_minus_one_device(int fr_field, const void* d_a, size_t n, uint64_t offset, int bitrev, const uint64_t* inv,
                                              size_t rho, void* d_out, void* stream);
/* fft.BitReverse (bitreverse.go:17-42) of d_a in place, n a power of two, without a domain */
int gmsm_fr_bit_reverse_device(int fr_field, void* d_a, size_t n, void* stream);
/* fr.Generator(m) (generator.go:18-36): the root of unity of order ecc.NextPowerOfTwo(m), host only, into out (fr.Limbs Montgomery
 * limbs); GMSM_EINVAL past the field's 2-adicity */
int gmsm_fr_generator(int fr_field, uint64_t m, uint64_t* out);

/* ---- kzg.ToLagrangeG1 (ecc/bn254/kzg/utils.go:25-64; the same for the other pairing curves): the canonical SRS [tau^i]G in,
 * its Lagrange form [L_i(tau)]G out, by an inverse FFT over G1 points on the device.  Curves: the G1 groups of bn254, bls12-381,
 * bls12-377, bls24-315, bls24-317, bw6-633 and bw6-761 (others: GMSM_EINVAL).  Points are the reference's in-memory G1Affine
 * (Montgomery limbs, infinity = zeroes), output in the affine normal form of BatchJacobianToAffineG1.  Errors, checked before
 * any device work: "len(coeffs) must be a power of 2" (n = 0 included) and fr.Generator's "m (<n>) is too big: the required
 * root of unity does not exist" (bls24-315 past 2^22, bw6-633 past 2^20); n is at most 2^31. ---- */
/* bytes of device workspace for n points (n extended-Jacobian points); 0 for unsupported curves */
size_t gmsm_g1_to_lagrange_workspace_bytes(gmsm_curve_t curve, size_t n);
/* host buffers; the input is left unmodified, out may equal points */
int gmsm_g1_to_lagrange(gmsm_curve_t curve, const uint64_t* points, size_t n, int device, uint64_t* out);
/* device buffers on the same device, ordered on `stream` (a cudaStream_t, NULL = default stream); nothing is allocated inside
 * the call.  d_points is left unmodified unless d_out == d_points (allowed: in place); d_work holds
 * gmsm_g1_to_lagrange_workspace_bytes(curve, n) bytes (unused for n = 1). */
int gmsm_g1_to_lagrange_device(gmsm_curve_t curve, const void* d_points, size_t n, void* d_out, void* d_work, void* stream);

/* ---- mpcsetup (ecc/bn254/mpcsetup/mpcsetup.go; the same for the other pairing curves): the point updates of a trusted-setup
 * contribution, out[i] = [c r^i] points[i] for i < n, by one variable-base scalar multiplication per point on the device.
 * UpdateMonomialsG1 / G2 (:365-381) is c = r on points[1:], the alpha tau^i and beta tau^i slices of a powers-of-tau contribution
 * are c = alpha (beta), the slice loop of UpdateValues (:64-81) is r = 1.  All thirteen groups.  Points are the reference's
 * in-memory affine points (Montgomery limbs, infinity = zeroes), output in the affine normal form of BatchJacobianToAffineG1;
 * c and r are fr.Elements (fr.Limbs u64 Montgomery limbs), reduced.  An infinity input stays infinity, as does every point whose
 * scalar is zero (c = 0; r = 0 past i = 0).  n = 0 is a no-op.  GMSM_EINVAL, before any device work: an unknown group, a null
 * pointer, an unreduced c or r, an output that overlaps the points without being equal to them. ---- */
/* host buffers, device `device`; out may equal points (in place).  Works in chunks of 2^20 points (chunk k scaled by
 * c r^(k 2^20)), so any n fits and the result does not depend on the chunking. */
int gmsm_scale_powers(gmsm_curve_t curve, const uint64_t* points, size_t n, const uint64_t* c, const uint64_t* r, int device,
                      uint64_t* out);
/* device buffers on one device, ordered on `stream` (a cudaStream_t, NULL = default stream); nothing is allocated inside the
 * call.  d_points is left unmodified unless d_out == d_points (allowed: in place); n < 2^32 (GMSM_EINVAL otherwise). */
int gmsm_scale_powers_device(gmsm_curve_t curve, const void* d_points, size_t n, const uint64_t* c, const uint64_t* r, void* d_out,
                             void* stream);

/* ---- pairings (bn254 and bls12-381) ----
 * Pair, PairingCheck's pairing, MillerLoop and FinalExponentiation of ecc/bn254/pairing.go and ecc/bls12-381/pairing.go.  `curve` is
 * the curve's G1 id (GMSM_BN254_G1 or GMSM_BLS12381_G1); any other id, n = 0 (the reference's "invalid inputs sizes") or a null
 * pointer is GMSM_EINVAL before any device work.  P: n G1Affine, Q: n G2Affine (reference layout, infinity = zeroes; a pair with a
 * point at infinity is skipped).  A GT element is E12{C0, C1} of E6{B0, B1, B2} of E2{A0, A1}: 12 Montgomery fp.Elements (48 u64
 * for bn254, 72 for bls12-381).  MillerLoop's result is limb-identical to the reference's multi-pair loop; final_exp raises the
 * product z[0] ... z[k-1] (k >= 1, the variadic form) to the reference's exponent.  The device entries take device buffers,
 * 16-byte aligned (GMSM_EINVAL otherwise), are ordered on `stream` and allocate nothing: the Miller loop and Pair use d_work of
 * gmsm_pairing_workspace_bytes(curve, n) bytes (the pairs run in chunks, so it stays bounded for any n < 2^32). */
size_t gmsm_pairing_workspace_bytes(gmsm_curve_t curve, size_t n);
int gmsm_pairing_miller_loop(gmsm_curve_t curve, const uint64_t* P, const uint64_t* Q, size_t n, uint64_t* out);
int gmsm_pairing_miller_loop_device(gmsm_curve_t curve, const void* d_P, const void* d_Q, size_t n, void* d_out, void* d_work,
                                    void* stream);
int gmsm_pairing_final_exp(gmsm_curve_t curve, const uint64_t* z, size_t k, uint64_t* out);
int gmsm_pairing_final_exp_device(gmsm_curve_t curve, const void* d_z, size_t k, void* d_out, void* stream);
int gmsm_pair(gmsm_curve_t curve, const uint64_t* P, const uint64_t* Q, size_t n, uint64_t* out);
int gmsm_pair_device(gmsm_curve_t curve, const void* d_P, const void* d_Q, size_t n, void* d_out, void* d_work, void* stream);

/* ---- 5. test hooks: element-wise device functions, used by tests/ to check the sm_90a field and
 * point arithmetic against the oracle.  a, b, out are HOST arrays of n elements each. ---- */
enum {
  GMSM_OP_FMUL = 0, GMSM_OP_FADD = 1, GMSM_OP_FSUB = 2, GMSM_OP_FSQR = 3, GMSM_OP_FNEG = 4,
  GMSM_OP_FDBL = 5, GMSM_OP_FINV = 6,      /* coordinate field (Fp for G1, Fp2 for G2) */
  GMSM_OP_ADD_MIXED = 7,                   /* a: xyzz, b: affine -> xyzz */
  GMSM_OP_SUB_MIXED = 8,
  GMSM_OP_ADD = 9,                         /* a: xyzz, b: xyzz -> xyzz */
  GMSM_OP_DOUBLE = 10,                     /* a: xyzz -> xyzz */
  GMSM_OP_TO_AFFINE = 11,                  /* a: xyzz -> affine */
  GMSM_OP_FR_FROM_MONT = 12,               /* a: scalar -> canonical scalar */
  GMSM_OP_FDOT2 = 13                       /* a: x||u, b: y||v (coordinate field) -> x*y + u*v */
};
int gmsm_test_op(gmsm_curve_t curve, int op, const uint32_t* a, const uint32_t* b, uint32_t* out,
                 size_t n);
/* digits of partitionScalars (multiexp.go:709-803) as the device computes them: out[w*n + i] */
int gmsm_test_digits(gmsm_curve_t curve, int c, const uint64_t* scalars, size_t n, uint32_t* out);

#ifdef __cplusplus
}
#endif
#endif /* GMSM_H */
