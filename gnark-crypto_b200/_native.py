"""ctypes loader for libgmsm.so (the C ABI declared in include/gmsm.h).

No fallback of any kind: if the library is missing it must be built (`python gnark-crypto_b200/build.py`),
and every compute entry point of the library itself fails with GMSM_ENODEV when there is no GPU."""
from __future__ import annotations

import ctypes
import os

HERE = os.path.dirname(os.path.abspath(__file__))
# GMSM_LIB=<tag> selects an experimental build variant (see build.py); default is libgmsm.so
_TAG = os.environ.get("GMSM_LIB", "")
LIB_PATH = os.path.join(HERE, "libgmsm%s.so" % ("_" + _TAG if _TAG else ""))

GMSM_OK, GMSM_EINVAL, GMSM_ECUDA, GMSM_ENOMEM, GMSM_ENODEV = 0, 1, 2, 3, 4

# every symbol include/gmsm.h declares (tests check the library exports all of them)
SYMBOLS = [
    "gmsm_last_error", "gmsm_version", "gmsm_affine_bytes", "gmsm_scalar_bytes", "gmsm_jac_bytes", "gmsm_xyzz_bytes",
    "gmsm_bn254_g1_multiexp", "gmsm_bn254_g2_multiexp", "gmsm_bls12381_g1_multiexp", "gmsm_bls12381_g2_multiexp", "gmsm_bls12377_g1_multiexp", "gmsm_bls12377_g2_multiexp",
    "gmsm_secp256k1_g1_multiexp", "gmsm_bw6761_g1_multiexp", "gmsm_bw6761_g2_multiexp",
    "gmsm_bls24315_g1_multiexp", "gmsm_bls24317_g1_multiexp", "gmsm_bw6633_g1_multiexp", "gmsm_bw6633_g2_multiexp",
    "gmsm_multiexp", "gmsm_choose_window_bits", "gmsm_multiexp_window_sums", "gmsm_last_oneshot_launches", "gmsm_bases_upload", "gmsm_bases_multiexp", "gmsm_bases_multiexp_device", "gmsm_bases_free",
    "gmsm_bases_precompute", "gmsm_bases_table_bits", "gmsm_ctx_create_tables", "gmsm_tables_build_device", "gmsm_ctx_msm_tables_device",
    "gmsm_ctx_create", "gmsm_ctx_destroy", "gmsm_ctx_window_bits", "gmsm_ctx_num_windows", "gmsm_ctx_workspace_bytes",
    "gmsm_ctx_last_launches", "gmsm_ctx_msm_device", "gmsm_ctx_window_sums_device", "gmsm_ctx_finalize_device",
    "gmsm_ctx_set_profiling", "gmsm_ctx_last_stage_ms", "gmsm_generate_multiples_device", "gmsm_batch_scalar_mul", "gmsm_g1_decode", "gmsm_g1_decode_device", "gmsm_fft_fr_bytes", "gmsm_fft_domain_create", "gmsm_fft_domain_free", "gmsm_fft_domain_cardinality",
    "gmsm_fft_domain_constants", "gmsm_fft", "gmsm_fft_inverse", "gmsm_fft_device", "gmsm_fft_bit_reverse_device",
    "gmsm_fr_poly_workspace_bytes", "gmsm_fr_poly_div_x_minus_a_device", "gmsm_fr_poly_fold_device", "gmsm_fr_poly_lincomb_device",
    "gmsm_fr_batch_invert_device", "gmsm_fr_permutation_workspace_bytes", "gmsm_fr_permutation_accumulate_device",
    "gmsm_fft_permutation_numerator_device",
    "gmsm_g1_to_lagrange_workspace_bytes", "gmsm_g1_to_lagrange", "gmsm_g1_to_lagrange_device", "gmsm_test_op", "gmsm_test_digits",
]

_lib = None


class NativeLibraryMissing(RuntimeError):
    pass


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NativeLibraryMissing(
            "%s not found: build it with `python gnark-crypto_b200/build.py` (there is no CPU fallback)" % LIB_PATH
        )
    L = ctypes.CDLL(LIB_PATH)
    vp, sz, i32 = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
    L.gmsm_last_error.restype = ctypes.c_char_p
    L.gmsm_version.restype = ctypes.c_char_p
    for f in ("gmsm_affine_bytes", "gmsm_scalar_bytes", "gmsm_jac_bytes", "gmsm_xyzz_bytes"):
        getattr(L, f).restype = sz
        getattr(L, f).argtypes = [i32]
    for f in ("gmsm_bn254_g1_multiexp", "gmsm_bn254_g2_multiexp", "gmsm_bls12381_g1_multiexp", "gmsm_bls12381_g2_multiexp",
              "gmsm_bls12377_g1_multiexp", "gmsm_bls12377_g2_multiexp", "gmsm_secp256k1_g1_multiexp", "gmsm_bw6761_g1_multiexp",
              "gmsm_bw6761_g2_multiexp", "gmsm_bls24315_g1_multiexp", "gmsm_bls24317_g1_multiexp", "gmsm_bw6633_g1_multiexp",
              "gmsm_bw6633_g2_multiexp"):
        getattr(L, f).argtypes = [vp, vp, sz, i32, vp]
    L.gmsm_multiexp.argtypes = [i32, vp, vp, sz, i32, vp]
    L.gmsm_choose_window_bits.argtypes = [i32, sz]
    L.gmsm_multiexp_window_sums.argtypes = [i32, vp, vp, sz, i32, i32, vp]
    L.gmsm_bases_upload.restype = vp
    L.gmsm_bases_upload.argtypes = [i32, vp, sz, i32]
    L.gmsm_bases_multiexp.argtypes = [vp, sz, vp, sz, i32, vp]
    L.gmsm_bases_multiexp_device.argtypes = [vp, sz, vp, sz, i32, vp, vp]
    L.gmsm_bases_free.argtypes = [vp]
    L.gmsm_bases_free.restype = None
    L.gmsm_bases_precompute.argtypes = [vp, i32]
    L.gmsm_bases_table_bits.argtypes = [vp]
    L.gmsm_ctx_create_tables.restype = vp
    L.gmsm_ctx_create_tables.argtypes = [i32, sz, i32, i32]
    L.gmsm_tables_build_device.argtypes = [i32, i32, vp, sz, vp, sz, vp]
    L.gmsm_ctx_msm_tables_device.argtypes = [vp, vp, sz, sz, vp, sz, vp, vp]
    L.gmsm_ctx_create.restype = vp
    L.gmsm_ctx_create.argtypes = [i32, sz, i32, i32]
    L.gmsm_ctx_destroy.argtypes = [vp]
    L.gmsm_ctx_destroy.restype = None
    L.gmsm_ctx_window_bits.argtypes = [vp]
    L.gmsm_ctx_num_windows.argtypes = [vp]
    L.gmsm_ctx_workspace_bytes.argtypes = [vp]
    L.gmsm_ctx_workspace_bytes.restype = sz
    L.gmsm_ctx_last_launches.argtypes = [vp]
    L.gmsm_ctx_msm_device.argtypes = [vp, vp, vp, sz, vp, vp]
    L.gmsm_ctx_window_sums_device.argtypes = [vp, vp, vp, sz, vp, vp]
    L.gmsm_ctx_finalize_device.argtypes = [vp, vp, i32, vp, vp]
    L.gmsm_ctx_set_profiling.argtypes = [vp, i32]
    L.gmsm_ctx_set_profiling.restype = None
    L.gmsm_ctx_last_stage_ms.argtypes = [vp, ctypes.POINTER(ctypes.c_float)]
    L.gmsm_generate_multiples_device.argtypes = [i32, vp, ctypes.c_uint64, sz, vp, vp]
    L.gmsm_batch_scalar_mul.argtypes = [i32, vp, vp, sz, vp]
    L.gmsm_g1_decode.argtypes = [i32, vp, sz, i32, i32, vp]
    L.gmsm_g1_decode_device.argtypes = [i32, vp, sz, i32, i32, vp, vp, vp]
    L.gmsm_fft_fr_bytes.restype = sz
    L.gmsm_fft_fr_bytes.argtypes = [i32]
    L.gmsm_fft_domain_create.restype = vp
    L.gmsm_fft_domain_create.argtypes = [i32, ctypes.c_uint64, vp, i32]
    L.gmsm_fft_domain_free.argtypes = [vp]
    L.gmsm_fft_domain_free.restype = None
    L.gmsm_fft_domain_cardinality.argtypes = [vp]
    L.gmsm_fft_domain_cardinality.restype = ctypes.c_uint64
    L.gmsm_fft_domain_constants.argtypes = [vp, vp]
    L.gmsm_fft.argtypes = [vp, vp, sz, i32, i32]
    L.gmsm_fft_inverse.argtypes = [vp, vp, sz, i32, i32]
    L.gmsm_fft_device.argtypes = [vp, vp, sz, i32, i32, i32, vp]
    L.gmsm_fft_bit_reverse_device.argtypes = [vp, vp, sz, vp]
    L.gmsm_fr_poly_workspace_bytes.restype = sz
    L.gmsm_fr_poly_workspace_bytes.argtypes = [i32, sz]
    L.gmsm_fr_poly_div_x_minus_a_device.argtypes = [i32, vp, sz, vp, vp, vp, vp, vp]
    L.gmsm_fr_poly_fold_device.argtypes = [i32, vp, vp, sz, vp, vp, sz, vp]
    L.gmsm_fr_poly_lincomb_device.argtypes = [i32, vp, vp, vp, vp, vp, sz, vp, sz, i32, vp]
    L.gmsm_fr_batch_invert_device.argtypes = [i32, vp, sz, vp, vp]
    L.gmsm_fr_permutation_workspace_bytes.restype = sz
    L.gmsm_fr_permutation_workspace_bytes.argtypes = [i32, sz]
    L.gmsm_fr_permutation_accumulate_device.argtypes = [i32, vp, vp, sz, vp, vp, vp, vp]
    L.gmsm_fft_permutation_numerator_device.argtypes = [vp, vp, vp, vp, sz, vp, vp, vp, vp]
    L.gmsm_g1_to_lagrange_workspace_bytes.restype = sz
    L.gmsm_g1_to_lagrange_workspace_bytes.argtypes = [i32, sz]
    L.gmsm_g1_to_lagrange.argtypes = [i32, vp, sz, i32, vp]
    L.gmsm_g1_to_lagrange_device.argtypes = [i32, vp, sz, vp, vp, vp]
    L.gmsm_test_op.argtypes = [i32, i32, vp, vp, vp, sz]
    L.gmsm_test_digits.argtypes = [i32, i32, vp, sz, vp]
    _lib = L
    return L


def last_error() -> str:
    return (lib().gmsm_last_error() or b"").decode()
