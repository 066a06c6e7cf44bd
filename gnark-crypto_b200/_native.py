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

vp, sz, i32, u64, cstr = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_uint64, ctypes.c_char_p
_MULTIEXP = [vp, vp, sz, i32, vp]
# (name, restype, argtypes) of every symbol include/gmsm.h declares (tests check the library exports all of them)
_SIGNATURES = [
    ("gmsm_last_error", cstr, []), ("gmsm_version", cstr, []),
    ("gmsm_affine_bytes", sz, [i32]), ("gmsm_scalar_bytes", sz, [i32]), ("gmsm_jac_bytes", sz, [i32]), ("gmsm_xyzz_bytes", sz, [i32]),
    ("gmsm_bn254_g1_multiexp", i32, _MULTIEXP), ("gmsm_bn254_g2_multiexp", i32, _MULTIEXP),
    ("gmsm_bls12381_g1_multiexp", i32, _MULTIEXP), ("gmsm_bls12381_g2_multiexp", i32, _MULTIEXP),
    ("gmsm_bls12377_g1_multiexp", i32, _MULTIEXP), ("gmsm_bls12377_g2_multiexp", i32, _MULTIEXP),
    ("gmsm_secp256k1_g1_multiexp", i32, _MULTIEXP), ("gmsm_bw6761_g1_multiexp", i32, _MULTIEXP), ("gmsm_bw6761_g2_multiexp", i32, _MULTIEXP),
    ("gmsm_bls24315_g1_multiexp", i32, _MULTIEXP), ("gmsm_bls24317_g1_multiexp", i32, _MULTIEXP),
    ("gmsm_bw6633_g1_multiexp", i32, _MULTIEXP), ("gmsm_bw6633_g2_multiexp", i32, _MULTIEXP),
    ("gmsm_multiexp", i32, [i32, vp, vp, sz, i32, vp]),
    ("gmsm_choose_window_bits", i32, [i32, sz]),
    ("gmsm_multiexp_window_sums", i32, [i32, vp, vp, sz, i32, i32, vp]),
    ("gmsm_last_oneshot_launches", i32, []),
    ("gmsm_bases_upload", vp, [i32, vp, sz, i32]),
    ("gmsm_bases_multiexp", i32, [vp, sz, vp, sz, i32, vp]),
    ("gmsm_bases_multiexp_device", i32, [vp, sz, vp, sz, i32, vp, vp]),
    ("gmsm_bases_free", None, [vp]),
    ("gmsm_bases_precompute", i32, [vp, i32]),
    ("gmsm_bases_table_bits", i32, [vp]),
    ("gmsm_ctx_create_tables", vp, [i32, sz, i32, i32]),
    ("gmsm_tables_build_device", i32, [i32, i32, vp, sz, vp, sz, vp]),
    ("gmsm_ctx_msm_tables_device", i32, [vp, vp, sz, sz, vp, sz, vp, vp]),
    ("gmsm_ctx_create", vp, [i32, sz, i32, i32]),
    ("gmsm_ctx_destroy", None, [vp]),
    ("gmsm_ctx_window_bits", i32, [vp]),
    ("gmsm_ctx_num_windows", i32, [vp]),
    ("gmsm_ctx_workspace_bytes", sz, [vp]),
    ("gmsm_ctx_last_launches", i32, [vp]),
    ("gmsm_ctx_msm_device", i32, [vp, vp, vp, sz, vp, vp]),
    ("gmsm_ctx_window_sums_device", i32, [vp, vp, vp, sz, vp, vp]),
    ("gmsm_ctx_finalize_device", i32, [vp, vp, i32, vp, vp]),
    ("gmsm_ctx_set_profiling", None, [vp, i32]),
    ("gmsm_ctx_last_stage_ms", i32, [vp, ctypes.POINTER(ctypes.c_float)]),
    ("gmsm_ctx_last_timeline_ms", i32, [vp, ctypes.POINTER(ctypes.c_float), i32, ctypes.POINTER(ctypes.c_int)]),
    ("gmsm_generate_multiples_device", i32, [i32, vp, u64, sz, vp, vp]),
    ("gmsm_batch_scalar_mul", i32, [i32, vp, vp, sz, vp]),
    ("gmsm_g1_decode", i32, [i32, vp, sz, i32, i32, vp]),
    ("gmsm_g1_decode_device", i32, [i32, vp, sz, i32, i32, vp, vp, vp]),
    ("gmsm_g2_decode", i32, [i32, vp, sz, i32, i32, vp]),
    ("gmsm_g2_decode_device", i32, [i32, vp, sz, i32, i32, vp, vp, vp]),
    ("gmsm_pairing_workspace_bytes", sz, [i32, sz]),
    ("gmsm_pairing_miller_loop", i32, [i32, vp, vp, sz, vp]),
    ("gmsm_pairing_miller_loop_device", i32, [i32, vp, vp, sz, vp, vp, vp]),
    ("gmsm_pairing_final_exp", i32, [i32, vp, sz, vp]),
    ("gmsm_pairing_final_exp_device", i32, [i32, vp, sz, vp, vp]),
    ("gmsm_pair", i32, [i32, vp, vp, sz, vp]),
    ("gmsm_pair_device", i32, [i32, vp, vp, sz, vp, vp, vp]),
    ("gmsm_points_encode", i32, [i32, vp, sz, i32, vp]),
    ("gmsm_points_encode_device", i32, [i32, vp, sz, i32, vp, vp]),
    ("gmsm_fft_fr_bytes", sz, [i32]),
    ("gmsm_fft_domain_create", vp, [i32, u64, vp, i32]),
    ("gmsm_fft_domain_free", None, [vp]),
    ("gmsm_fft_domain_cardinality", u64, [vp]),
    ("gmsm_fft_domain_constants", i32, [vp, vp]),
    ("gmsm_fft", i32, [vp, vp, sz, i32, i32]),
    ("gmsm_fft_inverse", i32, [vp, vp, sz, i32, i32]),
    ("gmsm_fft_device", i32, [vp, vp, sz, i32, i32, i32, vp]),
    ("gmsm_fft_bit_reverse_device", i32, [vp, vp, sz, vp]),
    ("gmsm_fr_poly_workspace_bytes", sz, [i32, sz]),
    ("gmsm_fr_poly_div_x_minus_a_device", i32, [i32, vp, sz, vp, vp, vp, vp, vp]),
    ("gmsm_fr_poly_fold_device", i32, [i32, vp, vp, sz, vp, vp, sz, vp]),
    ("gmsm_fr_poly_lincomb_device", i32, [i32, vp, vp, vp, vp, vp, sz, vp, sz, i32, vp]),
    ("gmsm_fr_batch_invert_device", i32, [i32, vp, sz, vp, vp]),
    ("gmsm_fr_permutation_workspace_bytes", sz, [i32, sz]),
    ("gmsm_fr_permutation_accumulate_device", i32, [i32, vp, vp, sz, vp, vp, vp, vp]),
    ("gmsm_fft_permutation_numerator_device", i32, [vp, vp, vp, vp, sz, vp, vp, vp, vp]),
    ("gmsm_fr_sort_workspace_bytes", sz, [i32, sz]),
    ("gmsm_fr_sort_device", i32, [i32, vp, sz, vp, vp, vp]),
    ("gmsm_fr_plookup_accumulate_device", i32, [i32, vp, vp, vp, vp, sz, vp, vp, vp, vp, vp]),
    ("gmsm_fft_plookup_numerator_device", i32, [vp, vp, vp, vp, vp, vp, sz, vp, vp, vp, vp, vp]),
    ("gmsm_fr_iop_workspace_bytes", sz, [i32, sz]),
    ("gmsm_fr_iop_ratio_shuffled_device", i32, [i32, vp, vp, vp, vp, sz, sz, vp, vp, vp, vp]),
    ("gmsm_fft_iop_ratio_copy_device", i32, [vp, vp, vp, sz, sz, vp, vp, vp, vp, vp, vp]),
    ("gmsm_fft_iop_lagrange_eval_device", i32, [vp, vp, sz, i32, vp, vp, vp, vp]),
    ("gmsm_fr_iop_evaluate_device", i32, [i32, vp, sz, sz, vp, sz, vp, vp, vp, sz, sz, i32, vp, vp]),
    ("gmsm_fr_iop_divide_by_xn_minus_one_device", i32, [i32, vp, sz, u64, i32, vp, sz, vp, vp]),
    ("gmsm_fr_bit_reverse_device", i32, [i32, vp, sz, vp]),
    ("gmsm_fr_generator", i32, [i32, u64, vp]),
    ("gmsm_g1_to_lagrange_workspace_bytes", sz, [i32, sz]),
    ("gmsm_g1_to_lagrange", i32, [i32, vp, sz, i32, vp]),
    ("gmsm_g1_to_lagrange_device", i32, [i32, vp, sz, vp, vp, vp]),
    ("gmsm_scale_powers", i32, [i32, vp, sz, vp, vp, i32, vp]),
    ("gmsm_scale_powers_device", i32, [i32, vp, sz, vp, vp, vp, vp]),
    ("gmsm_test_op", i32, [i32, i32, vp, vp, vp, sz]),
    ("gmsm_test_digits", i32, [i32, i32, vp, sz, vp]),
]
SYMBOLS = [name for name, _, _ in _SIGNATURES]

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
    for name, restype, argtypes in _SIGNATURES:
        f = getattr(L, name)
        f.restype = restype
        f.argtypes = argtypes
    _lib = L
    return L


def last_error() -> str:
    return (lib().gmsm_last_error() or b"").decode()
