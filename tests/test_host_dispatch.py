"""Host-side dispatch of libgmsm: the per-group and per-field tables, the argument checks that run before any device
access, and (on the GPU) the in-process shard runner of the one-shot MultiExp.

The CPU tests compare host-only answers of the library with literals: the sizes each group and scalar field reports, the
workspace sizes, the window widths of the fitted model, and the return code and error text of each early refusal."""
import ctypes
import importlib
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

EINVAL = 1
CURVES = range(-1, 15)     # 13 groups (ids 0..12) and unknown ids on both sides
FIELDS = range(-1, 9)      # 7 scalar fields (ids 0..6) and unknown ids
BN254_G1, BN254_G2, BLS12381_G2, BLS24315_G1, BW6633_G1 = 0, 1, 3, 9, 11
FAKE = 0x10000             # a device address that no check here dereferences


@pytest.fixture(scope="module")
def native():
    return importlib.import_module("gnark-crypto_b200._native")


@pytest.fixture(scope="module")
def L(native):
    return native.lib()


def _refused(native, rc, text):
    assert rc == EINVAL, (rc, native.last_error())
    assert native.last_error() == text


def test_group_sizes(L):
    assert [L.gmsm_affine_bytes(c) for c in CURVES] == [0, 64, 128, 96, 192, 96, 192, 64, 192, 192, 80, 80, 160, 160, 0, 0]
    assert [L.gmsm_scalar_bytes(c) for c in CURVES] == [0, 32, 32, 32, 32, 32, 32, 32, 48, 48, 32, 32, 40, 40, 0, 0]
    assert [L.gmsm_jac_bytes(c) for c in CURVES] == [0, 96, 192, 144, 288, 144, 288, 96, 288, 288, 120, 120, 240, 240, 0, 0]
    assert [L.gmsm_xyzz_bytes(c) for c in CURVES] == [0, 128, 256, 192, 384, 192, 384, 128, 384, 384, 160, 160, 320, 320, 0, 0]


def test_field_sizes(L, native):
    native.lib().gmsm_bases_precompute(None, 0)      # leaves "null bases" as the last error
    assert [L.gmsm_fft_fr_bytes(f) for f in FIELDS] == [0, 32, 32, 32, 32, 32, 40, 48, 0, 0]
    assert native.last_error() == "null bases"        # an unknown field is answered with 0, not an error


def test_to_lagrange_workspace(L):
    # non-zero exactly for the G1 groups of the seven pairing curves: n extended-Jacobian points
    got = [L.gmsm_g1_to_lagrange_workspace_bytes(c, 1024) for c in CURVES]
    assert got == [0, 131072, 0, 196608, 0, 196608, 0, 0, 393216, 0, 163840, 163840, 327680, 0, 0, 0]


def test_poly_workspace(L):
    sizes = (0, 1, 5, 1000, 1 << 16, (1 << 20) + 3)
    want = {-1: [0] * 6, 5: [0, 0, 0, 0, 2560, 41080], 6: [0, 0, 0, 96, 6144, 98592], 7: [0] * 6, 8: [0] * 6}
    for f in range(0, 5):
        want[f] = [0, 0, 0, 0, 2048, 32864]
    for f, w in want.items():
        assert [L.gmsm_fr_poly_workspace_bytes(f, n) for n in sizes] == w, f


def test_window_bits_every_group(L, monkeypatch):
    monkeypatch.delenv("GMSM_C", raising=False)
    want = {
        0: [15] * 15 + [16, 17, 17, 17, 17, 17, 20, 20, 20],
        1: [17] * 20 + [20, 20, 20, 22],
        2: [15] * 15 + [16, 16, 16, 17, 17, 20, 20, 20, 22],
        3: [17] * 21 + [20, 20, 20],
        4: [15] * 15 + [16, 16, 16, 17, 17, 20, 20, 20, 22],
        5: [17] * 21 + [20, 20, 20],
        6: [14] * 16 + [16, 16, 16, 16, 20, 20, 20, 20],
        7: [14] * 16 + [16, 16, 18, 18, 19, 20, 21, 21],
        8: [14] * 16 + [16, 16, 18, 18, 19, 20, 21, 21],
        9: [14] * 10 + [15] * 6 + [17, 17, 17, 17, 20, 20, 20, 22],
        10: [14] * 10 + [15] * 6 + [17, 17, 17, 17, 20, 20, 20, 22],
        11: [15] * 16 + [16, 16, 18, 18, 19, 20, 21, 21],
        12: [15] * 16 + [16, 16, 18, 18, 19, 20, 21, 21],
        -1: [0] * 24,
        13: [0] * 24,
    }
    for c, w in want.items():
        assert [L.gmsm_choose_window_bits(c, 1 << k) for k in range(4, 28)] == w, c


def test_ctx_create_refusals(L, native):
    for create in (L.gmsm_ctx_create, L.gmsm_ctx_create_tables):
        for curve, c, text in ((13, 0, "unknown curve id 13"), (-1, 0, "unknown curve id -1"),
                               (BN254_G1, 1, "window width c=1 out of range [2,24]"),
                               (BN254_G1, 25, "window width c=25 out of range [2,24]")):
            assert not create(curve, 1024, c, 0)
            assert native.last_error() == text


def test_tables_build_refusals(L, native):
    P = ctypes.c_void_p(FAKE)
    for curve, c, n, stride, text in (
        (13, 16, 10, 10, "unknown curve id 13"),
        (BN254_G1, 1, 10, 10, "window width c=1 out of range [2,24]"),
        (BN254_G1, 25, 10, 10, "window width c=25 out of range [2,24]"),
        (BN254_G1, 16, 10, 9, "row_stride 9 < n 10"),
        (BN254_G1, 16, 10, 1 << 27, "row_stride*W = 134217728*16 does not fit the 31-bit table index; shard the bases"),
    ):
        _refused(native, L.gmsm_tables_build_device(curve, c, P, n, P, stride, None), text)


def test_multiexp_nb_tasks(L, native):
    _refused(native, L.gmsm_multiexp(BN254_G1, None, None, 3, 1025, None), "invalid config: config.NbTasks > 1024")


def test_to_lagrange_refusals(L, native):
    for curve, n, text in (
        (13, 4, "unknown curve id 13"),
        (BN254_G2, 4, "ToLagrangeG1 is provided for the G1 groups of the pairing curves only (curve id 1)"),
        (BLS12381_G2, 4, "ToLagrangeG1 is provided for the G1 groups of the pairing curves only (curve id 3)"),
        (BN254_G1, 0, "len(coeffs) must be a power of 2"),
        (BN254_G1, 3, "len(coeffs) must be a power of 2"),
        (BW6633_G1, 1 << 21, "m (2097152) is too big: the required root of unity does not exist"),
        (BLS24315_G1, 1 << 23, "m (8388608) is too big: the required root of unity does not exist"),
    ):
        _refused(native, L.gmsm_g1_to_lagrange(curve, None, n, 0, None), text)
        _refused(native, L.gmsm_g1_to_lagrange_device(curve, None, n, None, None, None), text)


def test_fft_domain_unknown_field(L, native):
    for f in (-1, 7):
        assert not L.gmsm_fft_domain_create(f, 16, None, 0)
        assert native.last_error() == "unknown scalar field %d" % f


def test_bases_precompute_null(L, native):
    _refused(native, L.gmsm_bases_precompute(None, 0), "null bases")


def _u64(*limbs):
    return (ctypes.c_uint64 * len(limbs))(*limbs)


def test_poly_div_refusals(L, native):
    div = L.gmsm_fr_poly_div_x_minus_a_device
    zero, bad = _u64(0, 0, 0, 0), _u64(*[(1 << 64) - 1] * 4)
    W = ctypes.c_void_p(FAKE + (1 << 30))
    F, H = ctypes.c_void_p(FAKE), ctypes.c_void_p(FAKE + 32)
    for args, text in (
        ((7, F, 4, zero, None, F, W, None), "unknown scalar field 7"),
        ((0, F, 0, zero, None, F, W, None), "empty polynomial (n = 0)"),
        ((0, None, 4, zero, None, F, W, None), "null polynomial, point or value pointer"),
        ((0, F, 4, None, None, F, W, None), "null polynomial, point or value pointer"),
        ((0, F, 4, zero, None, None, W, None), "null polynomial, point or value pointer"),
        ((0, F, 4, zero, H, F, W, None), "the quotient must not overlap the polynomial"),
        ((0, F, 1 << 16, zero, None, F, None, None), "null workspace (gmsm_fr_poly_workspace_bytes)"),
        ((0, F, 4, bad, None, F, W, None), "the point is not a reduced fr.Element"),
        ((0, F, (1 << 41) + 1, zero, None, F, W, None), "polynomial too large (n = 2199023255553)"),
    ):
        _refused(native, div(*args), text)


def test_poly_lincomb_refusals(L, native):
    lin = L.gmsm_fr_poly_lincomb_device
    P = (ctypes.c_void_p * 2)(FAKE, FAKE + 4096)
    P_null = (ctypes.c_void_p * 2)(FAKE, None)
    lens, zlens = (ctypes.c_size_t * 2)(4, 4), (ctypes.c_size_t * 2)(0, 0)
    strides, zstride = (ctypes.c_size_t * 2)(1, 1), (ctypes.c_size_t * 2)(0, 1)
    offs = (ctypes.c_size_t * 2)(0, 0)
    s_ok, s_bad = _u64(1, 0, 0, 0, 2, 0, 0, 0), _u64(1, 0, 0, 0, *[(1 << 64) - 1] * 4)
    out, out_overlap = ctypes.c_void_p(FAKE + (1 << 20)), ctypes.c_void_p(FAKE + 64)
    for args, text in (
        ((7, P, lens, s_ok, strides, offs, 2, out, 4, 0, None), "unknown scalar field 7"),
        ((0, P, lens, s_ok, strides, offs, 0, out, 4, 0, None), "nothing to combine (k = 0, out_len = 4)"),
        ((0, P, lens, s_ok, strides, offs, 2, out, 0, 0, None), "nothing to combine (k = 2, out_len = 0)"),
        ((0, None, lens, s_ok, strides, offs, 2, out, 4, 0, None), "null argument"),
        ((0, P, lens, s_ok, strides, None, 2, out, 4, 0, None), "null argument"),
        ((0, P, lens, s_ok, strides, offs, 2, None, 4, 0, None), "null argument"),
        ((0, P, lens, s_ok, zstride, offs, 2, out, 4, 0, None), "stride of polynomial 0 is 0"),
        ((0, P_null, lens, s_ok, strides, offs, 2, out, 4, 0, None), "polynomial 1 is null"),
        ((0, P, lens, s_ok, strides, offs, 2, out_overlap, 4, 0, None), "polynomial 0 overlaps the output"),
        ((0, P, lens, s_bad, strides, offs, 2, out, 4, 0, None), "scalar 1 is not a reduced fr.Element"),
    ):
        _refused(native, lin(*args), text)
    # empty polynomials are neither null-checked nor overlap-checked
    _refused(native, lin(0, P_null, zlens, s_bad, strides, offs, 2, out, 4, 0, None), "scalar 1 is not a reduced fr.Element")


def test_poly_fold_refusals(L, native):
    fold = L.gmsm_fr_poly_fold_device
    P = (ctypes.c_void_p * 2)(FAKE, FAKE + 4096)
    P_null = (ctypes.c_void_p * 2)(None, FAKE)
    lens = (ctypes.c_size_t * 2)(4, 4)
    g_ok, g_bad = _u64(3, 0, 0, 0), _u64(*[(1 << 64) - 1] * 4)
    out = ctypes.c_void_p(FAKE + (1 << 20))
    for args, text in (
        ((7, P, lens, 2, g_ok, out, 4, None), "unknown scalar field 7"),
        ((0, P, lens, 0, g_ok, out, 4, None), "nothing to fold (k = 0, out_len = 4)"),
        ((0, P, None, 2, g_ok, out, 4, None), "null argument"),
        ((0, P, lens, 2, None, out, 4, None), "null argument"),
        ((0, P_null, lens, 2, g_ok, out, 4, None), "polynomial 0 is null"),
        ((0, P, lens, 2, g_bad, out, 4, None), "gamma is not a reduced fr.Element"),
    ):
        _refused(native, fold(*args), text)


@pytest.mark.gpu
def test_one_shot_multiexp_two_shards_on_one_device(native, monkeypatch):
    """GMSM_DEVICES=0,0 runs the multi-device branch of the one-shot MultiExp on one GPU: two shards of the call, one host
    thread each, their window partials joined on the first; the launch count is the one that branch has always reported"""
    import gnark_crypto_b200 as pkg
    from oracle import cref
    from tests.gpu_common import make_inputs

    L = native.lib()
    A1, _, A2, _ = pkg.curve_package("bn254")
    n = (1 << 17) + 5                       # above the 2^16 threshold below which a call stays on one device
    monkeypatch.setenv("GMSM_DEVICES", "0,0")
    # 1 (the join) + the launches of each shard's pipeline at the shared window width
    for g, Aff, launches in (("bn254_g1", A1, 67), ("bn254_g2", A2, 59)):
        pts, s = make_inputs(g, n, 21)
        want, _, _, _ = cref.msm(g, pts, s, c=0, nthreads=8)
        got = Aff().MultiExp(pts, s, pkg.MultiExpConfig())
        assert np.array_equal(got.limbs, want), g
        assert L.gmsm_last_oneshot_launches() == launches, g
