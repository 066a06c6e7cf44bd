"""The Fr polynomial kernels of a KZG opening (poly_kernels.cuh: chunk heads, carry levels, write pass, fold), run on the CPU through
the kernel emulation of tests/emu (tests/emu/emu_poly.cpp, cooperative launcher for the kernels with barriers) in the launch order
of fft.cu's entry points, for all seven scalar fields, and compared limb for limb with the host reference of kzg.py (`_eval`,
`_divide_by_x_minus_a`).  CPU only; a test artefact (build/libgmsm_emu_poly.so), never part of libgmsm.so."""
import ctypes
import importlib
import os
import random
import subprocess

import numpy as np
import pytest

curves = importlib.import_module("gnark-crypto_b200.curves")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "gnark-crypto_b200", "csrc")
EMU = os.path.join(ROOT, "tests", "emu")
OUT = os.path.join(ROOT, "gnark-crypto_b200", "build", "libgmsm_emu_poly.so")
FIELDS = {"bn254": 0, "bls12381": 1, "bls12377": 2, "bls24315": 3, "bls24317": 4, "bw6633": 5, "bw6761": 6}
# (log2 chunk length, log2 block size) of fft.cu for 32-, 40- and 48-byte elements
DEFAULT_SHAPE = {32: (2, 8), 40: (3, 7), 48: (2, 7)}
_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        bdir = os.path.dirname(OUT)
        os.makedirs(bdir, exist_ok=True)
        deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))] + [
            os.path.join(EMU, f) for f in os.listdir(EMU)]
        if not os.path.exists(OUT) or os.path.getmtime(OUT) < max(os.path.getmtime(d) for d in deps):
            # tests/emu FIRST: its cuda_runtime.h stands in for the real one
            subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-I", EMU, "-I", CSRC, os.path.join(EMU, "emu_poly.cpp"),
                            "-o", OUT], check=True)
        _LIB = ctypes.CDLL(OUT)
    return _LIB


def _kzg():
    return importlib.import_module("gnark-crypto_b200.kzg")


def _ptr(a):
    return ctypes.c_void_p(a.ctypes.data)


def _emu_div(c, coeffs, a, shape=None, quotient=True):
    """(f(a), h) from the emulated kernels; h is None when quotient is False (evaluation only)"""
    kzg = _kzg()
    r = kzg.CURVE_PARAMS[c].r
    n = len(coeffs)
    f = curves._fr_encode(coeffs, r)
    av = curves._fr_encode([a], r)
    fa = np.zeros_like(av)
    h = np.zeros((max(n - 1, 1), f.shape[1]), dtype=np.uint64)
    log_l, log_b = shape or (-1, -1)
    rc = _lib().emu_poly_div(FIELDS[c], _ptr(f), ctypes.c_uint64(n), _ptr(av), _ptr(h) if quotient else None, _ptr(fa), log_l, log_b)
    assert rc == 0, "rc = %d (2: the polynomial was modified)" % rc
    return curves._fr_decode(fa, r)[0], (curves._fr_decode(h[:n - 1], r) if quotient else None), fa


def _check(c, coeffs, a, shape=None):
    kzg = _kzg()
    r = kzg.CURVE_PARAMS[c].r
    fa, h, fa_limbs = _emu_div(c, coeffs, a, shape)
    want = kzg._eval(coeffs, a, r)
    assert fa == want
    assert np.array_equal(fa_limbs, curves._fr_encode([want], r))      # canonical limbs, not just the same residue
    assert h == kzg._divide_by_x_minus_a(coeffs, want, a, r)
    fa2, _, _ = _emu_div(c, coeffs, a, shape, quotient=False)
    assert fa2 == want


def _points(r, rng):
    return [0, 1, r - 1, rng.randrange(r)]


@pytest.mark.parametrize("c", list(FIELDS))
def test_divide_default_shape(c):
    """the tile shape of fft.cu: lengths 1, 2, 3, T - 1, T, T + 1 (T = tile length), a in {0, 1, r - 1, random}"""
    kzg = _kzg()
    cp = kzg.CURVE_PARAMS[c]
    log_l, log_b = DEFAULT_SHAPE[cp.fr_bytes]
    t = 1 << (log_l + log_b)
    rng = random.Random(11 + FIELDS[c])
    for n in (1, 2, 3, t - 1, t, t + 1):
        coeffs = [rng.randrange(cp.r) for _ in range(n)]
        for a in _points(cp.r, rng):
            _check(c, coeffs, a)


@pytest.mark.parametrize("c", list(FIELDS))
def test_divide_small_tiles_deep_levels(c):
    """small tiles (chunk length L = 2, 4 threads: T = 8; and L = 1, 2 threads: T = 2) so that short polynomials reach three and
    more carry levels: lengths 1, 2, 3, L - 1, L, L + 1, T - 1, T, T + 1, T^2 + 7 and T^3 + 5 (517: levels of 65, 9 and 2 heads)"""
    kzg = _kzg()
    r = kzg.CURVE_PARAMS[c].r
    rng = random.Random(29 + FIELDS[c])
    for shape, lengths in (((1, 2), (1, 2, 3, 7, 8, 9, 71, 517)), ((0, 1), (1, 2, 3, 11, 37))):
        for n in lengths:
            coeffs = [rng.randrange(r) for _ in range(n)]
            for a in _points(r, rng):
                _check(c, coeffs, a, shape)
    for a in _points(r, rng):                                     # every coefficient r - 1: the largest operands everywhere
        _check(c, [r - 1] * 517, a, (1, 2))
        _check(c, [r - 1] * 1025, a)


def _fold_ref(polys, gamma, r, out_len):
    out = [0] * out_len
    g = 1
    for p in polys:
        for j, v in enumerate(p[:out_len]):
            out[j] = (out[j] + g * v) % r
        g = g * gamma % r
    return out


@pytest.mark.parametrize("c", list(FIELDS))
def test_fold(c):
    """out[j] = sum_i gamma^i f_i[j] with unequal lengths (one of length 1), k = 1, gamma = 0, and k = 11 (two launches: the
    second accumulates)"""
    kzg = _kzg()
    r = kzg.CURVE_PARAMS[c].r
    rng = random.Random(47 + FIELDS[c])
    cases = [([300, 5, 1, 77], rng.randrange(r)), ([64], rng.randrange(r)), ([40, 90, 3], 0), ([33, 7, 1, 50, 2, 9, 64, 1, 12, 70, 5], r - 1)]
    for lens, gamma in cases:
        polys = [[rng.randrange(r) for _ in range(m)] for m in lens]
        polys[0][0] = r - 1
        enc = [curves._fr_encode(p, r) for p in polys]
        out_len = max(lens)
        out = np.full((out_len, enc[0].shape[1]), 0xFFFFFFFFFFFFFFFF, dtype=np.uint64)     # garbage: the first launch overwrites
        ptrs = (ctypes.c_void_p * len(enc))(*[e.ctypes.data for e in enc])
        ln = np.array(lens, dtype=np.uint64)
        g = curves._fr_encode([gamma], r)
        rc = _lib().emu_poly_fold(FIELDS[c], ptrs, _ptr(ln), ctypes.c_uint64(len(enc)), _ptr(g), _ptr(out), ctypes.c_uint64(out_len))
        assert rc == 0
        assert np.array_equal(out, curves._fr_encode(_fold_ref(polys, gamma, r, out_len), r)), (lens, gamma)
