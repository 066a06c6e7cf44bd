"""The strided linear combination of poly_kernels.cuh (k_poly_fold with per-input scalar, stride and offset; the kernel behind
gmsm_fr_poly_lincomb_device) run on the CPU through the kernel emulation of tests/emu (tests/emu/emu_lincomb.cpp) in the launch order
of fft.cu, for all seven scalar fields, against a big-integer restatement.  CPU only; a test artefact (build/libgmsm_emu_lincomb.so)."""
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
OUT = os.path.join(ROOT, "gnark-crypto_b200", "build", "libgmsm_emu_lincomb.so")
FIELDS = {"bn254": 0, "bls12381": 1, "bls12377": 2, "bls24315": 3, "bls24317": 4, "bw6633": 5, "bw6761": 6}
GRID = 8 * 256          # threads of one emulated launch (8 blocks of 256): the grid-stride loop wraps past it
_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        os.makedirs(os.path.dirname(OUT), exist_ok=True)
        deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))] + [
            os.path.join(EMU, f) for f in os.listdir(EMU)]
        if not os.path.exists(OUT) or os.path.getmtime(OUT) < max(os.path.getmtime(d) for d in deps):
            # tests/emu FIRST: its cuda_runtime.h stands in for the real one
            subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-I", EMU, "-I", CSRC, os.path.join(EMU, "emu_lincomb.cpp"),
                            "-o", OUT], check=True)
        _LIB = ctypes.CDLL(OUT)
    return _LIB


def _kzg():
    return importlib.import_module("gnark-crypto_b200.kzg")


def _ptr(a):
    return ctypes.c_void_p(a.ctypes.data)


def lincomb_ref(polys, scalars, strides, offsets, out_len, r, init=None):
    """out[m * stride_i + offset_i] += s_i * p_i[m] below out_len, from `init` (accumulate) or zeros"""
    out = list(init) if init is not None else [0] * out_len
    for p, s, st, off in zip(polys, scalars, strides, offsets):
        for m, v in enumerate(p):
            j = m * st + off
            if j < out_len:
                out[j] = (out[j] + s * v) % r
    return out


def _run(c, polys, scalars, strides, offsets, out_len, init=None):
    kzg = _kzg()
    r = kzg.CURVE_PARAMS[c].r
    w = kzg.CURVE_PARAMS[c].fr_words
    enc = [curves._fr_encode(p, r) if p else np.zeros((1, w), dtype=np.uint64) for p in polys]
    out = curves._fr_encode(init, r) if init is not None else np.full((out_len, w), 0xFFFFFFFFFFFFFFFF, dtype=np.uint64)
    ptrs = (ctypes.c_void_p * len(enc))(*[e.ctypes.data for e in enc])
    ln = np.array([len(p) for p in polys], dtype=np.uint64)
    st = np.array(strides, dtype=np.uint64)
    off = np.array(offsets, dtype=np.uint64)
    sc = curves._fr_encode(scalars, r)
    rc = _lib().emu_poly_lincomb(FIELDS[c], ptrs, _ptr(ln), _ptr(sc), _ptr(st), _ptr(off), ctypes.c_uint64(len(polys)), _ptr(out),
                                 ctypes.c_uint64(out_len), 1 if init is not None else 0)
    assert rc == 0
    want = lincomb_ref(polys, scalars, strides, offsets, out_len, r, init)
    assert np.array_equal(out, curves._fr_encode(want, r)), (len(polys), strides, offsets, out_len)


def cases(r, rng):
    """(lens, scalars, strides, offsets, out_len): strides 1, 2, 3 and 9 with offsets; lengths 1 and GRID +- 1; eleven inputs
    (two batches of at most 8); scalars 0, 1 and r - 1; an output shorter than the inputs reach"""
    out = [
        ([GRID - 1, GRID, GRID + 1, 1], [rng.randrange(r), 1, r - 1, 0], [1, 1, 1, 1], [0, 0, 0, 0], GRID + 1),   # the fold shape
        ([GRID // 2 + 1, GRID // 2, 1], [rng.randrange(r), r - 1, 1], [2, 2, 2], [0, 1, 7], GRID + 1),
        ([GRID // 3 + 1, 300, 5], [1, rng.randrange(r), r - 1], [3, 3, 3], [0, 1, 2], 3 * (GRID // 3 + 1)),
        ([100, 99, 1, 40, 7, 1, 100, 3, 100], [rng.randrange(r) for _ in range(9)], [9] * 9, list(range(9)), 900),
        ([33, 7, 1, 50, 2, 9, 64, 1, 12, 70, 5], [rng.randrange(r) for _ in range(10)] + [0], [1, 2, 3, 9, 1, 2, 3, 9, 1, 2, 3],
         [0, 1, 2, 5, 3, 0, 1, 8, 0, 4, 2], 200),
        ([GRID + 1, 64], [r - 1, 1], [1, 9], [5, 3], GRID - 1),                                                      # truncated
    ]
    return out


@pytest.mark.parametrize("c", list(FIELDS))
def test_lincomb(c):
    r = _kzg().CURVE_PARAMS[c].r
    rng = random.Random(83 + FIELDS[c])
    for lens, scalars, strides, offsets, out_len in cases(r, rng):
        polys = [[rng.randrange(r) for _ in range(m)] for m in lens]
        polys[0][0] = r - 1
        _run(c, polys, scalars, strides, offsets, out_len)
        _run(c, polys, scalars, strides, offsets, out_len, init=[rng.randrange(r) for _ in range(out_len)])     # accumulate
