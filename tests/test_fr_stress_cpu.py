"""The CPU twin of tests/test_gpu_fr_stress.py: the Fr linear combination, the n = 2 butterflies, every FFT variant on extreme
vectors up to 2^11 and the opening scan at three carry levels (small tile shapes), run through the kernel emulation of tests/emu
built with -DGMSM_EMULATE_PTX -- the device's carry-chain source over emulated carries, where a dropped carry traps -- and
checked with the generators and references of tests/fr_stress.py.  It checks those generators and references on a machine
without a GPU, and it separates a formulation error (fails here too) from a PTX / compiler one (fails on the device only).
CPU only; test artefacts (build/libgmsm_emu_*_ptx.so), never part of libgmsm.so."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

from tests import fr_stress as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "gnark-crypto_b200", "csrc")
EMU = os.path.join(ROOT, "tests", "emu")
BUILD = os.path.join(ROOT, "gnark-crypto_b200", "build")
SOURCES = ["emu_lincomb", "emu_fft_more", "emu_poly"]
_LIBS = {}


def _lib(src):
    """build/libgmsm_<src>_ptx.so; the three are compiled together on first use"""
    if not _LIBS:
        os.makedirs(BUILD, exist_ok=True)
        deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))] + [
            os.path.join(EMU, f) for f in os.listdir(EMU)]
        newest = max(os.path.getmtime(d) for d in deps)
        outs = {s: os.path.join(BUILD, "libgmsm_%s_ptx.so" % s) for s in SOURCES}
        procs = []
        for s, out in outs.items():
            if not os.path.exists(out) or os.path.getmtime(out) < newest:
                tmp = "%s.%d.tmp" % (out, os.getpid())
                # tests/emu FIRST: its cuda_runtime.h stands in for the real one
                p = subprocess.Popen(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-DGMSM_EMULATE_PTX", "-I", EMU, "-I", CSRC,
                                      os.path.join(EMU, s + ".cpp"), "-o", tmp])
                procs.append((p, tmp, out))
        for p, tmp, out in procs:
            assert p.wait() == 0, "g++ failed for " + out
            os.replace(tmp, out)
        for s, out in outs.items():
            _LIBS[s] = ctypes.CDLL(out)
    return _LIBS[src]


def _ptr(a):
    return ctypes.c_void_p(a.ctypes.data)


def _lincomb(c):
    def run(polys, scalars, strides, offsets, out_len, init):
        w = R.fr(c).limbs
        polys = [np.ascontiguousarray(p, dtype=np.uint64) for p in polys]
        ptrs = (ctypes.c_void_p * len(polys))(*[p.ctypes.data for p in polys])
        ln = np.array([len(p) for p in polys], dtype=np.uint64)
        st = np.array(strides, dtype=np.uint64)
        off = np.array(offsets, dtype=np.uint64)
        sc = np.ascontiguousarray(scalars, dtype=np.uint64)
        out = init.copy() if init is not None else np.full((out_len, w), 0xFFFFFFFFFFFFFFFF, dtype=np.uint64)
        rc = _lib("emu_lincomb").emu_poly_lincomb(R.FIELD[c], ptrs, _ptr(ln), _ptr(sc), _ptr(st), _ptr(off), ctypes.c_uint64(len(polys)),
                                                  _ptr(out), ctypes.c_uint64(out_len), 1 if init is not None else 0)
        assert rc == 0
        return out

    return run


def _consts(c, n):
    od = R.domain(c, n)
    f = R.fr(c)
    return R.pack([f.to_mont(v) for v in (od.generator, od.generator_inv, od.cardinality_inv, od.shift, od.shift_inv)], f.limbs)


def _fft_many(c, a, n, inverse, dec, coset):
    consts = _consts(c, n)
    rc = _lib("emu_fft_more").emu_fft_more_run_many(R.FIELD[c], _ptr(a), ctypes.c_uint64(len(a) // n), ctypes.c_uint64(n), n.bit_length() - 1,
                                                    int(inverse), int(dec), int(coset), _ptr(consts))
    assert rc == 0
    return a


@pytest.mark.parametrize("c", R.CURVES)
def test_lincomb_extremes_emulated(c):
    """every ordered pair of extremes through k_poly_fold<P, false> (x and accumulate) and k_poly_fold<P, true> (the table)"""
    R.check_lincomb_extremes(c, _lincomb(c), "emulated")


@pytest.mark.parametrize("c", R.CURVES)
def test_butterfly_extremes_emulated(c):
    R.check_butterflies(c, lambda buf, inverse, dec: _fft_many(c, buf, 2, inverse, dec, False), "emulated")


@pytest.mark.parametrize("c", R.CURVES)
@pytest.mark.parametrize("logn", [1, 2, 5, 10, 11])
def test_fft_extreme_vectors_emulated(c, logn):
    R.check_fft_extremes(c, logn, lambda a, inverse, dec, coset: _fft_many(c, a, 1 << logn, inverse, dec, coset), "emulated")


def _div(c, shape):
    log_l, log_b = shape

    def run(F, A, quotient):
        n = len(F)
        fa = np.zeros_like(A)
        h = np.zeros((max(n - 1, 1), F.shape[1]), dtype=np.uint64)
        rc = _lib("emu_poly").emu_poly_div(R.FIELD[c], _ptr(F), ctypes.c_uint64(n), _ptr(A), _ptr(h) if quotient else None, _ptr(fa),
                                           log_l, log_b)
        assert rc == 0, "rc = %d (2: the polynomial was modified)" % rc
        return fa, (h[: n - 1] if quotient else None)

    return run


@pytest.mark.parametrize("c", R.CURVES)
def test_scan_three_levels_emulated(c):
    """tiles of T = 8 (chunks of 2, 4 threads) and T = 2 (chunks of 1, 2 threads): n = T^2 + 1 (levels of T^2 + 1, T + 1 and 2
    elements) and T^2 + 5 T + 3 (partial last tiles on two levels), random coefficients, the a values of the device test"""
    rng = random.Random(61 + R.FIELD[c])
    for shape in ((1, 2), (0, 1)):
        t = 1 << sum(shape)
        for n in (t * t + 1, t * t + 5 * t + 3):
            R.check_scan(c, R.random_stored(c, n, 7 * n + R.FIELD[c]), R.scan_points(c, t, rng), _div(c, shape), "emulated T=%d" % t)
