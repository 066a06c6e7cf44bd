"""The Fr kernels of permutation.Prove (perm_kernels.cuh: tile batch inversion, ratio, prefix-product levels, numerator) run on the CPU
through the kernel emulation of tests/emu (tests/emu/emu_perm.cpp, cooperative launcher for the kernels with barriers) in the launch
order of fft.cu's entry points, for all seven scalar fields, and compared limb for limb with the big-int restatements of
tests/permutation_ref.py.  Also the argument errors permutation.Prove raises before any device work.  CPU only; a test artefact
(build/libgmsm_emu_perm.so), never part of libgmsm.so."""
import ctypes
import importlib
import os
import random
import subprocess

import numpy as np
import pytest

from tests import permutation_ref as ref

curves = importlib.import_module("gnark-crypto_b200.curves")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "gnark-crypto_b200", "csrc")
EMU = os.path.join(ROOT, "tests", "emu")
OUT = os.path.join(ROOT, "gnark-crypto_b200", "build", "libgmsm_emu_perm.so")
FIELDS = {"bn254": 0, "bls12381": 1, "bls12377": 2, "bls24315": 3, "bls24317": 4, "bw6633": 5, "bw6761": 6}
# (log2 chunk length, log2 block size) of the prefix-product scan in fft.cu for 32-, 40- and 48-byte elements
SCAN_SHAPE = {32: (2, 8), 40: (3, 7), 48: (2, 7)}
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
            subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-I", EMU, "-I", CSRC, os.path.join(EMU, "emu_perm.cpp"),
                            "-o", OUT], check=True)
        _LIB = ctypes.CDLL(OUT)
    return _LIB


def _kzg():
    return importlib.import_module("gnark-crypto_b200.kzg")


def _ptr(a):
    return ctypes.c_void_p(a.ctypes.data)


def _enc(vals, c):
    kzg = _kzg()
    return curves._fr_encode(vals, kzg.CURVE_PARAMS[c].r)


def _check_limbs(got, want_vals, c, what):
    want = _enc(want_vals, c)
    bad = np.nonzero((got != want).any(axis=1))[0]
    assert bad.size == 0, "%s %s: first mismatch at %d of %d" % (c, what, bad[0], len(want_vals))


def _invert(c, vals, log_t=-1, threads=0):
    a = _enc(vals, c)
    out = np.full_like(a, 0xFFFFFFFFFFFFFFFF)
    rc = _lib().emu_perm_invert(FIELDS[c], _ptr(a), ctypes.c_uint64(len(vals)), _ptr(out), log_t, ctypes.c_uint(threads))
    assert rc == 0, rc
    return out


def _accumulate(c, t1, t2, eps, log_t=-1, threads=0, shape=(-1, -1)):
    a, b, e = _enc(t1, c), _enc(t2, c), _enc([eps], c)
    z = np.full_like(a, 0xFFFFFFFFFFFFFFFF)
    rc = _lib().emu_perm_accumulate(FIELDS[c], _ptr(a), _ptr(b), ctypes.c_uint64(len(t1)), _ptr(e), _ptr(z), log_t, ctypes.c_uint(threads),
                                    shape[0], shape[1])
    assert rc == 0, "rc = %d (2: an input was modified)" % rc
    return z


def _zero_patterns(n, rng, r):
    vals = [rng.randrange(1, r) for _ in range(n)]
    out = [list(vals)]
    for pos in ([0], [n - 1], list(range(n // 3, n // 3 + max(n // 4, 1))), list(range(0, n, 3)), list(range(n))):
        v = list(vals)
        for p in pos:
            v[p] = 0
        out.append(v)
    v = list(vals)
    v[rng.randrange(n)] = r - 1
    v[rng.randrange(n)] = 1
    out.append(v)
    return out


@pytest.mark.parametrize("c", list(FIELDS))
def test_batch_invert(c):
    """fr.BatchInvert, zero -> zero: zeros at the start, at the end, in a run, every third and everywhere; lengths 1, T - 1, T,
    T + 1 and 2T + 5 (T = 512, the tile of fft.cu) and, at forced tiles of 8 and 1 elements, lengths crossing several tiles"""
    r = _kzg().CURVE_PARAMS[c].r
    rng = random.Random(3 + FIELDS[c])
    for n, log_t, threads in ((1, -1, 0), (511, -1, 0), (512, -1, 0), (513, -1, 0), (1029, -1, 0), (37, 3, 4), (8, 3, 1), (9, 0, 1)):
        for vals in _zero_patterns(n, rng, r):
            _check_limbs(_invert(c, vals, log_t, threads), ref.batch_invert(vals, r), c, "BatchInvert n=%d" % n)


def _perm_case(n, rng, r):
    t1 = [rng.randrange(r) for _ in range(n)]
    t2 = list(t1)
    rng.shuffle(t2)
    return t1, t2


@pytest.mark.parametrize("c", list(FIELDS))
def test_accumulate_levels(c):
    """the accumulation polynomial in the bit-reversed layout: one and two scan levels at the scan tile of fft.cu
    (T = 1024, n up to 4T; three need n > T^2) and at forced small tiles (T = 8 and T = 2: n up to 2^10 reaches four and more levels)"""
    cp = _kzg().CURVE_PARAMS[c]
    r = cp.r
    rng = random.Random(17 + FIELDS[c])
    log_l, log_b = SCAN_SHAPE[cp.fr_bytes]
    t = 1 << (log_l + log_b)
    cases = [(n, -1, 0, (-1, -1)) for n in (1, 2, t // 2, t, 2 * t, 4 * t)]
    cases += [(n, 3, 2, (1, 2)) for n in (1, 2, 4, 8, 16, 64, 128)] + [(n, 2, 1, (0, 1)) for n in (2, 8, 32, 1024)]
    for n, log_t, threads, shape in cases:
        t1, t2 = _perm_case(n, rng, r)
        eps = rng.randrange(r)
        _check_limbs(_accumulate(c, t1, t2, eps, log_t, threads, shape), ref.accumulate(t1, t2, eps, r), c, "accumulate n=%d" % n)


@pytest.mark.parametrize("c", list(FIELDS))
def test_accumulate_forced_epsilon(c):
    """eps equal to some t2[k] (every z_lin past k + 1 is zero in the reference and here) and to some t1[k] (the numerator factor
    vanishes), at the default shapes and at small tiles; both also at k = 0 and k = n - 1"""
    r = _kzg().CURVE_PARAMS[c].r
    rng = random.Random(41 + FIELDS[c])
    for n, log_t, threads, shape in ((2048, -1, 0, (-1, -1)), (256, 3, 2, (1, 2)), (16, 1, 1, (0, 1))):
        t1, t2 = _perm_case(n, rng, r)
        for k in (0, n // 3, n - 1):
            for eps in (t2[k], t1[k]):
                want = ref.accumulate(t1, t2, eps, r)
                _check_limbs(_accumulate(c, t1, t2, eps, log_t, threads, shape), want, c, "accumulate eps at k=%d n=%d" % (k, n))
        want = ref.accumulate(t1, t2, t2[n // 3], r)
        assert all(want[ref.rev(k, n)] == 0 for k in range(n // 3 + 1, n))   # the zero case is exercised: z_lin[k] = 0 past n / 3


def _numerator(c, n, lt1, lt2, lz, eps, omega, log_t=-1, threads=0):
    r = _kzg().CURVE_PARAMS[c].r
    d = ref.domain(c, n)
    w, g = d.generator, d.shift
    tw = _enc([pow(w, j, r) for j in range(max(n // 2, 1))], c)
    tn_inv = pow((pow(g, n, r) - 1) % r, r - 2, r)
    consts = _enc([eps, omega, g, tn_inv], c)
    a, b, z = _enc(lt1, c), _enc(lt2, c), _enc(lz, c)
    out = np.full_like(a, 0xFFFFFFFFFFFFFFFF)
    rc = _lib().emu_perm_numerator(FIELDS[c], _ptr(a), _ptr(b), _ptr(z), ctypes.c_uint64(n), _ptr(tw), _ptr(consts), _ptr(out), log_t,
                                   ctypes.c_uint(threads))
    assert rc == 0
    return out, ref.numerator(lt1, lt2, lz, eps, omega, n, g, w, r)


@pytest.mark.parametrize("c", list(FIELDS))
def test_numerator(c):
    """the numerator against evaluateFirstPartNumReverse / evaluateSecondPartNumReverse and the omega-fold at n = 1 ... 2^10 on
    random operands (one run with lz = 1 everywhere: the second part vanishes), at the tile of fft.cu and at tiles of 4"""
    r = _kzg().CURVE_PARAMS[c].r
    rng = random.Random(59 + FIELDS[c])
    for logn in range(0, 11):
        n = 1 << logn
        vals = [[rng.randrange(r) for _ in range(n)] for _ in range(3)]
        eps, omega = rng.randrange(r), rng.randrange(r)
        got, want = _numerator(c, n, *vals, eps, omega)
        _check_limbs(got, want, c, "numerator n=%d" % n)
        if logn in (3, 6):
            got, want = _numerator(c, n, *vals, eps, omega, log_t=2, threads=2)
            _check_limbs(got, want, c, "numerator n=%d tile 4" % n)
    got, want = _numerator(c, 64, [rng.randrange(r) for _ in range(64)], [0] * 64, [1] * 64, r - 1, 0)
    _check_limbs(got, want, c, "numerator lz = 1")


def test_prove_argument_errors():
    """the errors Prove raises before it touches a device: mismatched lengths, then a length that is not a power of two (0, 3, 6)"""
    perm = importlib.import_module("gnark-crypto_b200.permutation")
    kzg = _kzg()

    class NoDeviceKey:
        curve, device = "bn254_g1", 0
        G1 = np.zeros((64, 8), dtype=np.uint64)

    t = curves._fr_encode(list(range(8)), kzg.CURVE_PARAMS["bn254"].r)
    with pytest.raises(perm.ErrIncompatibleSize, match="^t1 and t2 should be of the same size$"):
        perm.Prove(NoDeviceKey(), t, t[:4])
    with pytest.raises(perm.ErrIncompatibleSize):
        perm.Prove(NoDeviceKey(), t[:0], t[:3])
    for n in (0, 3, 6):
        with pytest.raises(perm.ErrSize, match="^t1 and t2 should be of size a power of 2$"):
            perm.Prove(NoDeviceKey(), t[:n], t[:n])
    assert issubclass(perm.ErrSize, importlib.import_module("gnark-crypto_b200.multiexp").MultiExpError)
