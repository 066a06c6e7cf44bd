"""The kernels of the iop package (iop_kernels.cuh: the two ratio kernels with the permutation argument's prefix product, the Lagrange
evaluation, the Evaluate interpreter and the elementwise step of DivideByXMinusOne) run on the CPU through the kernel emulation of
tests/emu (tests/emu/emu_iop.cpp) in the launch order of fft.cu's entry points, for all seven scalar fields, and compared limb for
limb with the restatement of tests/iop_ref.py.  Forced small tiles make the prefix product run at three levels, and zero denominators
are planted at inversion-tile and scan-level boundaries.  CPU only; a test artefact (build/libgmsm_emu_iop.so), never part of
libgmsm.so."""
import ctypes
import importlib
import os
import random
import subprocess

import numpy as np
import pytest

from tests import iop_ref as R
from tests.permutation_ref import domain, rev

curves = importlib.import_module("gnark-crypto_b200.curves")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "gnark-crypto_b200", "csrc")
EMU = os.path.join(ROOT, "tests", "emu")
OUT = os.path.join(ROOT, "gnark-crypto_b200", "build", "libgmsm_emu_iop.so")
FIELDS = {"bn254": 0, "bls12381": 1, "bls12377": 2, "bls24315": 3, "bls24317": 4, "bw6633": 5, "bw6761": 6}
# forced shapes: inversion tiles of 8 elements on 2 threads, scan tiles of 4 (chunks of 2 on 2 threads): n = 64 runs the prefix
# product over the levels 64 -> 16 -> 4 -> 1
SMALL = dict(log_t=3, threads=2, log_l=1, log_b=1)
DEFAULT = dict(log_t=-1, threads=0, log_l=-1, log_b=-1)
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
            subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-I", EMU, "-I", CSRC, os.path.join(EMU, "emu_iop.cpp"),
                            "-o", OUT], check=True)
        _LIB = ctypes.CDLL(OUT)
    return _LIB


def _r(c):
    return curves.CURVE_PARAMS[c].r


def _enc(vals, c):
    return curves._fr_encode([v % _r(c) for v in vals], _r(c))


def _dec(a, c):
    return curves._fr_decode(a, _r(c))


def _ptr(a):
    return ctypes.c_void_p(a.ctypes.data)


def _ptrs(arrs):
    return (ctypes.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])


def _ints(v):
    return (ctypes.c_int * len(v))(*[int(x) for x in v])


def _tw(c, n):
    d = domain(c, n)
    return _enc([pow(d.generator, j, _r(c)) for j in range(max(n // 2, 1))], c), d


def _shuffled(c, num, num_br, den, den_br, beta, shape):
    n = len(num[0])
    N, D = [_enc(v, c) for v in num], [_enc(v, c) for v in den]
    z = np.full((n, curves.CURVE_PARAMS[c].fr_words), 0xFFFFFFFFFFFFFFFF, dtype=np.uint64)
    b = _enc([beta], c)        # every buffer is held for the call: a temporary's memory could be reused before the library reads it
    rc = _lib().emu_iop_ratio_shuffled(FIELDS[c], _ptrs(N), _ints(num_br), _ptrs(D), _ints(den_br), len(num), ctypes.c_uint64(n),
                                       _ptr(b), _ptr(z), shape["log_t"], ctypes.c_uint(shape["threads"]), shape["log_l"],
                                       shape["log_b"])
    assert rc == 0, rc
    return _dec(z, c)


def _copy(c, cols, br, sigma, beta, gamma, shape):
    n = len(cols[0])
    tw, d = _tw(c, n)
    C = [_enc(v, c) for v in cols]
    s = np.ascontiguousarray(sigma, dtype=np.int64)
    z = np.full((n, curves.CURVE_PARAMS[c].fr_words), 0xFFFFFFFFFFFFFFFF, dtype=np.uint64)
    z0 = z.copy()
    k = _enc([beta, gamma, d.shift], c)
    rc = _lib().emu_iop_ratio_copy(FIELDS[c], _ptrs(C), _ints(br), len(cols), ctypes.c_uint64(n), _ptr(s), _ptr(tw),
                                   _ptr(k), _ptr(z), shape["log_t"], ctypes.c_uint(shape["threads"]),
                                   shape["log_l"], shape["log_b"])
    if rc == 3:
        assert (z == z0).all(), "the output was written before sigma was refused"
        return None
    assert rc == 0, rc
    return _dec(z, c)


def _store(vals, br):
    """the storage of Lagrange values in a Regular or BitReverse layout"""
    return R.bit_reverse(vals) if br else list(vals)


ZERO_AT = (3, 4, 7, 8, 15, 16, 31, 32, 47, 48, 62)   # scan tiles of 4, levels of 16, inversion tiles of 8; i < n - 1 = 63


@pytest.mark.parametrize("c", list(FIELDS))
def test_ratio_shuffled(c):
    """the shuffled-vectors ratio at n = 1 ... 2^10 at the default shapes and with three scan levels at forced small tiles, k = 1 ... 3
    with mixed layouts; a zero denominator planted at every tile and level boundary zeroes every later Z[k], as in the reference"""
    r = _r(c)
    rng = random.Random(7 + FIELDS[c])
    cases = [(n, DEFAULT) for n in (1, 2, 64, 1024)] + [(n, SMALL) for n in (2, 8, 64)]
    for n, shape in cases:
        for k in (1, 2, 3):
            num = [[rng.randrange(r) for _ in range(n)] for _ in range(k)]
            den = [[rng.randrange(r) for _ in range(n)] for _ in range(k)]
            nb, db = [j % 2 for j in range(k)], [(j + 1) % 2 for j in range(k)]
            beta = rng.randrange(r)
            got = _shuffled(c, [_store(v, b) for v, b in zip(num, nb)], nb, [_store(v, b) for v, b in zip(den, db)], db, beta, shape)
            want = R.ratio_shuffled([R.poly(_store(v, b), 2, 16 if b else 8) for v, b in zip(num, nb)],
                                    [R.poly(_store(v, b), 2, 16 if b else 8) for v, b in zip(den, db)], beta, (2, 8), c, r)["c"]
            assert got == want, (c, n, k, shape)
    n = 64
    num = [[rng.randrange(r) for _ in range(n)] for _ in range(2)]
    for p in ZERO_AT:
        den = [[rng.randrange(r) for _ in range(n)] for _ in range(2)]
        beta = rng.randrange(r)
        den[1][p] = beta                                   # beta - Q_1[p] = 0
        got = _shuffled(c, num, [0, 0], [den[0], R.bit_reverse(den[1])], [0, 1], beta, SMALL)
        want = R.ratio_shuffled([R.poly(v, 2, 8) for v in num], [R.poly(den[0], 2, 8), R.poly(R.bit_reverse(den[1]), 2, 16)], beta,
                                (2, 8), c, r)["c"]
        assert got == want and all(v == 0 for v in got[p + 1:]) and got[p] != 0, (c, p)


def _sigma(k, n, rng):
    s = list(range(k * n))
    rng.shuffle(s)
    return s


@pytest.mark.parametrize("c", list(FIELDS))
def test_ratio_copy(c):
    """the copy-constraint ratio with ID[sigma] formed from the twiddles, k = 1 ... 4, mixed layouts, n = 1 ... 2^10 at the default
    shapes and n up to 64 at forced small tiles (three scan levels); gamma chosen to zero the denominator at every tile and level
    boundary; sigma with an entry outside [0, k n) is refused before the output is written"""
    r = _r(c)
    rng = random.Random(19 + FIELDS[c])
    cases = [(n, DEFAULT) for n in (1, 2, 64, 1024)] + [(n, SMALL) for n in (2, 8, 64)]
    for n, shape in cases:
        for k in (1, 2, 4):
            cols = [[rng.randrange(r) for _ in range(n)] for _ in range(k)]
            br = [j % 2 for j in range(k)]
            sigma = _sigma(k, n, rng)
            beta, gamma = rng.randrange(r), rng.randrange(r)
            st = [_store(v, b) for v, b in zip(cols, br)]
            got = _copy(c, st, br, sigma, beta, gamma, shape)
            want = R.ratio_copy([R.poly(v, 2, 16 if b else 8) for v, b in zip(st, br)], sigma, beta, gamma, (2, 8), c, r)["c"]
            assert got == want, (c, n, k, shape)
    n, k = 64, 2
    cols = [[rng.randrange(r) for _ in range(n)] for _ in range(k)]
    d = domain(c, n)
    for p in ZERO_AT:
        sigma = _sigma(k, n, rng)
        beta = rng.randrange(1, r)
        s = sigma[n + p]                                   # column 1 at position p
        gamma = (-cols[1][p] - beta * pow(d.shift, s // n, r) * pow(d.generator, s % n, r)) % r
        got = _copy(c, cols, [0, 0], sigma, beta, gamma, SMALL)
        want = R.ratio_copy([R.poly(v, 2, 8) for v in cols], sigma, beta, gamma, (2, 8), c, r)["c"]
        assert got == want and all(v == 0 for v in got[p + 1:]), (c, p)
    for bad in (-1, k * n, 1 << 40):
        sigma = _sigma(k, n, rng)
        sigma[rng.randrange(k * n)] = bad
        assert _copy(c, cols, [0, 0], sigma, 1, 2, SMALL) is None


@pytest.mark.parametrize("c", list(FIELDS))
def test_lagrange_eval(c):
    """evalLagrange in both layouts at n = 1 ... 2^10 at random x, at x on the domain (0) and at x = 0, at the default shapes and with
    tiles of 8 summed by 2 and 4 threads"""
    r = _r(c)
    rng = random.Random(23 + FIELDS[c])
    for n in (1, 2, 8, 64, 1024):
        tw, d = _tw(c, n)
        vals = [rng.randrange(r) for _ in range(n)]
        for x in (rng.randrange(r), pow(d.generator, n // 3, r), 0):
            scale = (pow(x, n, r) - 1) * pow(n, r - 2, r) % r
            for bitrev in (0, 1):
                for log_t, threads, sum_threads in ((-1, 0, 0), (3, 2, 4), (3, 4, 2)):
                    out = np.zeros((1, curves.CURVE_PARAMS[c].fr_words), dtype=np.uint64)
                    cv, k = _enc(vals, c), _enc([x, scale], c)
                    rc = _lib().emu_iop_lagrange_eval(FIELDS[c], _ptr(cv), ctypes.c_uint64(n), bitrev, _ptr(tw),
                                                      _ptr(k), _ptr(out), log_t, ctypes.c_uint(threads),
                                                      ctypes.c_uint(sum_threads))
                    assert rc == 0
                    want = R.evaluate(R.poly(vals, 2, 16 if bitrev else 8), x, c, r)
                    assert _dec(out, c)[0] == want, (c, n, x, bitrev, log_t)


@pytest.mark.parametrize("c", list(FIELDS))
def test_evaluate_interpreter(c):
    """traced programs run by the interpreter kernel over inputs of mixed layouts and shifts, into both result layouts, against
    Evaluate restated; one program over 20 inputs and one constant-only program"""
    iop = importlib.import_module("gnark-crypto_b200.iop")
    r = _r(c)
    rng = random.Random(29 + FIELDS[c])
    progs = [
        (lambda i, a, b, z: a * b + 3 * a - b ** 5 + z * i - 7, lambda i, a, b, z: a * b + 3 * a - pow(b, 5, r) + z * i - 7, 3),
        (lambda i, *x: sum(x[1:], x[0]) - x[3] * x[7] * i, lambda i, *x: sum(x) - x[3] * x[7] * i, 20),
        (lambda i, a: 11, lambda i, a: 11, 1),
    ]
    for n in (1, 8, 64):
        for f, fi, m in progs:
            prog = iop.trace(f, m, r)
            vals = [[rng.randrange(r) for _ in range(n)] for _ in range(m)]
            lay = [(16 if j % 3 == 1 else 8, j % 4, n >> (j % 3)) for j in range(m)]   # layout, shift, size
            polys = [R.poly(v, 2, L, s, max(sz, 1)) for v, (L, s, sz) in zip(vals, lay)]
            offs = np.array([((n // p["size"]) * p["shift"]) % n for p in polys], dtype=np.uint64)
            ins = [_enc(v, c) for v in vals]
            for out_br in (0, 1):
                out = np.zeros((n, curves.CURVE_PARAMS[c].fr_words), dtype=np.uint64)
                code = np.array(prog.code, dtype=np.uint32)
                consts = _enc(prog.consts, c) if prog.consts else np.zeros((1, curves.CURVE_PARAMS[c].fr_words), dtype=np.uint64)
                rc = _lib().emu_iop_evaluate(FIELDS[c], _ptr(code), len(prog.code), prog.out, _ptr(consts), len(prog.consts), _ptrs(ins),
                                             _ptr(offs), _ints([L == 16 for L, _, _ in lay]), m, ctypes.c_uint64(n), out_br, _ptr(out))
                assert rc == 0
                want = R.evaluate_expr(lambda i, *x: fi(i, *x) % r, (2, 16 if out_br else 8), polys, r)["c"]
                assert _dec(out, c) == want, (c, n, m, out_br)


@pytest.mark.parametrize("c", list(FIELDS))
def test_divide_step(c):
    """out[rev(i)] = a.GetCoeff(i) inv[i mod rho] for rho = 1, 2, 4, 8 and 64, both input layouts and shifts 0, 1 and 3"""
    r = _r(c)
    rng = random.Random(31 + FIELDS[c])
    for n, rho in ((8, 1), (16, 2), (64, 4), (64, 8), (128, 64)):
        a = [rng.randrange(r) for _ in range(n)]
        inv = [rng.randrange(r) for _ in range(rho)]
        for br in (0, 1):
            for shift in (0, 1, 3):
                p = R.poly(a, 4, 16 if br else 8, shift, n // rho)
                out = np.zeros((n, curves.CURVE_PARAMS[c].fr_words), dtype=np.uint64)
                av, iv = _enc(a, c), _enc(inv, c)
                rc = _lib().emu_iop_divide(FIELDS[c], _ptr(av), ctypes.c_uint64(n), ctypes.c_uint64((rho * shift) % n), br,
                                           _ptr(iv), ctypes.c_uint(rho), _ptr(out))
                assert rc == 0
                want = [0] * n
                for i in range(n):
                    want[rev(i, n)] = R.get_coeff(p, i) * inv[i % rho] % r
                assert _dec(out, c) == want, (c, n, rho, br, shift)
