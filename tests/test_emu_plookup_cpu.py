"""The Fr kernels of plookup.ProveLookupVector (plookup_kernels.cuh: the radix sort with its skipped byte passes, the ratio of the
accumulation polynomial over the permutation's prefix product, the quotient numerator) run on the CPU through the kernel emulation of
tests/emu (tests/emu/emu_plookup.cpp, cooperative launcher: the kernels have barriers and warp votes) in the launch order of fft.cu's
entry points, for all seven scalar fields, and compared limb for limb with the big-int restatements of tests/plookup_ref.py.  Also
the argument errors plookup raises before any device work.  CPU only; a test artefact (build/libgmsm_emu_plookup.so), never part of
libgmsm.so."""
import ctypes
import importlib
import os
import random
import subprocess

import numpy as np
import pytest

from tests import plookup_ref as ref

curves = importlib.import_module("gnark-crypto_b200.curves")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "gnark-crypto_b200", "csrc")
EMU = os.path.join(ROOT, "tests", "emu")
OUT = os.path.join(ROOT, "gnark-crypto_b200", "build", "libgmsm_emu_plookup.so")
FIELDS = {"bn254": 0, "bls12381": 1, "bls12377": 2, "bls24315": 3, "bls24317": 4, "bw6633": 5, "bw6761": 6}
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
            subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-I", EMU, "-I", CSRC, os.path.join(EMU, "emu_plookup.cpp"),
                            "-o", OUT], check=True)
        _LIB = ctypes.CDLL(OUT)
    return _LIB


def _kzg():
    return importlib.import_module("gnark-crypto_b200.kzg")


def _ptr(a):
    return ctypes.c_void_p(a.ctypes.data)


def _r(c):
    return _kzg().CURVE_PARAMS[c].r


def _enc(vals, c):
    return curves._fr_encode(vals, _r(c))


def _check_limbs(got, want_vals, c, what):
    want = _enc(want_vals, c)
    bad = np.nonzero((got != want).any(axis=1))[0]
    assert bad.size == 0, "%s %s: first mismatch at %d of %d" % (c, what, bad[0], len(want_vals))


def _sort(c, vals, log_r=-1, log_b=-1):
    a = _enc(vals, c)
    out = np.full_like(a, 0xFFFFFFFFFFFFFFFF)
    passes = ctypes.c_int(-1)
    rc = _lib().emu_plookup_sort(FIELDS[c], _ptr(a), ctypes.c_uint64(len(vals)), _ptr(out), log_r, log_b, ctypes.byref(passes))
    assert rc == 0, "rc = %d (2: the input was modified)" % rc
    _check_limbs(out, ref.sort(vals), c, "sort n=%d" % len(vals))
    return passes.value


def _varying_bytes(vals):
    """byte positions (of the canonical value) at which not every key agrees: the passes the sort runs"""
    diff = 0
    for v in vals:
        diff |= v ^ vals[0]
    return sum(1 for b in range(64) if (diff >> (8 * b)) & 0xFF)


@pytest.mark.parametrize("c", list(FIELDS))
def test_sort(c):
    """random keys, all keys equal, sorted and reversed input, 0 and r - 1 among random keys, small values (most passes skipped), one
    middle byte varying; at forced tiles of 32 keys (many blocks take part) and at the tile of fft.cu; the number of passes run is
    the number of varying byte positions"""
    r = _r(c)
    rng = random.Random(5 + FIELDS[c])
    small = ((5, 0), (5, 1), (6, 0))           # (log_b, log_r): tiles of 32, 64 and 64 keys
    rand = [rng.randrange(r) for _ in range(300)]
    mid = rng.randrange(1 << 100, r >> 8)
    cases = [
        ("random", rand, small),
        ("equal", [rng.randrange(r)] * 100, small),
        ("sorted", sorted(rand)[:150], small[:1]),
        ("reversed", sorted(rand, reverse=True)[:150], small[:1]),
        ("0 and r-1", [0, r - 1] + rand[:100] + [r - 1, 0], small[:1]),
        ("small", [rng.randrange(1 << 10) for _ in range(2000)], small + ((-1, -1),)),
        ("one middle byte", [mid ^ (rng.randrange(256) << 96) for _ in range(400)], small[:2]),
        ("one key", [rng.randrange(r)], small[:1] + ((-1, -1),)),
    ]
    for name, vals, shapes in cases:
        for log_b, log_r in shapes:
            passes = _sort(c, vals, log_r, log_b)
            assert passes == _varying_bytes(vals), (name, passes)
    assert _varying_bytes(cases[1][1]) == 0 and _varying_bytes(cases[6][1]) == 1


def _accumulate(c, f, t, h1, h2, beta, gamma, log_t=-1, threads=0, shape=(-1, -1)):
    vs = [_enc(v, c) for v in (f, t, h1, h2)]
    consts = _enc([beta, gamma], c)
    z = np.full_like(vs[0], 0xFFFFFFFFFFFFFFFF)
    rc = _lib().emu_plookup_accumulate(FIELDS[c], *(_ptr(v) for v in vs), ctypes.c_uint64(len(f)), _ptr(consts), _ptr(z), log_t,
                                       ctypes.c_uint(threads), shape[0], shape[1])
    assert rc == 0, rc
    return z


def _lookup_case(n, rng, r):
    """lf, lt (sorted) and the overlapping halves of sort(lt || lf[:n-1]), as ProveLookupVector builds them"""
    lt = sorted(rng.randrange(r) for _ in range(n))
    lf = [lt[rng.randrange(n)] for _ in range(n)]
    h = sorted(lt + lf[:n - 1])
    return lf, lt, h[:n], h[n - 1:]


@pytest.mark.parametrize("c", list(FIELDS))
def test_accumulate(c):
    """the accumulation polynomial at the tiles of fft.cu (one and two scan levels) and at forced small tiles (up to eight), n = 1 ... 2^11; and
    with beta, gamma chosen so that gamma(1 + beta) + h1[i] + beta h1[i + 1] = 0 (the zero -> zero inversion of fr.BatchInvert zeroes
    z past i + 1)"""
    r = _r(c)
    rng = random.Random(19 + FIELDS[c])
    cases = [(n, -1, 0, (-1, -1)) for n in (1, 2, 8, 512, 2048)] + [(n, 2, 1, (0, 1)) for n in (2, 16, 64, 256)]
    for n, log_t, threads, shape in cases:
        lf, lt, h1, h2 = _lookup_case(n, rng, r)
        beta, gamma = rng.randrange(r), rng.randrange(r)
        got = _accumulate(c, lf, lt, h1, h2, beta, gamma, log_t, threads, shape)
        _check_limbs(got, ref.accumulate(lf, lt, h1, h2, beta, gamma, r), c, "accumulate n=%d" % n)
    for n, log_t, threads, shape in ((1024, -1, 0, (-1, -1)), (64, 2, 1, (0, 1))):
        lf, lt, h1, h2 = _lookup_case(n, rng, r)
        for i in (0, n // 3, n - 2):
            beta = rng.randrange(r)
            gamma = -(h1[i] + beta * h1[i + 1]) * pow(1 + beta, r - 2, r) % r
            want = ref.accumulate(lf, lt, h1, h2, beta, gamma, r)
            assert all(v == 0 for v in want[i + 1:])
            _check_limbs(_accumulate(c, lf, lt, h1, h2, beta, gamma, log_t, threads, shape), want, c, "accumulate zero at %d" % i)


def _numerator(c, n, vals, beta, gamma, alpha, log_t=-1, threads=0):
    r = _r(c)
    d = ref.domain(c, n)
    w, g = d.generator, d.shift
    tw = _enc([pow(w, j, r) for j in range(max(n // 2, 1))], c)
    consts = _enc([beta, gamma, alpha, g, pow(w, r - 2, r)], c)
    a = np.ascontiguousarray(np.concatenate([_enc(v, c) for v in vals]))
    out = np.full((n, a.shape[1]), 0xFFFFFFFFFFFFFFFF, dtype=np.uint64)
    rc = _lib().emu_plookup_numerator(FIELDS[c], _ptr(a), ctypes.c_uint64(n), _ptr(tw), _ptr(consts), _ptr(out), log_t,
                                      ctypes.c_uint(threads))
    assert rc == 0
    return out, ref.numerator(*vals, beta, gamma, alpha, n, g, w, r)


@pytest.mark.parametrize("c", list(FIELDS))
def test_numerator(c):
    """the numerator against evaluateNumBitReversed, the three boundary terms and computeQuotientCanonical's fold at big-domain
    sizes 2 ... 2^10 on random operands, at the tile of fft.cu and at tiles of 4; one run with lz = 1 and lh1 = lh2 (only the
    constraint term is left)"""
    r = _r(c)
    rng = random.Random(61 + FIELDS[c])
    for logn in range(1, 11):
        n = 1 << logn
        vals = [[rng.randrange(r) for _ in range(n)] for _ in range(5)]
        ch = [rng.randrange(r) for _ in range(3)]
        got, want = _numerator(c, n, vals, *ch)
        _check_limbs(got, want, c, "numerator n=%d" % n)
        if logn in (3, 7):
            got, want = _numerator(c, n, vals, *ch, log_t=2, threads=2)
            _check_limbs(got, want, c, "numerator n=%d tile 4" % n)
    h = [rng.randrange(r) for _ in range(64)]
    got, want = _numerator(c, 64, [[1] * 64, h, h, [rng.randrange(r) for _ in range(64)], [0] * 64], 3, 5, 7)
    _check_limbs(got, want, c, "numerator lz = 1")


class _NoDeviceKey:
    curve, device = "bn254_g1", 0
    G1 = np.zeros((64, 8), dtype=np.uint64)


def test_prove_argument_errors():
    """the errors ProveLookupVector and ProveLookupTables raise before they touch a device: an empty f or t (the reference panics),
    an empty table list, unequal row counts and ragged rows (ErrIncompatibleSize)"""
    pl = importlib.import_module("gnark-crypto_b200.plookup")
    key = _NoDeviceKey()
    t = _enc(list(range(8)), "bn254")
    for f_, t_ in ((t[:0], t), (t, t[:0]), (t[:0], t[:0])):
        with pytest.raises(ValueError, match="must not be empty"):
            pl.ProveLookupVector(key, f_, t_)
    with pytest.raises(ValueError, match="must not be empty"):
        pl.ProveLookupTables(key, [], [])
    with pytest.raises(pl.ErrIncompatibleSize, match="^the tables in f and t are not of the same size$"):
        pl.ProveLookupTables(key, [t[:7]] * 3, [t] * 2)
    with pytest.raises(pl.ErrIncompatibleSize):
        pl.ProveLookupTables(key, [t[:7], t[:6], t[:7]], [t] * 3)
    with pytest.raises(pl.ErrIncompatibleSize):
        pl.ProveLookupTables(key, [t[:7]] * 3, [t, t, t[:5]])
    with pytest.raises(ValueError, match="must not be empty"):
        pl.ProveLookupTables(key, [t[:0]] * 2, [t] * 2)
    assert issubclass(pl.ErrIncompatibleSize, importlib.import_module("gnark-crypto_b200.multiexp").MultiExpError)
