"""The CPU twin of tests/test_gpu_perm_stress.py: the Fr kernels of permutation.Prove and plookup.ProveLookupVector run through the
kernel emulation of tests/emu (tests/emu/emu_perm.cpp, tests/emu/emu_plookup.cpp) at forced small tiles, so that short vectors
reach the shapes the device test reaches at production sizes, and checked with the generators and references of
tests/perm_stress.py: A at tiles of 8, B and C with three and more scan levels at scan tiles of 8 and 2, D at 2^5 and 2^10, E at
31, 33 and 4097 keys over warp-sized sort tiles.  It checks those generators and references on a machine without a GPU, and it
separates a formulation error (fails here too) from a device one (fails on the device only).  CPU only."""
import ctypes
import random

import numpy as np
import pytest

from tests import perm_stress as S
from tests import test_emu_perm_cpu as EP
from tests import test_emu_plookup_cpu as EL


def _ptr(a):
    return ctypes.c_void_p(a.ctypes.data)


def _c(a):
    return np.ascontiguousarray(a, dtype=np.uint64)


# (inverse tile log2, threads) and (chunk log2, block log2) of the scan: T = 8 with two levels below n = 64, T = 2 below n = 4
SMALL = [((3, 2), (1, 2)), ((1, 1), (0, 1))]


def _invert(c, log_t, threads):
    def run(A, in_place):                  # the emulation copies its input: one call covers both
        A = _c(A)
        out = np.full_like(A, 0xFFFFFFFFFFFFFFFF)
        rc = EP._lib().emu_perm_invert(S.FIELD[c], _ptr(A), ctypes.c_uint64(len(A)), _ptr(out), log_t, ctypes.c_uint(threads))
        assert rc == 0, rc
        return out

    return run


@pytest.mark.parametrize("c", S.CURVES)
def test_batch_invert_extremes_emulated(c):
    """tiles of 8 leaves, 4 threads (the thread mask splits at j = 0, 3, 4, 7)"""
    S.check_batch_invert(c, _invert(c, 3, 4), "emulated", random.Random(5 + S.FIELD[c]), log_t=3, threads=4)


def _perm_accumulate(c, inv, shape):
    def run(T1, T2, E):
        T1, T2, E = _c(T1), _c(T2), _c(E)
        z = np.full_like(T1, 0xFFFFFFFFFFFFFFFF)
        rc = EP._lib().emu_perm_accumulate(S.FIELD[c], _ptr(T1), _ptr(T2), ctypes.c_uint64(len(T1)), _ptr(E), _ptr(z), inv[0],
                                           ctypes.c_uint(inv[1]), shape[0], shape[1])
        assert rc == 0, "rc = %d (2: an input was modified)" % rc
        return z

    return run


@pytest.mark.parametrize("c", S.CURVES)
def test_perm_accumulate_levels_emulated(c):
    """n = 2 T^2 and 4 T^2 at T = 8 and T = 2 with eps = t2[k] and t1[k] at every level boundary; eps through the extremes at n = 64"""
    for inv, shape in SMALL:
        t = 1 << sum(shape)
        for n in (2 * t * t, 4 * t * t):
            S.check_perm_accumulate(c, n, t, _perm_accumulate(c, inv, shape), "emulated", n + S.FIELD[c])
    inv, shape = SMALL[0]
    S.check_perm_accumulate(c, 64, 8, _perm_accumulate(c, inv, shape), "emulated", 3, forced=False, eps_extremes=S.extremes(c))


def _plookup_accumulate(c, inv, shape):
    def run(F, T, H1, H2, B, G):
        F, T, H1, H2 = (_c(x) for x in (F, T, H1, H2))
        consts = _c(np.concatenate([B, G]))
        z = np.full_like(F, 0xFFFFFFFFFFFFFFFF)
        rc = EL._lib().emu_plookup_accumulate(S.FIELD[c], _ptr(F), _ptr(T), _ptr(H1), _ptr(H2), ctypes.c_uint64(len(F)), _ptr(consts),
                                              _ptr(z), inv[0], ctypes.c_uint(inv[1]), shape[0], shape[1])
        assert rc == 0, rc
        return z

    return run


@pytest.mark.parametrize("c", S.CURVES)
def test_plookup_accumulate_levels_emulated(c):
    """n = T^2 + 1, T^2 + T - 1 (with the challenge edge cases and the forced zeros at T^2 - 1 and T^2) and 4 T^2 - 1 at T = 8 and
    T = 2"""
    for inv, shape in SMALL:
        t = 1 << sum(shape)
        for n, edges in ((t * t + 1, False), (t * t + t - 1, True), (t * t + t + 1, True), (4 * t * t - 1, False)):
            S.check_plookup_accumulate(c, n, t, _plookup_accumulate(c, inv, shape), "emulated", n + S.FIELD[c], edges=edges)


def _perm_numerator(c, n, log_t, threads):
    f = S.fr(c)
    r = f.q
    d = S.domain(c, n)
    tw = S.pack([f.to_mont(pow(d.generator, j, r)) for j in range(max(n // 2, 1))], f.limbs)
    g = d.shift

    def run(LT1, LT2, LZ, E, O):
        LT1, LT2, LZ = _c(LT1), _c(LT2), _c(LZ)
        consts = _c(np.concatenate([E, O, S.pack([f.to_mont(g), f.to_mont(pow((pow(g, n, r) - 1) % r, -1, r))], f.limbs)]))
        out = np.full_like(LT1, 0xFFFFFFFFFFFFFFFF)
        rc = EP._lib().emu_perm_numerator(S.FIELD[c], _ptr(LT1), _ptr(LT2), _ptr(LZ), ctypes.c_uint64(n), _ptr(tw), _ptr(consts), _ptr(out),
                                          log_t, ctypes.c_uint(threads))
        assert rc == 0
        return out

    return run


def _plookup_numerator(c, n, log_t, threads):
    f = S.fr(c)
    r = f.q
    d = S.domain(c, n)
    tw = S.pack([f.to_mont(pow(d.generator, j, r)) for j in range(max(n // 2, 1))], f.limbs)
    tail = S.pack([f.to_mont(d.shift), f.to_mont(d.generator_inv)], f.limbs)

    def run(LZ, LH1, LH2, LT, LF, B, G, A):
        vec = _c(np.concatenate([LZ, LH1, LH2, LT, LF]))
        consts = _c(np.concatenate([B, G, A, tail]))
        out = np.full((n, f.limbs), 0xFFFFFFFFFFFFFFFF, dtype=np.uint64)
        rc = EL._lib().emu_plookup_numerator(S.FIELD[c], _ptr(vec), ctypes.c_uint64(n), _ptr(tw), _ptr(consts), _ptr(out), log_t,
                                             ctypes.c_uint(threads))
        assert rc == 0
        return out

    return run


@pytest.mark.parametrize("c", S.CURVES)
def test_numerators_emulated(c):
    """every challenge through the extremes on inputs cycling the extremes at n = 2^5 (tiles of 4), random inputs at n = 2^10 (the
    tile of fft.cu, every position)"""
    rng = random.Random(99 + S.FIELD[c])
    S.check_perm_numerator(c, 32, _perm_numerator(c, 32, 2, 2), "emulated", rng, sweep=True)
    S.check_plookup_numerator(c, 32, _plookup_numerator(c, 32, 2, 2), "emulated", rng, sweep=True)
    S.check_perm_numerator(c, 1 << 10, _perm_numerator(c, 1 << 10, -1, 0), "emulated", rng)
    S.check_plookup_numerator(c, 1 << 10, _plookup_numerator(c, 1 << 10, -1, 0), "emulated", rng)


def _sort(c, log_r, log_b):
    def run(A, in_place):                  # the emulation copies its input: one call covers both
        A = _c(A)
        out = np.full_like(A, 0xFFFFFFFFFFFFFFFF)
        passes = ctypes.c_int(0)
        rc = EL._lib().emu_plookup_sort(S.FIELD[c], _ptr(A), ctypes.c_uint64(len(A)), _ptr(out), log_r, log_b, ctypes.byref(passes))
        assert rc == 0, rc
        return out

    return run


@pytest.mark.parametrize("c", S.CURVES)
def test_sort_adversarial_emulated(c):
    """tiles of one warp and two rounds (64 keys): n = 31 and 33 with the single differing keys, the two-byte keys and the
    dominating digit; for bn254 every distribution at 33 and the short list at 4097 (a second tile of the difference mask).  The
    emulated passes cost milliseconds per block, so the long vectors are left to the device test"""
    for n, brief in ((31, True), (33, c != "bn254")) + (((4097, True),) if c == "bn254" else ()):
        S.check_sort(c, n, _sort(c, 1, 5), "emulated", n + 17 * S.FIELD[c], in_place_too=False, brief=brief)
