"""The sm_90a Fr kernels of permutation.Prove and plookup.ProveLookupVector of the seven pairing curves at extreme operands,
adversarial keys and production sizes (generators and references in tests/perm_stress.py; the CPU twin is
tests/test_perm_stress_cpu.py):

A. the tile batch inversion as the Fr fp_inv: every extreme alone in its tile of 512 (the tile root is the extreme), every
   extreme at n = 1, 4096 random values one per tile, dense tiles of r - 1, of zeros and of zeros where the thread mask splits;
   in place and out of place;
B. the permutation accumulation where the scan has three levels (n > T^2, T the scan tile: 2^21 for the 32-byte fields and
   bw6-633, 2^22 for bn254, 2^19 and 2^20 for bw6-761), the whole bit-reversed output against the sequential reference, with
   eps = t2[k] and eps = t1[k] at the level boundaries (at the smaller size of each field); eps through every extreme at n = 2^12;
C. the plookup accumulation at n = T^2 + 1, T^2 + T - 1 (with beta = r - 1, beta = 0, gamma = 0 and gamma zeroing a denominator at
   k = T^2 - 1 and T^2) and, for bn254, 2^22 - 1 and 2^22;
D. both numerators at 2^20 / 2^22 (permutation) and 2s = 2^21 / 2^23 (plookup) where the 2-adicity allows, at >= 4096 storage
   positions against per-position references (the twiddles past 2^13, the negated upper half, rev(p) and the neighbour's wrap);
   at 2^10 every challenge through the extremes on inputs cycling the extremes;
E. the sort on adversarial keys (one differing key far from key 0, one- and two-byte keys in place and out of place, 0 / 1 / r - 1,
   sorted and reversed, warp digit patterns, one dominating digit) at 31 ... 4097 and 2^21 + 1 for every field, 2^23 - 1 for
   bn254 and bw6-761.

The long sequential references of B and C run in a pool of worker processes while the device computes."""
import multiprocessing
import os
import random
from concurrent.futures import ProcessPoolExecutor
from importlib import import_module

import numpy as np
import pytest

from tests import perm_stress as S

pytestmark = pytest.mark.gpu


def _torch():
    return import_module("torch")


def _lib():
    return import_module("gnark-crypto_b200._native").lib()


def _err():
    return import_module("gnark-crypto_b200._native").last_error()


def _fft():
    import gnark_crypto_b200  # noqa: F401

    return import_module("gnark-crypto_b200.fft")


def _dev(a):
    return _torch().from_numpy(np.ascontiguousarray(a, dtype=np.uint64).view(np.int64).reshape(-1).copy()).cuda()


def _host(t, w):
    return t.cpu().numpy().view(np.uint64).reshape(-1, w)


def _stream():
    return _torch().cuda.current_stream().cuda_stream


@pytest.fixture(scope="module")
def refs():
    """map over a pool of spawned worker processes (no CUDA in them), shut down with the module"""
    ex = ProcessPoolExecutor(max_workers=max(1, min(16, (os.cpu_count() or 2) - 1)), mp_context=multiprocessing.get_context("spawn"))
    try:
        yield ex.map
    finally:
        ex.shutdown(cancel_futures=True)


# ---- A ----
def _invert(c):
    torch = _torch()
    w = S.fr(c).limbs

    def run(A, in_place):
        d_a = _dev(A)
        d_out = d_a if in_place else torch.full_like(d_a, -1)
        rc = _lib().gmsm_fr_batch_invert_device(S.FIELD[c], d_a.data_ptr(), len(A), d_out.data_ptr(), _stream())
        assert rc == 0, _err()
        if not in_place:
            assert np.array_equal(_host(d_a, w), A), "the input was modified"
        return _host(d_out, w)

    return run


@pytest.mark.parametrize("c", S.CURVES)
def test_batch_invert_extremes_device(c):
    S.check_batch_invert(c, _invert(c), "device", random.Random(5 + S.FIELD[c]))


# ---- B ----
def _perm_accumulate(c):
    torch = _torch()
    w = S.fr(c).limbs

    def run(T1, T2, E):
        n = len(T1)
        d_t1, d_t2 = _dev(T1), _dev(T2)
        ws = int(_lib().gmsm_fr_permutation_workspace_bytes(S.FIELD[c], n))
        work = torch.empty(max(ws // 8, 1), dtype=torch.int64, device="cuda")
        d_z = torch.full((n * w,), -1, dtype=torch.int64, device="cuda")
        e = np.ascontiguousarray(E[0], dtype=np.uint64)
        rc = _lib().gmsm_fr_permutation_accumulate_device(S.FIELD[c], d_t1.data_ptr(), d_t2.data_ptr(), n, e.ctypes.data, d_z.data_ptr(),
                                                          work.data_ptr(), _stream())
        assert rc == 0, _err()
        return _host(d_z, w)

    return run


B_SIZES = [(c, 21) for c in S.CURVES[:5]] + [("bn254", 22), ("bw6633", 21), ("bw6761", 19), ("bw6761", 20)]


@pytest.mark.parametrize("c,logn", B_SIZES)
def test_perm_accumulate_three_levels_device(c, logn, refs):
    """random t1, t2 (pools of 64 values plus unique values at the level positions); the forced eps cases at the smaller size of
    each field"""
    t = S.scan_tile(c)
    n = 1 << logn
    assert n > t * t
    forced = (c, logn - 1) not in B_SIZES
    S.check_perm_accumulate(c, n, t, _perm_accumulate(c), "device", 1000 * logn + S.FIELD[c], refs, forced=forced)


@pytest.mark.parametrize("c", S.CURVES)
def test_perm_accumulate_eps_extremes_device(c):
    S.check_perm_accumulate(c, 1 << 12, S.scan_tile(c), _perm_accumulate(c), "device", 77 + S.FIELD[c], forced=False,
                            eps_extremes=S.extremes(c))


# ---- C ----
def _plookup_accumulate(c):
    torch = _torch()
    w = S.fr(c).limbs

    def run(F, T, H1, H2, B, G):
        n = len(F)
        d_in = [_dev(x) for x in (F, T, H1, H2)]
        ws = int(_lib().gmsm_fr_permutation_workspace_bytes(S.FIELD[c], n))
        work = torch.empty(max(ws // 8, 1), dtype=torch.int64, device="cuda")
        d_z = torch.full((n * w,), -1, dtype=torch.int64, device="cuda")
        b, g = (np.ascontiguousarray(x[0], dtype=np.uint64) for x in (B, G))
        rc = _lib().gmsm_fr_plookup_accumulate_device(S.FIELD[c], *(d.data_ptr() for d in d_in), n, b.ctypes.data, g.ctypes.data,
                                                      d_z.data_ptr(), work.data_ptr(), _stream())
        assert rc == 0, _err()
        return _host(d_z, w)

    return run


def _c_cases():
    out = []
    for c in S.CURVES:
        t = S.scan_tile(c)
        out += [(c, t * t + 1, False), (c, t * t + t - 1, True)]
    return out + [("bn254", (1 << 22) - 1, False), ("bn254", 1 << 22, False)]


@pytest.mark.parametrize("c,n,edges", _c_cases())
def test_plookup_accumulate_levels_device(c, n, edges, refs):
    S.check_plookup_accumulate(c, n, S.scan_tile(c), _plookup_accumulate(c), "device", n + 31 * S.FIELD[c], refs, edges=edges)


# ---- D ----
def _perm_numerator(c, dom):
    torch = _torch()
    w = S.fr(c).limbs

    def run(LT1, LT2, LZ, E, O):
        d_in = [_dev(x) for x in (LT1, LT2, LZ)]
        d_out = torch.full_like(d_in[0], -1)
        e, o = (np.ascontiguousarray(x[0], dtype=np.uint64) for x in (E, O))
        rc = _lib().gmsm_fft_permutation_numerator_device(dom._h, *(d.data_ptr() for d in d_in), len(LT1), e.ctypes.data, o.ctypes.data,
                                                          d_out.data_ptr(), _stream())
        assert rc == 0, _err()
        return _host(d_out, w)

    return run


def _plookup_numerator(c, dom):
    torch = _torch()
    w = S.fr(c).limbs

    def run(LZ, LH1, LH2, LT, LF, B, G, A):
        d_in = [_dev(x) for x in (LZ, LH1, LH2, LT, LF)]
        d_out = torch.full_like(d_in[0], -1)
        ch = [np.ascontiguousarray(x[0], dtype=np.uint64) for x in (B, G, A)]
        rc = _lib().gmsm_fft_plookup_numerator_device(dom._h, *(d.data_ptr() for d in d_in), len(LZ), *(x.ctypes.data for x in ch),
                                                      d_out.data_ptr(), _stream())
        assert rc == 0, _err()
        return _host(d_out, w)

    return run


def _d_cases():
    out = []
    for c in S.CURVES:
        a = S.two_adicity(c)
        out += [("permutation", c, lg) for lg in (20, 22) if lg <= a and not (c == "bw6633" and lg > 20)]
        out += [("plookup", c, lg) for lg in (21, 23) if lg <= a] + ([("plookup", c, 20)] if a < 21 else [])
    return out


@pytest.mark.parametrize("which,c,logn", _d_cases())
def test_numerator_positions_large(which, c, logn):
    n = 1 << logn
    dom = _fft().NewDomain(c, n)
    rng = random.Random(logn * 13 + S.FIELD[c])
    try:
        if which == "permutation":
            S.check_perm_numerator(c, n, _perm_numerator(c, dom), "device", rng)
        else:
            S.check_plookup_numerator(c, n, _plookup_numerator(c, dom), "device", rng)
    finally:
        dom.close()


@pytest.mark.parametrize("c", S.CURVES)
def test_numerator_challenge_extremes_device(c):
    n = 1 << 10
    dom = _fft().NewDomain(c, n)
    rng = random.Random(99 + S.FIELD[c])
    try:
        S.check_perm_numerator(c, n, _perm_numerator(c, dom), "device", rng, sweep=True)
        S.check_plookup_numerator(c, n, _plookup_numerator(c, dom), "device", rng, sweep=True)
    finally:
        dom.close()


# ---- E ----
def _sort(c):
    torch = _torch()
    w = S.fr(c).limbs

    def run(A, in_place):
        n = len(A)
        d_in = _dev(A)
        d_out = d_in if in_place else torch.full_like(d_in, -1)
        work = torch.empty(int(_lib().gmsm_fr_sort_workspace_bytes(S.FIELD[c], n)) // 8 + 1, dtype=torch.int64, device="cuda")
        rc = _lib().gmsm_fr_sort_device(S.FIELD[c], d_in.data_ptr(), n, d_out.data_ptr(), work.data_ptr(), _stream())
        assert rc == 0, _err()
        if not in_place:
            assert np.array_equal(_host(d_in, w), A), "the input was modified"
        return _host(d_out, w)

    return run


E_CASES = [(c, n) for c in S.CURVES for n in (31, 32, 33, 4095, 4096, 4097, (1 << 21) + 1)] + [
    (c, (1 << 23) - 1) for c in ("bn254", "bw6761")]


@pytest.mark.parametrize("c,n", E_CASES)
def test_sort_adversarial_device(c, n):
    S.check_sort(c, n, _sort(c), "device", n + 17 * S.FIELD[c], brief=n > (1 << 22))
