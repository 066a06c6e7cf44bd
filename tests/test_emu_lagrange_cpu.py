"""The kzg.ToLagrangeG1 kernels (lagrange_kernels.cuh: butterfly stages with the variable-base twiddle multiplication, bit-reversed
gather, scaling by 1/n, batch normalisation) run on the CPU through the kernel emulation of tests/emu (tests/emu/emu_lagrange.cpp)
in the library's launch order, for the G1 groups of all seven pairing curves, and compared limb for limb with the big-int
restatement of the reference (lagrange_ref).  CPU only; a test artefact (build/libgmsm_emu_lagrange.so), never part of libgmsm.so."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

from tests import lagrange_ref as LR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "gnark-crypto_b200", "csrc")
EMU = os.path.join(ROOT, "tests", "emu")
OUT = os.path.join(ROOT, "gnark-crypto_b200", "build", "libgmsm_emu_lagrange.so")
GROUP_IDS = {"bn254": 0, "bls12381": 2, "bls12377": 4, "bw6761": 7, "bls24315": 9, "bls24317": 10, "bw6633": 11}
_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        bdir = os.path.dirname(OUT)
        os.makedirs(bdir, exist_ok=True)
        deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))] + [
            os.path.join(EMU, f) for f in os.listdir(EMU)]
        if not os.path.exists(OUT) or os.path.getmtime(OUT) < max(os.path.getmtime(d) for d in deps):
            objs, procs = [], []
            for k in GROUP_IDS.values():
                o = os.path.join(bdir, "emu_lagrange_%d.o" % k)
                objs.append(o)
                # tests/emu FIRST: its cuda_runtime.h stands in for the real one
                procs.append(subprocess.Popen(["g++", "-std=c++17", "-O1", "-fPIC", "-DEMU_GROUP=%d" % k, "-I", EMU, "-I", CSRC, "-c",
                                               os.path.join(EMU, "emu_lagrange.cpp"), "-o", o]))
            assert all(p.wait() == 0 for p in procs)
            subprocess.run(["g++", "-shared", "-o", OUT, *objs], check=True)
        _LIB = ctypes.CDLL(OUT)
    return _LIB


def emu_to_lagrange(curve: str, pts: np.ndarray) -> np.ndarray:
    G = LR.group(curve)
    pts = np.ascontiguousarray(pts, dtype=np.uint64)
    n = pts.shape[0]
    w_inv, n_inv = LR.domain_inverses(curve, n)
    wl, nl = G.encode_scalars([w_inv, n_inv])
    wl, nl = np.ascontiguousarray(wl), np.ascontiguousarray(nl)
    out = np.zeros_like(pts)
    rc = getattr(_lib(), "emu_to_lagrange_%d" % GROUP_IDS[curve])(
        ctypes.c_void_p(pts.ctypes.data), ctypes.c_uint64(n), ctypes.c_void_p(wl.ctypes.data), ctypes.c_void_p(nl.ctypes.data),
        ctypes.c_void_p(out.ctypes.data))
    assert rc == 0, "rc = %d (2: the kernels wrote to the input)" % rc
    return out


def special_input(curve: str, n: int, seed: int) -> list:
    """random points (multiples of the generator) with infinity, a point equal to its first-stage partner (i, i + n/2: the doubling
    branch of the first addition) and one that is its partner's negative (cancellation), as oracle affine points"""
    G = LR.group(curve)
    r = G.fr.q
    rng = random.Random(seed)
    ks = [rng.randrange(1, r) for _ in range(n)]
    h = n // 2
    if n == 2:
        ks[1] = ks[0]                  # equal partners
    if n >= 4:
        ks[h] = 0                      # infinity
        ks[h + 1] = ks[1]              # equal partners
    if n >= 8:
        ks[h + 2] = r - ks[2]          # negatives
        ks[h - 1] = 0                  # infinity in the lower half too
    return ks


def _points_of(curve: str, ks: list) -> list:
    G = LR.group(curve)
    return [G.scalar_mul(G.gen, k) if k else G.aff_inf() for k in ks]


def _check(curve: str, pts: list):
    G = LR.group(curve)
    enc = G.encode_affine(pts)
    got = emu_to_lagrange(curve, enc)
    want = G.encode_affine(LR.to_lagrange_g1(curve, pts))
    assert np.array_equal(got, want), curve


@pytest.mark.parametrize("curve", LR.CURVES)
def test_emu_to_lagrange_special(curve):
    """n = 1, 2, 4, 8, 16 and 64 with infinity, equal and opposite first-stage partners"""
    for n in (1, 2, 4, 8, 16, 64):
        ks = special_input(curve, n, 1000 + n)
        _check(curve, _points_of(curve, ks))


@pytest.mark.parametrize("curve", LR.CURVES)
def test_emu_to_lagrange_srs_and_degenerate(curve):
    """a random SRS [tau^i]G at n = 16; n = 2 with equal points (the first butterfly doubles, the difference is infinity) and with
    opposite points (the sum cancels); all points infinity; scalar-domain reference agrees with the point-domain one"""
    G = LR.group(curve)
    r = G.fr.q
    rng = random.Random(7 + GROUP_IDS[curve])
    tau = rng.randrange(2, r)
    srs = [pow(tau, i, r) for i in range(16)]
    _check(curve, _points_of(curve, srs))
    P = G.scalar_mul(G.gen, rng.randrange(1, r))
    _check(curve, [P, P])
    _check(curve, [P, G.aff_neg(P)])
    _check(curve, [G.aff_inf()] * 8)
    want = [G.scalar_mul(G.gen, b) for b in LR.to_lagrange_scalars(curve, srs)]
    assert G.encode_affine(want).tolist() == G.encode_affine(LR.to_lagrange_g1(curve, _points_of(curve, srs))).tolist()


def test_ref_errors():
    for n in (0, 3, 6):
        with pytest.raises(LR.LagrangeError, match="len\\(coeffs\\) must be a power of 2"):
            LR.domain_inverses("bn254", n)
    with pytest.raises(LR.LagrangeError, match="m \\(2097152\\) is too big: the required root of unity does not exist"):
        LR.domain_inverses("bw6633", 1 << 21)
