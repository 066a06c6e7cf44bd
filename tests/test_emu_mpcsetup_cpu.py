"""The mpcsetup kernel (mpc_kernels.cuh: out[i] = [c r^(start + i)] points[i], the ladder of lag_scalar_mul and the per-thread batch
normalisation) runs on the CPU through the kernel emulation of tests/emu (tests/emu/emu_mpcsetup.cpp) in the library's launch
schedule, for all thirteen groups, and is compared limb for limb with the big-int restatement (mpcsetup_ref).  CPU only; a test
artefact (build/libgmsm_emu_mpcsetup.so), never part of libgmsm.so."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

from oracle import oracle as O
from tests import mpcsetup_ref as MR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "gnark-crypto_b200", "csrc")
EMU = os.path.join(ROOT, "tests", "emu")
OUT = os.path.join(ROOT, "gnark-crypto_b200", "build", "libgmsm_emu_mpcsetup.so")
GROUP_IDS = {"bn254_g1": 0, "bn254_g2": 1, "bls12381_g1": 2, "bls12381_g2": 3, "bls12377_g1": 4, "bls12377_g2": 5, "secp256k1_g1": 6,
             "bw6761_g1": 7, "bw6761_g2": 8, "bls24315_g1": 9, "bls24317_g1": 10, "bw6633_g1": 11, "bw6633_g2": 12}
SCALE_M = 8   # points per thread of k_scale_powers
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
                o = os.path.join(bdir, "emu_mpcsetup_%d.o" % k)
                objs.append(o)
                # tests/emu FIRST: its cuda_runtime.h stands in for the real one
                procs.append(subprocess.Popen(["g++", "-std=c++17", "-O1", "-fPIC", "-DEMU_GROUP=%d" % k, "-I", EMU, "-I", CSRC, "-c",
                                               os.path.join(EMU, "emu_mpcsetup.cpp"), "-o", o]))
            assert all(p.wait() == 0 for p in procs)
            subprocess.run(["g++", "-shared", "-o", OUT, *objs], check=True)
        _LIB = ctypes.CDLL(OUT)
    return _LIB


def emu_scale_powers(name: str, pts: np.ndarray, c: int, r: int, start: int = 0) -> np.ndarray:
    G = O.GROUPS[name]
    pts = np.ascontiguousarray(pts, dtype=np.uint64)
    cl, rl = (np.ascontiguousarray(x) for x in G.encode_scalars([c, r]))
    out = np.zeros_like(pts)
    rc = getattr(_lib(), "emu_scale_powers_%d" % GROUP_IDS[name])(
        ctypes.c_void_p(pts.ctypes.data), ctypes.c_uint64(pts.shape[0]), ctypes.c_void_p(cl.ctypes.data), ctypes.c_void_p(rl.ctypes.data),
        ctypes.c_uint64(start), ctypes.c_void_p(out.ctypes.data))
    assert rc == 0, "rc = %d (2: the kernel wrote to the input)" % rc
    return out


def points_with_infinity(G: O.Group, n: int, seed: int) -> list:
    """n consecutive multiples of a random point, with infinity at 0, at the last index and at every 5th index from 3"""
    rng = random.Random(seed)
    pts = O.consecutive_multiples(G, n, 1, G.scalar_mul(G.gen, rng.randrange(1, G.fr.q)))
    for i in [0, n - 1] + list(range(3, n, 5)):
        pts[i] = G.aff_inf()
    return pts


def _check(name: str, pts: list, c: int, r: int, start: int = 0):
    G = O.GROUPS[name]
    q = G.fr.q
    got = emu_scale_powers(name, G.encode_affine(pts), c, r, start)
    want = G.encode_affine(MR.scale_powers(G, pts, c * pow(r, start, q) % q, r))
    bad = [i for i in range(len(pts)) if not np.array_equal(got[i], want[i])]
    assert not bad, "%s n=%d c=%d r=%d start=%d: first wrong index %d" % (name, len(pts), c, r, start, bad[0])


@pytest.mark.parametrize("name", sorted(GROUP_IDS, key=GROUP_IDS.get))
def test_emu_scale_powers_edge_scalars(name):
    """c and r through {0, 1, r - 1, random} at n = 11 (one full thread and a tail of 3), with infinity inputs"""
    G = O.GROUPS[name]
    q = G.fr.q
    rng = random.Random(GROUP_IDS[name])
    pts = points_with_infinity(G, SCALE_M + 3, 10 + GROUP_IDS[name])
    vals = [0, 1, q - 1, rng.randrange(2, q - 1)]
    for c in vals:
        for r in vals:
            _check(name, pts, c, r)


@pytest.mark.parametrize("name", sorted(GROUP_IDS, key=GROUP_IDS.get))
def test_emu_scale_powers_sizes(name):
    """n = 1, a single partial thread, and 3 blocks' worth of threads cut short at n = 203 (each a multiple of M plus a tail);
    a start index past 2^32 (the chunks of the host entry point); r = 1 (UpdateValues)"""
    G = O.GROUPS[name]
    q = G.fr.q
    rng = random.Random(100 + GROUP_IDS[name])
    c, r = rng.randrange(1, q), rng.randrange(1, q)
    P = G.scalar_mul(G.gen, rng.randrange(1, q))
    _check(name, [P], c, r)
    _check(name, [G.aff_inf()], c, r)
    _check(name, points_with_infinity(G, 5, 1), c, r)
    pts = points_with_infinity(G, 203, 2)
    _check(name, pts, c, r)
    _check(name, pts[:40], c, r, start=(1 << 33) + 12345)
    _check(name, pts[:40], c, 1)


def test_ref_update_monomials_and_linear_combinations():
    """the restatement's UpdateMonomials is geometric scaling by (r, r) from index 1, and its linear combinations of a geometric
    sequence satisfy shifted = [tau] truncated"""
    G = O.GROUPS["bn254_g1"]
    q = G.fr.q
    rng = random.Random(5)
    tau, r = rng.randrange(2, q), rng.randrange(2, q)
    A = [G.scalar_mul(G.gen, pow(tau, i, q)) for i in range(6)]
    got = MR.update_monomials(G, A, r)
    assert got[0] == A[0] and got[1:] == MR.scale_powers(G, A[1:], r, r)
    assert got == [G.scalar_mul(G.gen, pow(tau * r, i, q)) for i in range(6)]
    powers = [pow(7, i, q) for i in range(6)]
    trunc, shifted = MR.linear_combinations(G, got, powers, [6])
    assert shifted == G.scalar_mul(trunc, tau * r % q)
    with pytest.raises(IndexError):
        MR.update_monomials(G, A[:1], r)
