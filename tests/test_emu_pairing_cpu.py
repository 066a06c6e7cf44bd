"""The pairing kernels (pairing_kernels.cuh: k_miller_loop, k_gt_reduce, k_gt_accumulate, k_final_exp) run on the CPU through the
kernel emulation of tests/emu (tests/emu/emu_pairing.cpp) in the library's launch order, with forced small chunks and block sizes and
shuffled block orders, and are compared limb for limb with the big-int restatement (tests/pairing_ref.py).  CPU only; a test
artefact (build/libgmsm_emu_pairing.so), never part of libgmsm.so."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

from tests import pairing_cases as PC
from tests import pairing_ref as PR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "gnark-crypto_b200", "csrc")
EMU = os.path.join(ROOT, "tests", "emu")
OUT = os.path.join(ROOT, "gnark-crypto_b200", "build", "libgmsm_emu_pairing.so")
IDS = {"bn254": 0, "bls12381": 1}
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
            for k in IDS.values():
                o = os.path.join(bdir, "emu_pairing_%d.o" % k)
                objs.append(o)
                # tests/emu FIRST: its cuda_runtime.h stands in for the real one
                procs.append(subprocess.Popen(["g++", "-std=c++17", "-O1", "-fPIC", "-DEMU_CURVE=%d" % k, "-I", EMU, "-I", CSRC, "-c",
                                               os.path.join(EMU, "emu_pairing.cpp"), "-o", o]))
            assert all(p.wait() == 0 for p in procs)
            subprocess.run(["g++", "-shared", "-o", OUT, *objs], check=True)
        _LIB = ctypes.CDLL(OUT)
    return _LIB


def emu_miller(curve, pa, qa, chunk, threads, order):
    T = PR.tower(curve)
    out = np.zeros((1, 12 * T.fp.limbs), dtype=np.uint64)
    getattr(_lib(), "emu_miller_loop_%d" % IDS[curve])(
        ctypes.c_void_p(pa.ctypes.data), ctypes.c_void_p(qa.ctypes.data), ctypes.c_uint64(pa.shape[0]), ctypes.c_uint64(chunk),
        ctypes.c_uint(threads), ctypes.c_uint(order), ctypes.c_void_p(out.ctypes.data))
    return out


def emu_final_exp(curve, z):
    z = np.ascontiguousarray(z, dtype=np.uint64)
    out = np.zeros((1, z.shape[1]), dtype=np.uint64)
    getattr(_lib(), "emu_final_exp_%d" % IDS[curve])(ctypes.c_void_p(z.ctypes.data), ctypes.c_uint64(z.shape[0]),
                                                     ctypes.c_void_p(out.ctypes.data))
    return out


@pytest.mark.parametrize("curve", sorted(IDS))
@pytest.mark.parametrize("n", [1, 2, 3, 5, 17])
def test_emu_miller_loop(curve, n):
    T = PR.tower(curve)
    P, Q = PC.random_pairs(curve, n, seed=100 + n)
    pa, qa = PC.encode_pairs(curve, P, Q)
    want = T.encode([T.miller_loop(P, Q)])
    for chunk, threads, order in [(1 << 16, 64, 0), (2, 2, 1), (3, 1, 5), (5, 4, 7)]:
        got = emu_miller(curve, pa, qa, chunk, threads, order)
        assert np.array_equal(got, want), "%s n=%d chunk=%d threads=%d order=%d" % (curve, n, chunk, threads, order)


@pytest.mark.parametrize("curve", sorted(IDS))
def test_emu_infinity_and_duplicates(curve):
    T = PR.tower(curve)
    P, Q = PC.random_pairs(curve, 4, seed=7)
    for i in range(4):
        for side in (0, 1):
            P2, Q2 = list(P), list(Q)
            if side == 0:
                P2[i] = T.G1.aff_inf()
            else:
                Q2[i] = T.G2.aff_inf()
            pa, qa = PC.encode_pairs(curve, P2, Q2)
            assert np.array_equal(emu_miller(curve, pa, qa, 3, 2, 2), T.encode([T.miller_loop(P2, Q2)]))
    pa, qa = PC.encode_pairs(curve, [T.G1.aff_inf()] * 3, Q[:3])
    assert np.array_equal(emu_miller(curve, pa, qa, 2, 1, 0), T.encode([T.one()]))
    dup_P, dup_Q = [P[0]] * 3 + [P[1]], [Q[0]] * 3 + [Q[1]]
    pa, qa = PC.encode_pairs(curve, dup_P, dup_Q)
    assert np.array_equal(emu_miller(curve, pa, qa, 2, 2, 3), T.encode([T.miller_loop(dup_P, dup_Q)]))


def test_emu_bn254_off_subgroup_g2():
    T = PR.tower("bn254")
    Q = PC.off_subgroup_g2(3, seed=11)
    P, _ = PC.random_pairs("bn254", 3, seed=12)
    pa, qa = PC.encode_pairs("bn254", P, Q)
    ml = T.miller_loop(P, Q)
    assert np.array_equal(emu_miller("bn254", pa, qa, 2, 1, 4), T.encode([ml]))
    assert np.array_equal(emu_final_exp("bn254", T.encode([ml])), T.encode([T.final_exp(ml)]))


@pytest.mark.parametrize("curve", sorted(IDS))
def test_emu_final_exp(curve):
    T = PR.tower(curve)
    rng = random.Random(3)
    cases = [[T.one()], [T.unflat([5] + [0] * 11)], [T.zero()],
             [T.unflat([rng.randrange(T.q) for _ in range(12)]) for _ in range(3)]]
    P, Q = PC.random_pairs(curve, 1, seed=4)
    cases.append([T.miller_loop(P, Q)])
    for zs in cases:
        assert np.array_equal(emu_final_exp(curve, T.encode(zs)), T.encode([T.final_exp(*zs)]))
