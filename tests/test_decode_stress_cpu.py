"""The CPU twin of tests/test_gpu_decode_stress.py: families A to E of tests/decode_stress.py at small n through the kernel
emulation of k_g1_decode (emu_g1_decode_run, the library of tests/test_emu_fft_decode_more_curves.py), compared limb for limb
with the big-int restatement of setBytes, and the reference itself checked against kzg.g1_set_bytes."""
import ctypes
import importlib
import time

import numpy as np
import pytest

from tests import decode_stress as S
from tests.test_emu_fft_decode_more_curves import _lib


def emu_decode(s: S.Stream):
    """one emulated launch over the stream's bytes (tail included: bytes past the last point) -> (rows, first error)"""
    c = S.curve(s.curve)
    data = s.data()
    buf = np.frombuffer(data, dtype=np.uint8).copy() if data else np.zeros(1, dtype=np.uint8)
    out = np.zeros((s.n, c.words), dtype=np.uint64)
    err = ctypes.c_ulonglong(0)
    assert _lib().emu_g1_decode_run(S.GID[s.curve], buf.ctypes.data_as(ctypes.c_void_p), ctypes.c_uint32(s.n), int(s.raw),
                                    int(s.check), out.ctypes.data_as(ctypes.c_void_p), ctypes.byref(err)) == 0
    e = err.value
    return out, (None if e == (1 << 64) - 1 else (e >> 8, e & 0xFF))


@pytest.fixture(scope="module")
def fams():
    return {}


def _families(cache, name):
    if name not in cache:
        cache[name] = S.families(name)
    return cache[name]


@pytest.mark.parametrize("name", S.CURVES)
def test_reference_and_generators(name, fams):
    """every accepted point of the families equals kzg.g1_set_bytes on it, and every rejected one is rejected there with the same
    message; A reaches every square-root depth, B every limb, and D holds the cases of the other kind's infinity flag"""
    kzg = importlib.import_module("gnark-crypto_b200.kzg")
    c = S.curve(name)
    msgs = {S.BAD_INFINITY: "invalid infinity point encoding", S.BAD_ELEMENT: "invalid fp.Element encoding",
            S.NO_SQRT: "invalid compressed coordinate: square root doesn't exist", S.BAD_FLAGS: "invalid point encoding"}
    fam = _families(fams, name)
    for letter, streams in fam.items():
        for s in streams:
            rows, _, codes = s.expected()
            for i, (e, k) in enumerate(zip(s.points, codes)):
                # a pattern outside its kind's row of the table is rejected by the homogeneous rule before setBytes is asked
                if S.FLAGS[c.nflag][s.raw].get((e[0] & c.mask) >> c.shift) is None:
                    assert k == S.BAD_FLAGS, (s.title(), i, s.labels[i])
                    continue
                if k == S.NOT_ON_CURVE or (s.raw and not s.check):
                    continue
                try:
                    want = kzg.g1_set_bytes(e, name)[0]
                except ValueError as ex:
                    assert k != S.OK and str(ex) == msgs[k], (s.title(), i, s.labels[i], str(ex), k)
                    continue
                assert k == S.OK and np.array_equal(rows[i], want), (s.title(), i, s.labels[i])
    depths = sorted({int(lab.split()[1]) for s in fam["A"] for lab in s.labels if lab.startswith("depth")})
    assert depths == list(range(c.s)), (name, depths)
    assert any(S.NO_SQRT in s.expected()[2] for s in fam["A"])
    # the highest 32-bit limb where y differs from h = (q + 1)/2 is where lexicographically_largest decides: every limb, both ways
    hl = S.limbs32((c.q + 1) // 2, c)
    decided = set()
    for _, _, y in S.sign_points(name):
        yl = S.limbs32(y, c)
        j = max(j for j in range(c.limbs32) if yl[j] != hl[j])
        decided.add((j, yl[j] > hl[j]))
    assert {j for j, _ in decided} == set(range(c.limbs32)), (name, decided)
    assert len(decided) >= 2 * c.limbs32 - 1, (name, decided)
    cases = {s.case for s in fam["D"]}
    assert any("at the last index" in x for x in cases) and any("before a zero point" in x for x in cases)


@pytest.mark.parametrize("letter", ["A", "B", "C", "D", "E"])
@pytest.mark.parametrize("name", S.CURVES)
def test_decode_families_emulated(name, letter, fams):
    """family `letter` of one curve through the emulated k_g1_decode: every row limb for limb and the first error"""
    t0 = time.perf_counter()
    streams = _families(fams, name)[letter]
    assert streams
    for s in streams:
        S.compare(s, *emu_decode(s))
    print("%s %s: %d streams, %d points, %.1f s" % (name, letter, len(streams), sum(s.n for s in streams), time.perf_counter() - t0))
