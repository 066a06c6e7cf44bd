"""The counting sort of the bucket pass as the engine launches it, run on the CPU over the stand-in tests/emu/cuda_runtime.h
(tests/emu/emu_scatter_ends.cpp): K1b's last scan kernel turns the histogram into bucket END pointers (k_scan_final_ends)
and the scatter kernels take the position from them -- one returning atomicSub per entry in plain mode, end - 1 - rank in
rank mode -- with no offsets array.  Checked against a host counting sort: the offsets are the exclusive scan of the bucket
counts, every bucket's slice of `entries` holds exactly its (scalar, window) pairs with their signs, and each counter ends
at its bucket's offset in plain mode (and at its end in rank mode).  CPU only; a test artefact, never part of libgmsm.so."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from oracle import oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "gnark-crypto_b200", "csrc")
EMU = os.path.join(ROOT, "tests", "emu")
OUT = os.path.join(ROOT, "gnark-crypto_b200", "build", "libgmsm_emu_scatter_ends.so")
_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        os.makedirs(os.path.dirname(OUT), exist_ok=True)
        deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))] + [
            os.path.join(EMU, "cuda_runtime.h"), os.path.join(EMU, "emu_scatter_ends.cpp")]
        if not os.path.exists(OUT) or os.path.getmtime(OUT) < max(os.path.getmtime(d) for d in deps):
            # tests/emu FIRST: its cuda_runtime.h stands in for the real one
            subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-I", EMU, "-I", CSRC,
                            os.path.join(EMU, "emu_scatter_ends.cpp"), "-o", OUT], check=True)
        _LIB = ctypes.CDLL(OUT)
    return _LIB


def _scalars(n, kind, seed):
    """bn254 fr elements as 4 u64 Montgomery limbs (any value below r; the engine reads them as Montgomery form)"""
    rng = np.random.default_rng(seed)
    r = O.GROUPS["bn254_g1"].fr.q
    if kind == "random":
        vals = [int.from_bytes(rng.bytes(32), "little") % r for _ in range(n)]
    elif kind == "runs":                       # runs of equal scalars: hot buckets, the rank mode's case
        heads = [int(rng.integers(1, 2**62)) for _ in range(n // 16 + 1)]
        vals = [heads[i // 16] for i in range(n)]
    else:                                      # zeros and small values: empty windows
        vals = [0 if i % 3 == 0 else i % 7 for i in range(n)]
    return np.array([[(v >> (64 * k)) & (2**64 - 1) for k in range(4)] for v in vals], dtype=np.uint64)


def _sort(s, c, tables, passes, rank):
    L = _lib()
    n = s.shape[0]
    nwin = -(-254 // c)
    nb_max = nwin << c                          # a bound on nb_total + 1
    offsets = np.zeros(nb_max + 1, dtype=np.uint32)
    counters = np.zeros(nb_max + 1, dtype=np.uint32)
    entries = np.zeros(n * nwin + 16, dtype=np.uint32)
    digits = np.zeros(n * nwin + 16, dtype=np.uint32)
    nbt = ctypes.c_uint32(0)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    rc = L.emu_sort_entries(p(np.ascontiguousarray(s)), ctypes.c_size_t(n), c, tables, passes, rank, p(offsets), p(counters),
                            p(entries), p(digits), ctypes.byref(nbt))
    assert rc == 0
    nb_total = nbt.value
    return offsets[: nb_total + 1], counters[: nb_total + 1], entries, digits[: n * nwin].reshape(nwin, n), nb_total


def _bucket_of(code, j, nb, tables):
    b = (code >> 1) - 1 + (code & 1)
    return b if tables else j * nb + b


@pytest.mark.parametrize("tables", [0, 1])
@pytest.mark.parametrize("rank", [0, 1])
@pytest.mark.parametrize("kind", ["random", "runs", "small"])
def test_scatter_from_end_pointers(tables, rank, kind):
    n, c = 1500, 9
    s = _scalars(n, kind, seed=11 + 3 * tables + rank)
    offsets, counters, entries, digits, nb_total = _sort(s, c, tables, 3, rank)
    nwin = digits.shape[0]
    nb = 1 << (c - 1)
    want = {}
    for j in range(nwin):
        for i in range(n):
            code = int(digits[j, i])
            if code:
                idx = (j * n + i) if tables else i      # the table point of (i, j) has index j * row_stride + i (row_stride = n)
                want.setdefault(_bucket_of(code, j, nb, tables), []).append((idx << 1) | (code & 1))
    counts = np.zeros(nb_total + 1, dtype=np.int64)
    for b, v in want.items():
        counts[b] = len(v)
    assert np.array_equal(offsets.astype(np.int64), np.concatenate([[0], np.cumsum(counts)[:-1]]))
    for b in range(nb_total):
        got = sorted(int(x) for x in entries[offsets[b]: offsets[b + 1]])
        assert got == sorted(want.get(b, [])), (b, tables, rank, kind)
    # plain mode: every counter was taken down from its end pointer to its offset; rank mode leaves the end pointers
    end = np.concatenate([offsets[1:], [offsets[-1]]])
    assert np.array_equal(counters[:nb_total], offsets[:nb_total] if not rank else end[:nb_total])
