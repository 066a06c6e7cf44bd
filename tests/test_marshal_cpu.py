"""Point (de)serialisation kernels (csrc/marshal_kernels.cuh) on the CPU through the kernel emulation of tests/emu
(tests/emu/emu_marshal.cpp): k_g2_decode for the G2 groups over Fp2, k_g1_decode with the twist's b for the bw6 G2 groups, and
k_points_encode for all twelve G1 and G2 groups of the pairing curves, compared byte- and limb-exact with the big-int
restatement of tests/marshal_ref.py.  Also the bls12-381 deserialization_G2 vectors and the refusals of the Python layer that
need no library.  CPU only; the emulation library is a test artefact (build/libgmsm_emu_marshal.so), never part of libgmsm.so."""
import ctypes
import importlib
import io
import json
import os
import random
import struct
import subprocess

import numpy as np
import pytest

from tests import marshal_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "gnark-crypto_b200", "csrc")
EMU = os.path.join(ROOT, "tests", "emu")
OUT = os.path.join(ROOT, "gnark-crypto_b200", "build", "libgmsm_emu_marshal.so")
GOLDEN = os.path.join(ROOT, "tests", "golden", "bls12381_deserialization_g2.json")
_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        bdir = os.path.dirname(OUT)
        os.makedirs(bdir, exist_ok=True)
        deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))] + [
            os.path.join(EMU, f) for f in os.listdir(EMU)] + [os.path.join(ROOT, "include", "gmsm.h")]
        if not os.path.exists(OUT) or os.path.getmtime(OUT) < max(os.path.getmtime(d) for d in deps):
            obj = os.path.join(bdir, "marshal_emu_marshal.o")
            # tests/emu FIRST: its cuda_runtime.h stands in for the real one
            subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-I", EMU, "-I", CSRC, "-c", os.path.join(EMU, "emu_marshal.cpp"), "-o", obj],
                           check=True)
            subprocess.run(["g++", "-shared", "-o", OUT, obj], check=True)
        _LIB = ctypes.CDLL(OUT)
    return _LIB


def emu_decode(G: R.Group, data: bytes, n: int, raw: bool, check: bool = True):
    """one emulated decode launch -> (rows, first error (index, code) or None)"""
    buf = np.frombuffer(data, dtype=np.uint8).copy() if data else np.zeros(1, dtype=np.uint8)
    out = np.zeros((n, G.words), dtype=np.uint64)
    err = ctypes.c_ulonglong(0)
    if G.name.endswith("_g1"):
        from tests.test_emu_fft_decode_more_curves import _lib as g1_lib
        rc = g1_lib().emu_g1_decode_run(G.id, buf.ctypes.data_as(ctypes.c_void_p), ctypes.c_uint32(n), int(raw), int(check),
                                        out.ctypes.data_as(ctypes.c_void_p), ctypes.byref(err))
    else:
        rc = _lib().emu_g2_decode_run(G.id, buf.ctypes.data_as(ctypes.c_void_p), ctypes.c_uint32(n), int(raw), int(check),
                                      out.ctypes.data_as(ctypes.c_void_p), ctypes.byref(err))
    assert rc == 0
    e = err.value
    return out, (None if e == (1 << 64) - 1 else (e >> 8, e & 0xFF))


def emu_encode(G: R.Group, rows: np.ndarray, raw: bool) -> bytes:
    rows = np.ascontiguousarray(rows, dtype=np.uint64).reshape(-1, G.words)
    n = rows.shape[0]
    size = (2 if raw else 1) * G.comp_bytes()
    out = np.zeros(max(n * size, 4), dtype=np.uint8)
    assert _lib().emu_points_encode_run(G.id, rows.ctypes.data_as(ctypes.c_void_p), ctypes.c_uint32(n), int(raw),
                                        out.ctypes.data_as(ctypes.c_void_p)) == 0
    return out[:n * size].tobytes()


def _check_case(G, c):
    got, first = emu_decode(G, c.data, c.n, c.raw, c.check)
    want, wfirst = G.decode_stream(c.data, c.n, c.raw, c.check)
    assert first == wfirst, (G.name, c.title, first, wfirst)
    for i in range(c.n):
        assert np.array_equal(got[i], want[i]), (G.name, c.title, i)


@pytest.mark.parametrize("name", R.G2_GROUPS)
def test_reference_matches_kzg_on_fp_groups_and_curve(name):
    """the restatement's codec: its Bytes / RawBytes equal kzg's G1 codec on Fp (bw6 G2 uses the same field and flags, with the
    twist's b), random points are on the curve, and b' is the twist's (the oracle's G2 generator lies on it)"""
    G = R.group(name)
    rng = random.Random(3)
    pts = G.random_points(6, rng) + [None]
    assert all(G.on_curve(*p) for p in pts if p)
    O = importlib.import_module("oracle.oracle")
    gen = O.GROUPS[name].gen
    gx, gy = gen[0], gen[1]
    tup = (lambda v: (v,)) if G.D == 1 else (lambda v: (v[0], v[1]) if isinstance(v, (tuple, list)) else (v.a0, v.a1))
    assert G.on_curve(tup(gx), tup(gy)), name
    if G.D == 1:
        K = R.kzg()
        c = name.split("_")[0]
        for p in pts:
            assert G.bytes_(p) == K.g1_bytes(G.row(p), c)
            assert G.raw_bytes(p) == K.g1_raw_bytes(G.row(p), c)
            assert G.set_bytes(G.raw_bytes(p), True)[0] == p


@pytest.mark.parametrize("name", R.G2_GROUPS)
def test_g2_decode_families_emulated(name):
    """every family of marshal_ref.decode_cases through the emulated decoder: rows limb for limb and the first error"""
    G = R.group(name)
    cases = R.decode_cases(G)
    codes = set()
    for c in cases:
        _check_case(G, c)
        codes.add((G.decode_stream(c.data, c.n, c.raw, c.check)[1] or (0, 0))[1])
    assert codes == {0, R.BAD_INFINITY, R.BAD_ELEMENT, R.NO_SQRT, R.BAD_FLAGS}, codes
    # not on the curve: Y + 1 in a raw stream, rejected with the check and taken as given without it
    rng = random.Random(5)
    p = G.random_points(3, rng)
    bad = (p[1][0], G.add(p[1][1], G.one()))
    data = G.encode([p[0], bad, p[2]], True)
    for check in (True, False):
        _check_case(G, R.Case("not on curve check=%d" % check, data, 3, True, check))
    assert emu_decode(G, data, 3, True)[1] == (1, R.NOT_ON_CURVE)


def test_bls12377_square_root_depths_emulated():
    """bls12-377 (q = 1 mod 4, 2-adicity 46): compressed G2 points whose norm takes the shallowest and the deepest
    Tonelli-Shanks rounds decode to the reference's points, with both signs"""
    G = R.group("bls12377_g2")
    assert G.two_adicity == 46
    pts = R.depth_points(G, random.Random(11))
    assert set(pts) == {0, 45}
    allp = [q for d in pts for p in pts[d] for q in (p, (p[0], G.neg(p[1])))]
    data = G.encode(allp, False)
    got, first = emu_decode(G, data, len(allp), False)
    assert first is None
    for i, p in enumerate(allp):
        assert np.array_equal(got[i], G.row(p)), i


@pytest.mark.parametrize("name", R.ALL_GROUPS)
def test_encode_emulated(name):
    """k_points_encode against the reference's Bytes / RawBytes on 3 blocks (a partial last one): every family, both kinds"""
    G = R.group(name)
    rng = random.Random(17)
    base = R.encode_points(G, rng)
    pts = [base[i % len(base)] if i % 7 else (None if i % 2 else base[i % len(base)]) for i in range(300)]
    rows = np.stack([G.row(p) for p in pts])
    for raw in (False, True):
        got = emu_encode(G, rows, raw)
        want = R.encode_ref(G, pts, raw)
        size = len(want) // len(pts)
        for i in range(len(pts)):
            assert got[i * size:(i + 1) * size] == want[i * size:(i + 1) * size], (name, raw, i, pts[i])


@pytest.mark.parametrize("name", R.ALL_GROUPS)
def test_round_trips_emulated(name):
    """decode(encode(P)) = P and encode(decode(b)) = b, both kinds, through the emulated kernels"""
    G = R.group(name)
    rng = random.Random(23)
    pts = G.random_points(40, rng) + [None, None]
    if G.D == 2:
        pts.append(G.point_with_y((rng.randrange(1, G.q), 0)) or None)
    rows = np.stack([G.row(p) for p in pts])
    for raw in (False, True):
        b = emu_encode(G, rows, raw)
        back, first = emu_decode(G, b, len(pts), raw)
        assert first is None and np.array_equal(back, rows), (name, raw)
        assert emu_encode(G, back, raw) == b


def _golden():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.mark.parametrize("vec", _golden(), ids=lambda v: v["name"])
def test_bls12381_deserialization_g2_vectors(vec):
    """bls12-381 deserialization_G2 (the reference's testing/bls vectors, as JSON): each one read as G2Affine.setBytes reads a
    buffer -- the kind from the flags, io.ErrShortBuffer below its size, extra bytes ignored -- and decoded through the emulated
    kernel.  The outcome is the reference's under NoSubgroupChecks, which differs from its SetBytes where only the subgroup check
    rejects: fails_not_in_G2 holds a point on the curve outside the subgroup, so it decodes here, and so does
    fails_too_many_bytes, which is the same 96 bytes followed by one more (setBytes reads a point's size and ignores the rest)."""
    G = R.group("bls12381_g2")
    data = bytes.fromhex(vec["signature"])
    valid = vec["output"] is not None or vec["name"] in ("deserialization_fails_not_in_G2", "deserialization_fails_too_many_bytes")
    f = G.flags
    m = data[0] & f["mask"] if data else None
    raw = m in (f["unc"], f["unc_inf"])
    size = (2 if raw else 1) * G.comp_bytes()
    if len(data) < G.comp_bytes() or len(data) < size:
        ok = False                                              # io.ErrShortBuffer
    else:
        _, first = emu_decode(G, data[:size], 1, raw, check=False)
        ref = G.set_bytes(data[:size], raw, check=False)[1]
        assert (first is None) == (ref == R.OK), vec["name"]
        ok = first is None
    assert ok == valid, vec["name"]


def test_python_refusals_without_library():
    """the G2 functions refuse bls24-315 / bls24-317 (G2 over Fp4) with ValueError before any library call; slices read their
    kind from the first point's flags, refuse a short stream, and refuse a raw-first mixed stream as "invalid point encoding"
    """
    K = R.kzg()
    for c in ("bls24315", "bls24317"):
        with pytest.raises(ValueError):
            K.decode_g2_points(c, b"", 0)
        with pytest.raises(ValueError):
            K.encode_g2_points(c, np.zeros((0, 20), dtype=np.uint64))
    with pytest.raises(ValueError):
        K.encode_g1_points("secp256k1", np.zeros((0, 8), dtype=np.uint64))
    with pytest.raises(EOFError):
        K.read_points(io.BytesIO(struct.pack(">I", 2) + b"\x80" * 40), "bn254_g1")
    pts = K.read_points(io.BytesIO(struct.pack(">I", 0)), "bn254_g2")
    assert pts.shape == (0, 16)
    # a raw point followed by compressed ones: short of three raw strides, refused at the first compressed point
    G = R.group("bls12381_g1")
    p = G.random_points(3, random.Random(4))
    mixed = struct.pack(">I", 3) + G.encode(p[:1], True) + G.encode(p[1:], False)
    with pytest.raises(K.MultiExpError, match="point 1: invalid point encoding"):
        K.read_points(io.BytesIO(mixed), "bls12381_g1")
