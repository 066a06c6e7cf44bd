"""The Fr FFT kernels (fft_kernels.cuh, through tests/emu/emu_fft_more.cpp) for the scalar fields of bls24-315, bls24-317, bw6-633 and bw6-761, and the G1
decoding kernel (decode_kernels.cuh) for the seven pairing curves, run on the CPU through the kernel emulation of tests/emu
(one emulated thread at a time; the FFT tile kernel under the cooperative launcher) and compared with the oracle.  CPU only;
a test artefact (build/libgmsm_emu_fft_decode.so), never part of libgmsm.so."""
import ctypes
import importlib
import os
import random
import subprocess

import numpy as np
import pytest

from oracle import cref
from oracle import oracle as O
from tests import fft_more_fields as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "gnark-crypto_b200", "csrc")
EMU = os.path.join(ROOT, "tests", "emu")
OUT = os.path.join(ROOT, "gnark-crypto_b200", "build", "libgmsm_emu_fft_decode.so")
FR_IDS = {"bn254_fr": 0, "bls12381_fr": 1, "bls12377_fr": 2, "bls24315_fr": 3, "bls24317_fr": 4, "bw6633_fr": 5, "bw6761_fr": 6}
NEW_FR = ["bls24315_fr", "bls24317_fr", "bw6633_fr", "bw6761_fr"]
# G1 groups of the pairing curves: (kzg curve name, gmsm_curve_t id)
G1 = {"bn254_g1": ("bn254", 0), "bls12381_g1": ("bls12381", 2), "bls12377_g1": ("bls12377", 4), "bls24315_g1": ("bls24315", 9),
      "bls24317_g1": ("bls24317", 10), "bw6633_g1": ("bw6633", 11), "bw6761_g1": ("bw6761", 7)}
DEC_BAD_INFINITY, DEC_BAD_ELEMENT, DEC_NO_SQRT, DEC_NOT_ON_CURVE, DEC_BAD_FLAGS = 1, 2, 3, 4, 5
_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        bdir = os.path.dirname(OUT)
        os.makedirs(bdir, exist_ok=True)
        deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))] + [
            os.path.join(EMU, f) for f in os.listdir(EMU)] + [os.path.join(ROOT, "include", "gmsm.h")]
        if not os.path.exists(OUT) or os.path.getmtime(OUT) < max(os.path.getmtime(d) for d in deps):
            objs, procs = [], []
            for src in ("emu_fft_more.cpp", "emu_decode.cpp"):
                o = os.path.join(bdir, "n23_" + src.replace(".cpp", ".o"))
                objs.append(o)
                # tests/emu FIRST: its cuda_runtime.h stands in for the real one
                procs.append(subprocess.Popen(["g++", "-std=c++17", "-O1", "-fPIC", "-I", EMU, "-I", CSRC, "-c", os.path.join(EMU, src), "-o", o]))
            assert all(p.wait() == 0 for p in procs)
            subprocess.run(["g++", "-shared", "-o", OUT, *objs], check=True)
        _LIB = ctypes.CDLL(OUT)
    return _LIB


def _kzg():
    return importlib.import_module("gnark-crypto_b200.kzg")


# ---- Fr FFT ----
def _enc(f, xs):
    return np.array([f.to_limbs(f.to_mont(v)) for v in xs], dtype=np.uint64)


def _emu_fft(frname, vals, inverse, decimation, coset, shift=None):
    f = O.FIELDS[frname]
    n = len(vals)
    od = M.FFTDomain(frname, n, shift=shift)
    a = _enc(f, vals)
    consts = _enc(f, [od.generator, od.generator_inv, od.cardinality_inv, od.shift, od.shift_inv])
    rc = _lib().emu_fft_more_run(FR_IDS[frname], a.ctypes.data_as(ctypes.c_void_p), ctypes.c_uint64(n), n.bit_length() - 1, int(inverse),
                            int(decimation), int(coset), consts.ctypes.data_as(ctypes.c_void_p))
    assert rc == 0
    return [f.from_mont(O.Field.from_limbs([int(x) for x in r])) for r in a], od


@pytest.mark.parametrize("frname", NEW_FR)
@pytest.mark.parametrize("logn", [0, 1, 5, 10, 11, 12])
def test_emulated_fft_kernels_new_fields(frname, logn):
    """Domain.FFT / FFTInverse, both decimations, plain and on the coset, below, at and above the 2^10 shared-memory tile"""
    f = O.FIELDS[frname]
    n = 1 << logn
    rng = random.Random(200 + logn)
    vals = [rng.randrange(f.q) for _ in range(n)]
    cases = [(dec, coset) for dec in (O.DIT, O.DIF) for coset in (False, True)]
    if logn >= 11:
        cases = [(O.DIT, True), (O.DIF, False)]     # keep the big sizes cheap: still both decimations, the coset and the inverse
    for dec, coset in cases:
        got, od = _emu_fft(frname, vals, False, dec, coset)
        assert got == od.fft(vals, dec, coset), (dec, coset)
        got, od = _emu_fft(frname, vals, True, dec, coset)
        assert got == od.fft_inverse(vals, dec, coset), (dec, coset)


@pytest.mark.parametrize("frname", ["bw6633_fr", "bw6761_fr"])
def test_emulated_fft_custom_shift_wide_limbs(frname):
    """WithShift with a shift that fills all 5 / 6 limbs"""
    f = O.FIELDS[frname]
    n = 256
    shift = (f.q - 1) // 3 + 12345                      # > 2^256: every limb of the element is used
    assert shift.bit_length() > 256
    vals = [(7 * i * i + 3) % f.q for i in range(n)]
    for inverse, dec in ((False, O.DIF), (False, O.DIT), (True, O.DIF)):
        got, od = _emu_fft(frname, vals, inverse, dec, True, shift=shift)
        want = od.fft_inverse(vals, dec, True) if inverse else od.fft(vals, dec, True)
        assert got == want, (inverse, dec)


# ---- G1 decoding ----
def _emu_decode(gid, data, n, raw, check=True, words=None):
    out = np.zeros((n, words), dtype=np.uint64)
    err = ctypes.c_ulonglong(0)
    buf = np.frombuffer(data, dtype=np.uint8).copy() if data else np.zeros(1, dtype=np.uint8)
    rc = _lib().emu_g1_decode_run(gid, buf.ctypes.data_as(ctypes.c_void_p), ctypes.c_uint32(n), int(raw), int(check),
                                  out.ctypes.data_as(ctypes.c_void_p), ctypes.byref(err))
    assert rc == 0
    e = err.value
    return out, (None if e == (1 << 64) - 1 else (e >> 8, e & 0xFF))


def _non_residue_x(c, start=1):
    """smallest x >= start with x^3 + b a non-residue mod q: a compressed x without a point"""
    cp = _kzg().CURVE_PARAMS[c]
    x = start
    while pow((x ** 3 + cp.b) % cp.q, (cp.q - 1) // 2, cp.q) != cp.q - 1:
        x += 1
    return x


@pytest.mark.parametrize("g", list(G1))
def test_emulated_g1_decode(g):
    """k_g1_decode for every pairing G1 group: compressed and raw streams of oracle points with both signs of y and
    infinity points == the original points; then one stream per error code, with the index of the first bad point"""
    kzg = _kzg()
    c, gid = G1[g]
    G = O.GROUPS[g]
    cp = kzg.CURVE_PARAMS[c]
    n = 24
    pts = cref.generate_multiples(g, G.encode_affine([G.gen])[0], 1000003, n, nthreads=2)
    pts[4] = 0
    pts[n - 1] = 0
    words = pts.shape[1]
    comp = b"".join(kzg.g1_bytes(p, c) for p in pts)
    raw = b"".join(kzg.g1_raw_bytes(p, c) for p in pts)
    assert len(comp) == n * cp.fp_bytes and len(raw) == 2 * n * cp.fp_bytes
    f = cp.flags
    assert {comp[i * cp.fp_bytes] & f["mask"] for i in range(n)} == {f["small"], f["large"], f["inf"]}
    got, err = _emu_decode(gid, comp, n, raw=False, words=words)
    assert err is None and np.array_equal(got, pts)
    got, err = _emu_decode(gid, raw, n, raw=True, words=words)
    assert err is None and np.array_equal(got, pts)
    nb = cp.fp_bytes
    # DEC_BAD_INFINITY: the infinity flag with a non-zero byte (point 4); a later error does not hide it
    bad = bytearray(comp)
    bad[4 * nb + 3] = 1
    bad[9 * nb] = 0x20 if f["unc_inf"] is not None else 0x00
    assert _emu_decode(gid, bytes(bad), n, raw=False, words=words)[1] == (4, DEC_BAD_INFINITY)
    # DEC_BAD_ELEMENT: x >= q (all value bits set)
    bad = bytearray(comp)
    bad[6 * nb:7 * nb] = bytes([f["small"] | (~f["mask"] & 0xFF)]) + b"\xff" * (nb - 1)
    assert _emu_decode(gid, bytes(bad), n, raw=False, words=words)[1] == (6, DEC_BAD_ELEMENT)
    bad = bytearray(raw)
    bad[(2 * 8 + 1) * nb:(2 * 8 + 2) * nb] = b"\xff" * nb             # y of point 8
    assert _emu_decode(gid, bytes(bad), n, raw=True, words=words)[1] == (8, DEC_BAD_ELEMENT)
    # DEC_NO_SQRT: an x whose x^3 + b is a non-residue
    x = _non_residue_x(c)
    bad = bytearray(comp)
    xb = bytearray(x.to_bytes(nb, "big"))
    xb[0] |= f["large"]
    bad[10 * nb:11 * nb] = xb
    assert _emu_decode(gid, bytes(bad), n, raw=False, words=words)[1] == (10, DEC_NO_SQRT)
    # DEC_NOT_ON_CURVE: y + 1 (raw, check_on_curve); without the check the point is taken as given
    bad = bytearray(raw)
    y = int.from_bytes(bad[(2 * 11 + 1) * nb:(2 * 11 + 2) * nb], "big")
    bad[(2 * 11 + 1) * nb:(2 * 11 + 2) * nb] = ((y + 1) % cp.q).to_bytes(nb, "big")
    assert _emu_decode(gid, bytes(bad), n, raw=True, words=words)[1] == (11, DEC_NOT_ON_CURVE)
    got, err = _emu_decode(gid, bytes(bad), n, raw=True, check=False, words=words)
    assert err is None and np.array_equal(np.delete(got, 11, 0), np.delete(pts, 11, 0))
    # DEC_BAD_FLAGS: a compressed point in a raw stream, and (three-bit curves) the unused pattern 001 in a compressed stream
    bad = bytearray(raw)
    bad[2 * 12 * nb] |= f["small"]
    assert _emu_decode(gid, bytes(bad), n, raw=True, words=words)[1] == (12, DEC_BAD_FLAGS)
    bad = bytearray(comp)
    bad[13 * nb] = (bad[13 * nb] & ~f["mask"] & 0xFF) | (0b001 << 5 if f["unc_inf"] is not None else f["unc"])
    assert _emu_decode(gid, bytes(bad), n, raw=False, words=words)[1] == (13, DEC_BAD_FLAGS)


def test_emulated_decode_square_root_corner_cases():
    """x^3 + b = 0 has the root 0 (bw6-761: x = 1, b = -1; y = 0 is then on the curve); curves with q = 1 mod 4 at many x
    (Tonelli-Shanks with 2-adicity 46, 20 and 2) agree with the host restatement of SetBytes"""
    kzg = _kzg()
    c, gid = G1["bw6761_g1"]
    cp = kzg.CURVE_PARAMS[c]
    xb = bytearray((1).to_bytes(cp.fp_bytes, "big"))
    xb[0] |= cp.flags["small"]
    got, err = _emu_decode(gid, bytes(xb), 1, raw=False, words=2 * cp.fp_words)
    want, _ = kzg.g1_set_bytes(bytes(xb), c)
    assert err is None and np.array_equal(got[0], want)
    for g in ("bls12377_g1", "bls24315_g1", "bw6633_g1"):
        c, gid = G1[g]
        cp = kzg.CURVE_PARAMS[c]
        assert cp.q % 4 == 1
        stream, wants = b"", []
        x = 0
        while len(wants) < 12:
            x += 1
            if pow((x ** 3 + cp.b) % cp.q, (cp.q - 1) // 2, cp.q) != 1:
                continue
            for flag in ("small", "large"):
                xb = bytearray(x.to_bytes(cp.fp_bytes, "big"))
                xb[0] |= cp.flags[flag]
                stream += bytes(xb)
                wants.append(kzg.g1_set_bytes(bytes(xb), c)[0])
        got, err = _emu_decode(gid, stream, len(wants), raw=False, words=2 * cp.fp_words)
        assert err is None and np.array_equal(got, np.stack(wants)), g
