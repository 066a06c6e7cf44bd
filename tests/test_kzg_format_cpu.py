"""unsafe.WriteSlice / ReadSlice image (utils/unsafe/dump_slice.go:16-76) -- CPU-only format checks."""
import importlib
import io
import struct

import numpy as np
import pytest

curves = importlib.import_module("gnark-crypto_b200.curves")


def test_slice_roundtrip_and_limits():
    kzg = importlib.import_module("gnark-crypto_b200.kzg")
    pts = np.arange(5 * 8, dtype=np.uint64).reshape(5, 8)
    buf = io.BytesIO()
    kzg.write_marker(buf)
    kzg.write_slice(buf, pts)
    buf.write(b"tail")
    raw = buf.getvalue()
    assert raw[:8] == struct.pack("<Q", 0xDEADBEEF) and raw[8:16] == struct.pack("<Q", 5)
    assert raw[16 : 16 + 64] == pts[0].tobytes()              # raw little-endian memory of the first element
    buf.seek(0)
    kzg.read_marker(buf)
    got = kzg.read_slice(buf, 8, max_elements=3)
    assert np.array_equal(got, pts[:3]) and buf.read() == b"tail"   # the unread elements are skipped
    buf.seek(8)
    assert np.array_equal(kzg.read_slice(buf, 8), pts)
    with pytest.raises(ValueError):
        kzg.read_marker(io.BytesIO(b"\x00" * 8))
    with pytest.raises(EOFError):
        kzg.read_slice(io.BytesIO(struct.pack("<Q", 4) + b"\x00" * 10), 8)
    e = io.BytesIO()
    kzg.write_slice(e, pts[:0])
    e.seek(0)
    assert kzg.read_slice(e, 8).shape == (0, 8)


def test_open_host_polynomial_arithmetic():
    """eval / dividePolyByXminusA (kzg.go:55-63, 567-584) as kzg.Open uses them, and the Montgomery codec"""
    import random

    kzg = importlib.import_module("gnark-crypto_b200.kzg")
    rng = random.Random(7)
    for cp in kzg.CURVE_PARAMS.values():
        r = cp.r
        f = [rng.randrange(r) for _ in range(37)]
        a = rng.randrange(r)
        fa = kzg._eval(f, a, r)
        assert fa == sum(c * pow(a, i, r) for i, c in enumerate(f)) % r
        h = kzg._divide_by_x_minus_a(f, fa, a, r)
        assert len(h) == len(f) - 1
        for x in (0, 1, rng.randrange(r)):
            assert (kzg._eval(h, x, r) * (x - a) + fa) % r == kzg._eval(f, x, r)
        enc = curves._fr_encode(f, r)
        assert curves._fr_decode(enc, r) == f
    # fr.One of bn254 in Montgomery form (ecc/bn254/fr/element.go:227)
    one = curves._fr_encode([1], kzg.CURVE_PARAMS["bn254"].r)[0]
    assert [int(x) for x in one] == [12436184717236109307, 3962172157175319849, 7381016538464732718, 1011752739694698287]


def test_point_marshal_host_restatement():
    """G1Affine.Bytes / RawBytes / SetBytes restated on the host (kzg.g1_bytes, g1_raw_bytes, g1_set_bytes; marshal.go:801-950):
    flag bits per curve family, known encodings of the generators (bn254 generator (1, 2): compressed 0x80..01, bn254.go:111),
    round trips against the oracle's points for both signs of y, infinity in both forms, the reference's error cases."""
    kzg = importlib.import_module("gnark-crypto_b200.kzg")
    from oracle import oracle as O

    G = O.GROUPS["bn254_g1"]
    gen = G.encode_affine([G.gen])[0]
    assert kzg.g1_bytes(gen, "bn254") == bytes([0x80] + [0] * 30 + [1])                       # y = 2 is the smaller root
    assert kzg.g1_raw_bytes(gen, "bn254") == bytes([0] * 31 + [1] + [0] * 31 + [2])
    neg = G.encode_affine([G.aff_neg(G.gen)])[0]
    assert kzg.g1_bytes(neg, "bn254")[0] == 0xC0                                                # -G: largest root
    for c, g in (("bn254", "bn254_g1"), ("bls12381", "bls12381_g1"), ("bls12377", "bls12377_g1")):
        G = O.GROUPS[g]
        seen = set()
        for m in range(1, 40):
            P = G.encode_affine([G.scalar_mul(G.gen, m * 7919)])[0]
            cb, rb = kzg.g1_bytes(P, c), kzg.g1_raw_bytes(P, c)
            seen.add(cb[0] & kzg.CURVE_PARAMS[c].flags["mask"])
            for b in (cb, rb):
                q, used = kzg.g1_set_bytes(b + b"trailing", c)
                assert np.array_equal(q, P) and used == len(b)
            x, y = G.decode_affine(P.reshape(1, -1))[0]
            assert int.from_bytes(rb[: len(rb) // 2], "big") == int(x) and int.from_bytes(rb[len(rb) // 2 :], "big") == int(y)
        assert seen == {kzg.CURVE_PARAMS[c].flags["small"], kzg.CURVE_PARAMS[c].flags["large"]}
        z = np.zeros_like(P)
        assert kzg.g1_bytes(z, c)[0] == kzg.CURVE_PARAMS[c].flags["inf"] and not any(kzg.g1_bytes(z, c)[1:])
        for b in (kzg.g1_bytes(z, c), kzg.g1_raw_bytes(z, c)):
            q, used = kzg.g1_set_bytes(b, c)
            assert not q.any() and used == len(b)
        bad = bytearray(kzg.g1_bytes(z, c))
        bad[-1] = 1
        with pytest.raises(ValueError, match="invalid infinity point encoding"):
            kzg.g1_set_bytes(bytes(bad), c)
        with pytest.raises(ValueError, match="invalid fp.Element encoding"):
            kzg.g1_set_bytes(bytes([kzg.CURVE_PARAMS[c].flags["small"] | (~kzg.CURVE_PARAMS[c].flags["mask"] & 0xFF)] + [0xFF] * (len(bad) - 1)), c)


def test_derive_gamma_transcript():
    """deriveGamma (kzg.go:531-563) = sha256("gamma" || point || RawBytes(digests) || claimed values || data) mod r"""
    import hashlib

    kzg = importlib.import_module("gnark-crypto_b200.kzg")
    from oracle import oracle as O

    G = O.GROUPS["bn254_g1"]
    r = G.fr.q
    d = [G.encode_affine([G.scalar_mul(G.gen, k)])[0] for k in (5, 9)]
    point = G.encode_scalars([1234567])[0]
    vals = G.encode_scalars([42, r - 1])
    h = hashlib.sha256(b"gamma" + (1234567).to_bytes(32, "big"))
    for k in (5, 9):
        x, y = G.scalar_mul(G.gen, k)
        h.update(int(x).to_bytes(32, "big") + int(y).to_bytes(32, "big"))
    h.update((42).to_bytes(32, "big") + (r - 1).to_bytes(32, "big") + b"xyz")
    assert kzg.derive_gamma(point, d, vals, hashlib.sha256, "bn254", b"xyz") == int.from_bytes(h.digest(), "big") % r
