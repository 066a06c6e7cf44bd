"""The per-curve table of the KZG prover (kzg.CURVE_PARAMS) and the host point codec for bls24-315, bls24-317, bw6-633 and
bw6-761: sizes agree with the MSM engine and the moduli, b puts the oracle's generator on the curve, G1Affine.Bytes /
RawBytes / SetBytes round-trip oracle points, and the Fiat-Shamir transcript of deriveGamma binds fr.Bytes-long scalars and
2 x fp.Bytes-long digests (kzg.go:531-563).  CPU only."""
import hashlib
import importlib

import numpy as np
import pytest

from oracle import oracle as O

curves = importlib.import_module("gnark-crypto_b200.curves")

ALL = ["bn254", "bls12381", "bls12377", "bls24315", "bls24317", "bw6633", "bw6761"]
NEW = ["bls24315", "bls24317", "bw6633", "bw6761"]
# (fr.Limbs, fp.Limbs, q mod 4) as the reference states them (fr|fp/element.go:41)
SIZES = {"bn254": (4, 4, 3), "bls12381": (4, 6, 3), "bls12377": (4, 6, 1), "bls24315": (4, 5, 1), "bls24317": (4, 5, 3),
         "bw6633": (5, 10, 1), "bw6761": (6, 12, 3)}


def _kzg():
    return importlib.import_module("gnark-crypto_b200.kzg")


@pytest.mark.parametrize("c", ALL)
def test_curve_table(c):
    kzg = _kzg()
    cp = kzg.CURVE_PARAMS[c]
    G = O.GROUPS[c + "_g1"]
    fr_words, fp_words, qmod4 = SIZES[c]
    assert (cp.fr_words, cp.fp_words, cp.q % 4) == (fr_words, fp_words, qmod4)
    assert (cp.fr_bytes, cp.fp_bytes) == (8 * fr_words, 8 * fp_words)
    assert cp.r == G.fr.q and cp.q == G.K.q and cp.b == G.b % cp.q
    assert curves._limbs(cp.r) == cp.fr_words and curves._limbs(cp.q) == cp.fp_words
    g1 = curves.GROUPS[c + "_g1"]
    assert g1.scalar_words == cp.fr_words and g1.words == cp.fp_words
    x, y = G.gen
    assert (x ** 3 + cp.b - y * y) % cp.q == 0                   # the generator is on y^2 = x^3 + b
    assert cp.flags["mask"] == (0b11 << 6 if c == "bn254" else 0b111 << 5)
    # the scalar codec sizes itself from r
    vals = [0, 1, cp.r - 1, 123456789]
    enc = curves._fr_encode(vals, cp.r)
    assert enc.shape == (4, cp.fr_words) and np.array_equal(enc, G.encode_scalars(vals)) and curves._fr_decode(enc, cp.r) == vals


def test_group_table_matches_library_and_oracle():
    """the one curve table against the library's layout queries and the oracle (pure host calls): every group's affine point and
    scalar sizes and its scalar bits, every pairing curve's GMSM_FR_* element size"""
    L = importlib.import_module("gnark-crypto_b200._native").lib()
    assert sorted(g.id for g in curves.GROUPS.values()) == list(range(13))
    for name, g in curves.GROUPS.items():
        assert L.gmsm_affine_bytes(g.id) == 16 * g.words, name
        assert L.gmsm_scalar_bytes(g.id) == 8 * g.scalar_words, name
        assert g.scalar_bits == O.GROUPS[name].fr.bits, name
    assert sorted(cp.fr_id for cp in curves.CURVE_PARAMS.values()) == list(range(7))
    for c, cp in curves.CURVE_PARAMS.items():
        assert L.gmsm_fft_fr_bytes(cp.fr_id) == cp.fr_bytes, c


def test_bw6761_b_is_minus_one():
    cp = _kzg().CURVE_PARAMS["bw6761"]
    assert cp.b == cp.q - 1


@pytest.mark.parametrize("c", NEW)
def test_point_codec_roundtrip(c):
    """G1Affine.Bytes / RawBytes / SetBytes (marshal.go:801-950) on the host against the oracle's points, both signs of y,
    infinity in both forms, and the reference's error cases"""
    kzg = _kzg()
    G = O.GROUPS[c + "_g1"]
    cp = kzg.CURVE_PARAMS[c]
    f = cp.flags
    seen = set()
    for m in range(1, 25):
        P = G.encode_affine([G.scalar_mul(G.gen, m * 7919)])[0]
        cb, rb = kzg.g1_bytes(P, c), kzg.g1_raw_bytes(P, c)
        assert len(cb) == cp.fp_bytes and len(rb) == 2 * cp.fp_bytes
        seen.add(cb[0] & f["mask"])
        for b in (cb, rb):
            q, used = kzg.g1_set_bytes(b + b"trailing", c)
            assert np.array_equal(q, P) and used == len(b)
        x, y = G.decode_affine(P.reshape(1, -1))[0]
        assert int.from_bytes(rb[: cp.fp_bytes], "big") == int(x) and int.from_bytes(rb[cp.fp_bytes:], "big") == int(y)
    assert seen == {f["small"], f["large"]}
    z = np.zeros(2 * cp.fp_words, dtype=np.uint64)
    assert kzg.g1_bytes(z, c)[0] == f["inf"] and not any(kzg.g1_bytes(z, c)[1:])
    assert kzg.g1_raw_bytes(z, c)[0] == f["unc_inf"] and not any(kzg.g1_raw_bytes(z, c)[1:])
    for b in (kzg.g1_bytes(z, c), kzg.g1_raw_bytes(z, c)):
        q, used = kzg.g1_set_bytes(b, c)
        assert not q.any() and used == len(b)
    bad = bytearray(kzg.g1_bytes(z, c))
    bad[-1] = 1
    with pytest.raises(ValueError, match="invalid infinity point encoding"):
        kzg.g1_set_bytes(bytes(bad), c)
    with pytest.raises(ValueError, match="invalid fp.Element encoding"):
        kzg.g1_set_bytes(bytes([f["small"] | (~f["mask"] & 0xFF)] + [0xFF] * (cp.fp_bytes - 1)), c)
    x = 1
    while pow((x ** 3 + cp.b) % cp.q, (cp.q - 1) // 2, cp.q) != cp.q - 1:
        x += 1
    xb = bytearray(x.to_bytes(cp.fp_bytes, "big"))
    xb[0] |= f["small"]
    with pytest.raises(ValueError, match="square root doesn't exist"):
        kzg.g1_set_bytes(bytes(xb), c)


class _Recorder:
    """a hash object that records the chunks written to it (the transcript's byte layout), digesting like sha256"""

    def __init__(self):
        self.chunks = []
        self._h = hashlib.sha256()

    def update(self, b):
        self.chunks.append(bytes(b))
        self._h.update(b)

    def digest(self):
        return self._h.digest()


@pytest.mark.parametrize("c", ALL)
def test_derive_gamma_byte_lengths(c):
    """deriveGamma writes "gamma", the point (fr.Bytes), every digest (RawBytes: 2 x fp.Bytes), every claimed value (fr.Bytes)
    and the extra data; gamma is the digest read big-endian mod r"""
    kzg = _kzg()
    G = O.GROUPS[c + "_g1"]
    cp = kzg.CURVE_PARAMS[c]
    r = cp.r
    digests = [G.encode_affine([G.scalar_mul(G.gen, k)])[0] for k in (5, 9)]
    point = G.encode_scalars([r - 2])[0]
    vals = G.encode_scalars([42, r - 1])
    rec = []
    gamma = kzg.derive_gamma(point, digests, vals, lambda: rec.append(_Recorder()) or rec[-1], c, b"xyz")
    chunks = rec[0].chunks
    assert [len(x) for x in chunks] == [5, cp.fr_bytes, 2 * cp.fp_bytes, 2 * cp.fp_bytes, cp.fr_bytes, cp.fr_bytes, 3]
    want = hashlib.sha256(b"gamma" + (r - 2).to_bytes(cp.fr_bytes, "big"))
    for k in (5, 9):
        x, y = G.scalar_mul(G.gen, k)
        want.update(int(x).to_bytes(cp.fp_bytes, "big") + int(y).to_bytes(cp.fp_bytes, "big"))
    want.update((42).to_bytes(cp.fr_bytes, "big") + (r - 1).to_bytes(cp.fr_bytes, "big") + b"xyz")
    assert gamma == int.from_bytes(want.digest(), "big") % r
