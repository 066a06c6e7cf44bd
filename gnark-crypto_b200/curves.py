"""The one table of the curves this package serves, and the Fr helpers the provers share.

  * GROUPS: the thirteen groups of the MultiExp engine (gmsm_curve_t of include/gmsm.h), from which CURVES and the point and
    scalar sizes derive;
  * CURVE_PARAMS: the seven pairing curves of the prover (fr/element.go and fp/element.go: moduli and Limbs; the curve's .go
    file: b; marshal.go: flags; fr/fft/domain.go: GeneratorFullMultiplicativeGroup) and their GMSM_FR_* scalar-field id;
  * the fr.Element codec (Montgomery limbs <-> integers) and the Fiat-Shamir challenge read as an fr.Element.
Nothing here touches libgmsm.so, so importing the package does not load it."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

_TWO_BIT = dict(mask=0b11 << 6, unc=0b00 << 6, unc_inf=None, small=0b10 << 6, large=0b11 << 6, inf=0b01 << 6)
_THREE_BIT = dict(mask=0b111 << 5, unc=0b000 << 5, unc_inf=0b010 << 5, small=0b100 << 5, large=0b101 << 5, inf=0b110 << 5)


@dataclass(frozen=True)
class CurveParams:
    """What the prover and the point codec need of one pairing curve.  fr.Element / fp.Element hold v * 2^(64 * words) mod
    the modulus (Montgomery form, little-endian u64 limbs); fr.Bytes / fp.Bytes = 8 * words (fr|fp/element.go:36-49)."""

    fr_words: int           # fr.Limbs
    fp_words: int           # fp.Limbs
    r: int                  # scalar-field modulus
    q: int                  # base-field modulus
    b: int                  # y^2 = x^3 + b, as an integer mod q
    flags: dict             # flag bits of the most significant byte of a serialised point (marshal.go:25-34)
    fr_id: int              # GMSM_FR_* of include/gmsm.h: the scalar field of fft.Domain and kzg._DevicePoly
    mult_gen: int           # fft.GeneratorFullMultiplicativeGroup (fr/fft/domain.go:56-60)

    @property
    def fr_bytes(self) -> int:
        return 8 * self.fr_words

    @property
    def fp_bytes(self) -> int:
        return 8 * self.fp_words


_Q_BW6761 = int("122E824FB83CE0AD187C94004FAFF3EB926186A81D14688528275EF8087BE41707BA638E584E91903CEBAFF25B423048689C8ED12F9FD9071DCD3DC73EBF"
                "F2E98A116C25667A8F8160CF8AEEAF0A437E6913E6870000082F49D00000000008B", 16)
CURVE_PARAMS = {
    "bn254": CurveParams(4, 4, 0x30644E72E131A029B85045B68181585D2833E84879B9709143E1F593F0000001,
                         0x30644E72E131A029B85045B68181585D97816A916871CA8D3C208C16D87CFD47, 3, _TWO_BIT, 0, 5),
    "bls12381": CurveParams(4, 6, 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001,
                            0x1A0111EA397FE69A4B1BA7B6434BACD764774B84F38512BF6730D2A0F6B0F6241EABFFFEB153FFFFB9FEFFFFFFFFAAAB, 4, _THREE_BIT,
                            1, 7),
    "bls12377": CurveParams(4, 6, 0x12AB655E9A2CA55660B44D1E5C37B00159AA76FED00000010A11800000000001,
                            0x01AE3A4617C510EAC63B05C06CA1493B1A22D9F300F5138F1EF3622FBA094800170B5D44300000008508C00000000001, 1, _THREE_BIT,
                            2, 22),
    "bls24315": CurveParams(4, 5, 0x196DEAC24A9DA12B25FC7EC9CF927A98C8C480ECE644E36419D0C5FD00C00001,
                            0x4C23A02B586D650D3F7498BE97C5EAFDEC1D01AA27A1AE0421EE5DA52BDE5026FE802FF40300001, 1, _THREE_BIT, 3, 7),
    "bls24317": CurveParams(4, 5, 0x443F917EA68DAFC2D0B097F28D83CD491CD1E79196BF0E7AF000000000000001,
                            0x1058CA226F60892CF28FC5A0B7F9D039169A61E684C73446D6F339E43424BF7E8D512E565DAB2AAB, 4, _THREE_BIT, 4, 7),
    "bw6633": CurveParams(5, 10, 0x4C23A02B586D650D3F7498BE97C5EAFDEC1D01AA27A1AE0421EE5DA52BDE5026FE802FF40300001,
                          int("126633CC0F35F63FC1A174F01D72AB5A8FCD8C75D79D2C74E59769AD9BBDA2F8152A6C0FADEA490B8DA9F5E83F57C497E0E8850EDBDA40"
                              "7D7B5CE7AB839C2253D369BD31147F73CD74916EA4570000D", 16), 4, _THREE_BIT, 5, 13),
    "bw6761": CurveParams(6, 12, 0x01AE3A4617C510EAC63B05C06CA1493B1A22D9F300F5138F1EF3622FBA094800170B5D44300000008508C00000000001,
                          _Q_BW6761, _Q_BW6761 - 1, _THREE_BIT, 6, 15),     # b = -1 (bw6-761.go)
}
# secp256k1 is no pairing curve: the engine only needs its group order (ecc/secp256k1/fr/element.go)
_R_SECP256K1 = 0xFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFEBAAEDCE6AF48A03BBFD25E8CD0364141


@dataclass(frozen=True)
class Group:
    """One group of the MultiExp engine.  A point coordinate is `degree` base-field elements of `fp_words` u64 limbs; a scalar is
    an fr.Element of the curve's scalar field."""

    id: int                 # gmsm_curve_t
    fp_words: int           # fp.Limbs
    degree: int             # extension degree of the coordinates: 1 = Fp, 2 = Fp2
    curve: str

    @property
    def words(self) -> int:
        """u64 words of one coordinate"""
        return self.fp_words * self.degree

    @property
    def r(self) -> int:
        return _R_SECP256K1 if self.curve == "secp256k1" else CURVE_PARAMS[self.curve].r

    @property
    def scalar_words(self) -> int:
        """fr.Limbs: a scalar is scalar_words x uint64 in Montgomery form"""
        return _limbs(self.r)

    @property
    def scalar_bits(self) -> int:
        """fr.Bits"""
        return self.r.bit_length()


# ecc/<curve>/multiexp.go of each: G2 of bw6-761 and bw6-633 is over Fp too; bls24-315 and bls24-317 have G1 only (their G2 is
# over Fp4), secp256k1 has no G2
GROUPS = {
    "bn254_g1": Group(0, 4, 1, "bn254"), "bn254_g2": Group(1, 4, 2, "bn254"),
    "bls12381_g1": Group(2, 6, 1, "bls12381"), "bls12381_g2": Group(3, 6, 2, "bls12381"),
    "bls12377_g1": Group(4, 6, 1, "bls12377"), "bls12377_g2": Group(5, 6, 2, "bls12377"),
    "secp256k1_g1": Group(6, 4, 1, "secp256k1"),
    "bw6761_g1": Group(7, 12, 1, "bw6761"), "bw6761_g2": Group(8, 12, 1, "bw6761"),
    "bls24315_g1": Group(9, 5, 1, "bls24315"), "bls24317_g1": Group(10, 5, 1, "bls24317"),
    "bw6633_g1": Group(11, 10, 1, "bw6633"), "bw6633_g2": Group(12, 10, 1, "bw6633"),
}
CURVES = {name: g.id for name, g in GROUPS.items()}


def _g1_name(curve: str) -> str:
    """the G1 group of a curve named with or without its "_g1" suffix"""
    return curve if curve.endswith("_g1") else curve + "_g1"


def _curve(name: str) -> str:
    """the curve of a curve or group name ("bn254_g1" -> "bn254")"""
    return name.split("_")[0]


def _params(curve: str) -> CurveParams:
    return CURVE_PARAMS[_curve(curve)]


def _limbs(modulus: int) -> int:
    """u64 limbs of an element mod `modulus` (fr.Limbs / fp.Limbs: the modulus' bit length rounded up to 64)"""
    return (modulus.bit_length() + 63) // 64


def _fr_decode(limbs: np.ndarray, r: int) -> list:
    """Montgomery limbs -> regular integers"""
    L = _limbs(r)
    rinv = pow(1 << (64 * L), -1, r)
    a = np.ascontiguousarray(limbs, dtype=np.uint64).reshape(-1, L)
    return [sum(int(x[i]) << (64 * i) for i in range(L)) * rinv % r for x in a]


def _fr_encode(vals, r: int) -> np.ndarray:
    L = _limbs(r)
    out = np.empty((len(vals), L), dtype=np.uint64)
    m64 = (1 << 64) - 1
    for i, v in enumerate(vals):
        m = (v << (64 * L)) % r
        out[i] = [(m >> (64 * k)) & m64 for k in range(L)]
    return out


def _reduced(limbs, r: int) -> np.ndarray:
    """Montgomery limbs of an fr.Element, reduced mod r (the device takes reduced elements only)"""
    return _fr_encode([_fr_decode(limbs, r)[0]], r)[0]


def _fr_marshal(limbs, r: int) -> bytes:
    """fr.Element.Marshal (fr/element.go:868-871): fr.Bytes (8 * fr.Limbs) bytes big-endian, canonical value"""
    return _fr_decode(np.asarray(limbs, dtype=np.uint64), r)[0].to_bytes(8 * _limbs(r), "big")


def _challenge(fs, name: str, r: int) -> int:
    """fr.Element.SetBytes of the raw challenge `name` of the transcript `fs`: big-endian, reduced mod r (fr/element.go:880-903)"""
    return int.from_bytes(fs.ComputeChallenge(name), "big") % r
