"""Next-row N2 (SURVEY.md section 8f): the caller on top of MultiExp and its raw SRS format.

  * kzg.Commit(p, pk, nbTasks...)            ecc/bn254/kzg/kzg.go:159-176  -> MultiExp over pk.G1[:len(p)]
  * kzg.NewSRS's G1 side (powers of alpha)   ecc/bn254/kzg/kzg.go:100-135  -> BatchScalarMultiplicationG1
  * unsafe.WriteSlice / ReadSlice            utils/unsafe/dump_slice.go:16-76 (uint64 LE length + raw
    []G1Affine memory) and the 0xdeadbeef marker that precedes it in SRS.WriteDump,
    ecc/bn254/kzg/marshal.go:70-115 -- the raw image IS the layout the device wants, so a dump streams
    straight into resident bases.
  * kzg.Open(p, point, pk)                   ecc/bn254/kzg/kzg.go:180-204  -> eval + dividePolyByXminusA on the device
    (gmsm_fr_poly_div_x_minus_a_device: one suffix scan gives f(a) and the quotient) and one MultiExp of the quotient, which
    stays in device memory
  * kzg.ToLagrangeG1(coeffs)                 ecc/bn254/kzg/utils.go:25-64 -> inverse FFT over G1 points on the device
    (gmsm_g1_to_lagrange, csrc/lagrange_kernels.cuh)
Polynomials are numpy (n, fr.Limbs) uint64 arrays or torch CUDA int64 tensors in the same fr.Element layout on the proving key's
device.  Proving keys sharded over several GPUs (device = -1) open on the host (Fr loops, as in the reference).
Only the G1 proving-key side is handled (the verifying key / pairing side is out of scope)."""
from __future__ import annotations

import ctypes
import io
import struct
from dataclasses import dataclass

import numpy as np

from . import _native
from .fft import _FIELDS
from .multiexp import CURVES, BatchScalarMultiplication, MultiExpConfig, MultiExpError, ResidentBases, _check, _words
from .transcript import Transcript

MARKER = 0xDEADBEEF  # utils/unsafe/dump_slice.go:78


class ErrInvalidPolynomialSize(MultiExpError):
    """kzg.ErrInvalidPolynomialSize (kzg.go:24)"""


def write_slice(w, points: np.ndarray) -> None:
    """unsafe.WriteSlice: uint64 little-endian length, then the raw element memory"""
    points = np.ascontiguousarray(points, dtype=np.uint64)
    w.write(struct.pack("<Q", points.shape[0]))
    if points.shape[0]:
        w.write(points.tobytes())


def read_slice(r, words_per_element: int, max_elements: int = 0) -> np.ndarray:
    """unsafe.ReadSlice (dump_slice.go:36-76): reads min(length, max_elements) elements, skips the rest"""
    hdr = r.read(8)
    if len(hdr) != 8:
        raise EOFError("unexpected EOF")
    (length,) = struct.unpack("<Q", hdr)
    limit = length
    if max_elements > 0 and length > max_elements:
        limit = max_elements
    size = 8 * words_per_element
    data = r.read(size * limit)
    if len(data) != size * limit:
        raise EOFError("unexpected EOF")
    if length > limit:
        r.seek((length - limit) * size, io.SEEK_CUR)
    return np.frombuffer(data, dtype=np.uint64).reshape(limit, words_per_element).copy()


def write_marker(w) -> None:
    w.write(struct.pack("<Q", MARKER))


def read_marker(r) -> None:
    b = r.read(8)
    if len(b) != 8 or struct.unpack("<Q", b)[0] != MARKER:
        raise ValueError("marker mismatch")  # dump_slice.go:92-99


class ProvingKey:
    """kzg.ProvingKey{G1 []G1Affine} (kzg.go:38-41) with the bases resident in HBM"""

    def __init__(self, curve: str, g1_points: np.ndarray, device: int = 0, window_tables: bool = False):
        self.curve = curve + "_g1" if not curve.endswith("_g1") else curve
        self.words = 2 * _words(CURVES[self.curve])
        self.G1 = np.ascontiguousarray(g1_points, dtype=np.uint64).reshape(-1, self.words)
        self.device = device       # -1: sharded over GMSM_DEVICES (host scalars only)
        self._bases = ResidentBases(self.curve, self.G1, device)
        if window_tables:          # the SRS is static: trade W x the device memory for faster commitments
            self._bases.Precompute()

    @classmethod
    def from_dump(cls, curve: str, r, max_pk_points: int = 0, device: int = 0):
        """the marker + slice tail of SRS.ReadDump (marshal.go:98-115); `r` positioned at the marker"""
        read_marker(r)
        cname = curve + "_g1" if not curve.endswith("_g1") else curve
        pts = read_slice(r, 2 * _words(CURVES[cname]), max_pk_points)
        return cls(curve, pts, device)

    @classmethod
    def from_bytes(cls, curve: str, data: bytes, n: int, raw: bool = False, check_on_curve: bool = True, device: int = 0):
        """n G1 points in the standard encoding (Encoder.Encode of a []G1Affine without its length prefix: Bytes() each, or
        RawBytes() each with RawEncoding, marshal.go:560-640) decoded on the device into resident bases"""
        return cls(curve, decode_g1_points(curve, data, n, raw, check_on_curve), device)

    def close(self):
        self._bases.close()


def new_srs_g1(curve: str, size: int, alpha: int, generator: np.ndarray, r_modulus: int, encode_scalars) -> np.ndarray:
    """G1 side of kzg.NewSRS (kzg.go:100-135): [1, alpha, alpha^2, ...] * G via BatchScalarMultiplicationG1.
    `encode_scalars` turns Python ints into Montgomery fr limbs (the caller's fr.Element constructor)."""
    alphas, a = [], 1
    for _ in range(size):
        alphas.append(a)
        a = a * alpha % r_modulus
    cname = curve + "_g1" if not curve.endswith("_g1") else curve
    return BatchScalarMultiplication(cname, generator, encode_scalars(alphas))


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

    @property
    def fr_bytes(self) -> int:
        return 8 * self.fr_words

    @property
    def fp_bytes(self) -> int:
        return 8 * self.fp_words


_Q_BW6761 = int("122E824FB83CE0AD187C94004FAFF3EB926186A81D14688528275EF8087BE41707BA638E584E91903CEBAFF25B423048689C8ED12F9FD9071DCD3DC73EBF"
                "F2E98A116C25667A8F8160CF8AEEAF0A437E6913E6870000082F49D00000000008B", 16)
# one entry per curve: fr/element.go and fp/element.go (q, Limbs), the curve's .go file (b), marshal.go (flags)
CURVE_PARAMS = {
    "bn254": CurveParams(4, 4, 0x30644E72E131A029B85045B68181585D2833E84879B9709143E1F593F0000001,
                         0x30644E72E131A029B85045B68181585D97816A916871CA8D3C208C16D87CFD47, 3, _TWO_BIT),
    "bls12381": CurveParams(4, 6, 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001,
                            0x1A0111EA397FE69A4B1BA7B6434BACD764774B84F38512BF6730D2A0F6B0F6241EABFFFEB153FFFFB9FEFFFFFFFFAAAB, 4, _THREE_BIT),
    "bls12377": CurveParams(4, 6, 0x12AB655E9A2CA55660B44D1E5C37B00159AA76FED00000010A11800000000001,
                            0x01AE3A4617C510EAC63B05C06CA1493B1A22D9F300F5138F1EF3622FBA094800170B5D44300000008508C00000000001, 1, _THREE_BIT),
    "bls24315": CurveParams(4, 5, 0x196DEAC24A9DA12B25FC7EC9CF927A98C8C480ECE644E36419D0C5FD00C00001,
                            0x4C23A02B586D650D3F7498BE97C5EAFDEC1D01AA27A1AE0421EE5DA52BDE5026FE802FF40300001, 1, _THREE_BIT),
    "bls24317": CurveParams(4, 5, 0x443F917EA68DAFC2D0B097F28D83CD491CD1E79196BF0E7AF000000000000001,
                            0x1058CA226F60892CF28FC5A0B7F9D039169A61E684C73446D6F339E43424BF7E8D512E565DAB2AAB, 4, _THREE_BIT),
    "bw6633": CurveParams(5, 10, 0x4C23A02B586D650D3F7498BE97C5EAFDEC1D01AA27A1AE0421EE5DA52BDE5026FE802FF40300001,
                          int("126633CC0F35F63FC1A174F01D72AB5A8FCD8C75D79D2C74E59769AD9BBDA2F8152A6C0FADEA490B8DA9F5E83F57C497E0E8850EDBDA40"
                              "7D7B5CE7AB839C2253D369BD31147F73CD74916EA4570000D", 16), 4, _THREE_BIT),
    "bw6761": CurveParams(6, 12, 0x01AE3A4617C510EAC63B05C06CA1493B1A22D9F300F5138F1EF3622FBA094800170B5D44300000008508C00000000001,
                          _Q_BW6761, _Q_BW6761 - 1, _THREE_BIT),            # b = -1 (bw6-761.go)
}
# views of the table by field, kept for callers of the earlier per-constant dictionaries
FR_MODULUS = {c: p.r for c, p in CURVE_PARAMS.items()}
FP_MODULUS = {c: p.q for c, p in CURVE_PARAMS.items()}
CURVE_B = {c: p.b for c, p in CURVE_PARAMS.items()}
_FLAGS = {c: p.flags for c, p in CURVE_PARAMS.items()}


def _params(curve: str) -> CurveParams:
    return CURVE_PARAMS[curve.split("_")[0]]


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


def _eval(p: list, point: int, r: int) -> int:
    """eval (kzg.go:55-63): Horner from the top coefficient"""
    res = p[-1]
    for i in range(len(p) - 2, -1, -1):
        res = (res * point + p[i]) % r
    return res


def _divide_by_x_minus_a(f: list, fa: int, a: int, r: int) -> list:
    """dividePolyByXminusA (kzg.go:567-584): (f - f(a)) / (X - a) by synthetic division, result of degree deg(f) - 1"""
    f = list(f)
    f[0] = (f[0] - fa) % r
    for i in range(len(f) - 2, -1, -1):
        f[i] = (f[i] + f[i + 1] * a) % r
    return f[1:]


def _is_device(p) -> bool:
    """a torch tensor (device polynomial) rather than an array-like of host limbs"""
    return hasattr(p, "data_ptr") and hasattr(p, "is_cuda")


def _host_poly(p, words: int) -> np.ndarray:
    if _is_device(p):
        p = p.detach().cpu().numpy().view(np.uint64)
    return np.ascontiguousarray(p, dtype=np.uint64).reshape(-1, words)


def _poly_len(p, words: int) -> int:
    if _is_device(p):
        if p.numel() % words:
            raise ValueError("a device polynomial holds whole fr.Elements (%d int64 each)" % words)
        return p.numel() // words
    return _host_poly(p, words).shape[0]


def _device_poly(p, words: int, device: int):
    """p as a torch int64 tensor on cuda:device: device tensors are used in place (never modified), host arrays uploaded once"""
    import torch

    if _is_device(p):
        if not p.is_cuda or p.device.index != device or p.dtype != torch.int64 or not p.is_contiguous():
            raise ValueError("a device polynomial must be a contiguous torch.int64 CUDA tensor on cuda:%d" % device)
        return p
    h = _host_poly(p, words).view(np.int64).reshape(-1)
    if not h.flags.writeable:           # torch.from_numpy wants a writable buffer; it is only read
        h = h.copy()
    return torch.from_numpy(h).to(torch.device("cuda", device))


def _reduced(limbs, r: int) -> np.ndarray:
    """Montgomery limbs of an fr.Element, reduced mod r (the device takes reduced elements only)"""
    return _fr_encode([_fr_decode(limbs, r)[0]], r)[0]


def _digest(jac: np.ndarray, w: int) -> np.ndarray:
    return jac[:w].copy() if jac[w:].any() else np.zeros(w, dtype=np.uint64)


class _DevicePoly:
    """gmsm_fr_poly_* of one proving key's curve on its device, ordered on the device's current torch stream"""

    def __init__(self, pk: ProvingKey, max_len: int):
        import torch

        self.torch = torch
        self.field = _FIELDS[pk.curve.split("_")[0]]
        self.words = _params(pk.curve).fr_words
        self.dev = torch.device("cuda", pk.device)
        self.stream = torch.cuda.current_stream(self.dev).cuda_stream
        ws = int(_native.lib().gmsm_fr_poly_workspace_bytes(self.field, max_len))
        self.work = torch.empty(ws // 8, dtype=torch.int64, device=self.dev) if ws else None

    def empty(self, n: int):
        return self.torch.empty(n * self.words, dtype=self.torch.int64, device=self.dev)

    def div(self, d_f, n: int, a: np.ndarray, d_h, d_fa):
        """d_fa = f(a); d_h = (f - f(a)) / (X - a) unless None"""
        _check(_native.lib().gmsm_fr_poly_div_x_minus_a_device(
            self.field, d_f.data_ptr(), n, a.ctypes.data, None if d_h is None else d_h.data_ptr(), d_fa.data_ptr(),
            None if self.work is None else self.work.data_ptr(), self.stream))

    def fold(self, d_polys, lens, gamma: np.ndarray, d_out, out_len: int):
        ptrs = (ctypes.c_void_p * len(d_polys))(*[d.data_ptr() for d in d_polys])
        ln = np.array(lens, dtype=np.uint64)
        _check(_native.lib().gmsm_fr_poly_fold_device(self.field, ptrs, ln.ctypes.data, len(d_polys), gamma.ctypes.data, d_out.data_ptr(),
                                                       out_len, self.stream))

    def lincomb(self, d_polys, lens, scalars: np.ndarray, strides, offsets, d_out, out_len: int, accumulate: bool = False):
        """d_out[m * strides[i] + offsets[i]] (+)= scalars[i] * d_polys[i][m]; scalars: (k, fr.Limbs) reduced limbs"""
        k = len(d_polys)
        ptrs = (ctypes.c_void_p * k)(*[d.data_ptr() for d in d_polys])
        ln, st, off = (np.array(v, dtype=np.uint64) for v in (lens, strides, offsets))
        sc = np.ascontiguousarray(scalars, dtype=np.uint64)
        _check(_native.lib().gmsm_fr_poly_lincomb_device(self.field, ptrs, ln.ctypes.data, sc.ctypes.data, st.ctypes.data, off.ctypes.data,
                                                          k, d_out.data_ptr(), out_len, 1 if accumulate else 0, self.stream))


@dataclass
class OpeningProof:
    """kzg.OpeningProof{H G1Affine, ClaimedValue fr.Element} (kzg.go:43-51), both in Go memory layout"""

    H: np.ndarray
    ClaimedValue: np.ndarray


def Open(p, point: np.ndarray, pk: ProvingKey) -> OpeningProof:
    """kzg.Open (kzg.go:180-204): ClaimedValue = p(point); H = Commit((p - p(point)) / (X - point)).  On a single-device proving key
    the value and the quotient come from one scan on the device and the quotient feeds the MultiExp there; only f(a) and H come
    back."""
    cp = _params(pk.curve)
    r = cp.r
    if pk.device >= 0:
        n = _poly_len(p, cp.fr_words)
        # n == 1: Commit of the empty quotient errors in the reference (kzg.go:160-162): a constant polynomial cannot be opened
        if n <= 1 or n > pk.G1.shape[0]:
            raise ErrInvalidPolynomialSize("invalid polynomial size (larger than SRS or == 0)")
        import torch

        with torch.cuda.device(pk.device):
            dp = _DevicePoly(pk, n)
            d_f = _device_poly(p, cp.fr_words, pk.device)
            d_h, d_fa = dp.empty(n - 1), dp.empty(1)
            dp.div(d_f, n, _reduced(point, r), d_h, d_fa)
            jac = pk._bases.MultiExpDevice(d_h, n - 1, stream=dp.stream)
            fa = d_fa.cpu().numpy().view(np.uint64)
        return OpeningProof(H=_digest(jac, pk.words), ClaimedValue=fa.copy())
    p = _host_poly(p, cp.fr_words)
    if p.shape[0] == 0 or p.shape[0] > pk.G1.shape[0]:
        raise ErrInvalidPolynomialSize("invalid polynomial size (larger than SRS or == 0)")
    coeffs = _fr_decode(p, r)
    a = _fr_decode(point, r)[0]
    fa = _eval(coeffs, a, r)
    h = _divide_by_x_minus_a(coeffs, fa, a, r)
    w = pk.words
    # Commit(h, pk) errors on an empty h in the reference (kzg.go:160-162): a constant polynomial cannot be opened
    H = Commit(_fr_encode(h, r), pk) if h else None
    if H is None:
        raise ErrInvalidPolynomialSize("invalid polynomial size (larger than SRS or == 0)")
    return OpeningProof(H=H.reshape(w), ClaimedValue=_fr_encode([fa], r)[0])


def Commit(p, pk: ProvingKey, *nbTasks: int) -> np.ndarray:
    """kzg.Commit (kzg.go:159-176): Digest = MultiExp(pk.G1[:len(p)], p) as an affine point.  A device polynomial (torch tensor)
    goes straight to the MultiExp on a single-device proving key."""
    words = _params(pk.curve).fr_words
    cfg = MultiExpConfig(NbTasks=nbTasks[0] if nbTasks else 0)
    if _is_device(p) and pk.device >= 0:
        n = _poly_len(p, words)
        if n == 0 or n > pk.G1.shape[0]:
            raise ErrInvalidPolynomialSize("invalid polynomial size (larger than SRS or == 0)")
        import torch

        with torch.cuda.device(pk.device):
            d = _device_poly(p, words, pk.device)
            jac = pk._bases.MultiExpDevice(d, n, cfg, stream=torch.cuda.current_stream(d.device).cuda_stream)
        return _digest(jac, pk.words)
    p = _host_poly(p, words)
    if p.shape[0] == 0 or p.shape[0] > pk.G1.shape[0]:
        raise ErrInvalidPolynomialSize("invalid polynomial size (larger than SRS or == 0)")
    return _digest(pk._bases.MultiExp(p, cfg), pk.words)


# ----------------------------------------------------------------------------------------------------------------
# point (de)serialisation on the host -- G1Affine.RawBytes / Bytes / SetBytes (ecc/bn254/marshal.go:801-950,
# ecc/bls12-381/marshal.go:830-1000).  Used for the few points a Fiat-Shamir transcript binds (G1Affine.Marshal is
# RawBytes, marshal.go:779-782); bulk SRS decoding runs on the device (gmsm_g1_decode, csrc/decode.cu).
# ----------------------------------------------------------------------------------------------------------------
def _fp_words(curve: str) -> int:
    return _params(curve).fp_words


def _fp_decode(limbs, curve: str) -> int:
    L = _fp_words(curve)
    p = _params(curve).q
    v = sum(int(limbs[i]) << (64 * i) for i in range(L))
    return v * pow(1 << (64 * L), -1, p) % p


def _fp_encode(v: int, curve: str) -> np.ndarray:
    L = _fp_words(curve)
    p = _params(curve).q
    m = (v << (64 * L)) % p
    return np.array([(m >> (64 * i)) & (2**64 - 1) for i in range(L)], dtype=np.uint64)


def g1_raw_bytes(point: np.ndarray, curve: str) -> bytes:
    """G1Affine.RawBytes (marshal.go:826-846): big-endian X || Y, canonical; infinity = flag + zeroes"""
    L = _fp_words(curve)
    point = np.ascontiguousarray(point, dtype=np.uint64).reshape(2 * L)
    nb = 8 * L
    if not point.any():
        f = _params(curve).flags
        out = bytearray(2 * nb)
        out[0] = f["unc"] if f["unc_inf"] is None else f["unc_inf"]
        return bytes(out)
    x, y = _fp_decode(point[:L], curve), _fp_decode(point[L:], curve)
    return x.to_bytes(nb, "big") + y.to_bytes(nb, "big")      # mUncompressed = 0: no bits to set


def g1_bytes(point: np.ndarray, curve: str) -> bytes:
    """G1Affine.Bytes (marshal.go:801-823): compressed -- big-endian X with the flag bits in the top byte"""
    L = _fp_words(curve)
    point = np.ascontiguousarray(point, dtype=np.uint64).reshape(2 * L)
    nb = 8 * L
    f = _params(curve).flags
    if not point.any():
        out = bytearray(nb)
        out[0] = f["inf"]
        return bytes(out)
    p = _params(curve).q
    x, y = _fp_decode(point[:L], curve), _fp_decode(point[L:], curve)
    out = bytearray(x.to_bytes(nb, "big"))
    out[0] |= f["large"] if y > (p - 1) // 2 else f["small"]        # LexicographicallyLargest, fp/element.go:282-296
    return bytes(out)


def g1_set_bytes(buf: bytes, curve: str):
    """G1Affine.SetBytes without the subgroup check (marshal.go:858-950) for ONE point on the host -> (point limbs, consumed).
    Raises ValueError with the reference's messages on invalid encodings."""
    cp = _params(curve)
    L = cp.fp_words
    nb = cp.fp_bytes
    f = cp.flags
    p = cp.q
    if len(buf) < nb:
        raise EOFError("short buffer")
    m = buf[0] & f["mask"]
    if m == f["inf"]:
        if (buf[0] & ~f["mask"] & 0xFF) or any(buf[1:nb]):
            raise ValueError("invalid infinity point encoding")
        return np.zeros(2 * L, dtype=np.uint64), nb
    if f["unc_inf"] is not None and m == f["unc_inf"]:
        if len(buf) < 2 * nb:
            raise EOFError("short buffer")
        if (buf[0] & ~f["mask"] & 0xFF) or any(buf[1:2 * nb]):
            raise ValueError("invalid infinity point encoding")
        return np.zeros(2 * L, dtype=np.uint64), 2 * nb
    xb = bytearray(buf[:nb])
    xb[0] &= ~f["mask"] & 0xFF
    x = int.from_bytes(xb, "big")
    if x >= p:
        raise ValueError("invalid fp.Element encoding")
    if m == f["unc"]:
        if len(buf) < 2 * nb:
            raise EOFError("short buffer")
        y = int.from_bytes(buf[nb:2 * nb], "big")
        if y >= p:
            raise ValueError("invalid fp.Element encoding")
        return np.concatenate([_fp_encode(x, curve), _fp_encode(y, curve)]), 2 * nb
    if m not in (f["small"], f["large"]):
        raise ValueError("invalid point encoding")
    y2 = (x * x * x + cp.b) % p
    if p % 4 == 3:
        y = pow(y2, (p + 1) // 4, p)
    else:                                   # Tonelli-Shanks (bls12-377, bls24-315, bw6-633: q = 1 mod 4, fp/element.go Sqrt)
        y = _tonelli(y2, p)
    if y is None or y * y % p != y2:
        raise ValueError("invalid compressed coordinate: square root doesn't exist")
    if (y > (p - 1) // 2) != (m == f["large"]):
        y = p - y
    return np.concatenate([_fp_encode(x, curve), _fp_encode(y, curve)]), nb


def _tonelli(a: int, p: int):
    if a == 0:
        return 0
    if pow(a, (p - 1) // 2, p) != 1:
        return None
    q, s = p - 1, 0
    while q % 2 == 0:
        q //= 2
        s += 1
    z = 2
    while pow(z, (p - 1) // 2, p) != p - 1:
        z += 1
    m, c, t, r = s, pow(z, q, p), pow(a, q, p), pow(a, (q + 1) // 2, p)
    while t != 1:
        i, t2 = 0, t
        while t2 != 1:
            t2 = t2 * t2 % p
            i += 1
        b = pow(c, 1 << (m - i - 1), p)
        m, c, t, r = i, b * b % p, t * b * b % p, r * b % p
    return r


# ----------------------------------------------------------------------------------------------------------------
# batched openings at one point (kzg.go:246-420): the prover side; verification (pairings) is out of scope
# ----------------------------------------------------------------------------------------------------------------
class ErrInvalidNbDigests(MultiExpError):
    """kzg.ErrInvalidNbDigests (kzg.go:23)"""


@dataclass
class BatchOpeningProof:
    """kzg.BatchOpeningProof{H G1Affine, ClaimedValues []fr.Element} (kzg.go:66-77)"""

    H: np.ndarray
    ClaimedValues: np.ndarray


def _fr_marshal(limbs, r: int) -> bytes:
    """fr.Element.Marshal (fr/element.go:868-871): fr.Bytes (8 * fr.Limbs) bytes big-endian, canonical value"""
    return _fr_decode(np.asarray(limbs, dtype=np.uint64), r)[0].to_bytes(8 * _limbs(r), "big")


def derive_gamma(point, digests, claimed_values, hf, curve: str, *data_transcript: bytes) -> int:
    """deriveGamma (kzg.go:531-563) over fiatshamir.Transcript (fiat-shamir/transcript.go:61-131) with the single challenge
    "gamma": H("gamma" || point || digests (RawBytes) || claimed values || extra data), read big-endian and reduced mod r
    (fr.SetBytes, fr/element.go:880-903).  `hf` is a hashlib constructor (e.g. hashlib.sha256)."""
    c = curve.split("_")[0]
    cp = CURVE_PARAMS[c]
    r = cp.r
    fs = Transcript(hf, "gamma")
    fs.Bind("gamma", _fr_marshal(point, r))
    for d in digests:
        fs.Bind("gamma", g1_raw_bytes(d, c))
    for v in np.ascontiguousarray(claimed_values, dtype=np.uint64).reshape(-1, cp.fr_words):
        fs.Bind("gamma", _fr_marshal(v, r))
    for b in data_transcript:
        fs.Bind("gamma", b)
    return int.from_bytes(fs.ComputeChallenge("gamma"), "big") % r


def BatchOpenSinglePoint(polynomials, digests, point: np.ndarray, hf, pk: ProvingKey, *data_transcript: bytes) -> BatchOpeningProof:
    """kzg.BatchOpenSinglePoint (kzg.go:246-331): ClaimedValues[i] = f_i(point); gamma by Fiat-Shamir; the folded polynomial
    sum_i gamma^i f_i is divided by (X - point) and committed with ONE MultiExp over the resident bases.  On a single-device
    proving key the evaluations, the fold and the division run on the device: the claimed values come back in one copy for
    the transcript, the folded polynomial and its quotient never leave the device."""
    if len(digests) != len(polynomials):
        raise ErrInvalidNbDigests("number of digests is not the same as the number of polynomials")
    c = pk.curve.split("_")[0]
    cp = CURVE_PARAMS[c]
    r = cp.r
    if pk.device >= 0:
        return _batch_open_device(polynomials, digests, point, hf, pk, *data_transcript)
    polys = []
    for p in polynomials:
        p = _host_poly(p, cp.fr_words)
        if p.shape[0] == 0 or p.shape[0] > pk.G1.shape[0]:
            raise ErrInvalidPolynomialSize("invalid polynomial size (larger than SRS or == 0)")
        polys.append(_fr_decode(p, r))
    a = _fr_decode(point, r)[0]
    claimed = [_eval(f, a, r) for f in polys]
    claimed_limbs = _fr_encode(claimed, r)
    gamma = derive_gamma(point, digests, claimed_limbs, hf, c, *data_transcript)
    folded_eval = claimed[-1]
    for v in reversed(claimed[:-1]):
        folded_eval = (folded_eval * gamma + v) % r
    largest = max(len(f) for f in polys)
    folded = list(polys[0]) + [0] * (largest - len(polys[0]))
    g = 1
    for f in polys[1:]:
        g = g * gamma % r
        for j, v in enumerate(f):
            folded[j] = (folded[j] + v * g) % r
    h = _divide_by_x_minus_a(folded, folded_eval, a, r)
    if not h:
        raise ErrInvalidPolynomialSize("invalid polynomial size (larger than SRS or == 0)")
    H = Commit(_fr_encode(h, r), pk)
    return BatchOpeningProof(H=H.reshape(pk.words), ClaimedValues=claimed_limbs)


def _batch_open_device(polynomials, digests, point, hf, pk: ProvingKey, *data_transcript: bytes) -> BatchOpeningProof:
    import torch

    c = pk.curve.split("_")[0]
    cp = CURVE_PARAMS[c]
    r, w = cp.r, cp.fr_words
    lens = []
    for p in polynomials:
        n = _poly_len(p, w)
        if n == 0 or n > pk.G1.shape[0]:
            raise ErrInvalidPolynomialSize("invalid polynomial size (larger than SRS or == 0)")
        lens.append(n)
    largest = max(lens)
    a = _reduced(point, r)
    with torch.cuda.device(pk.device):
        dp = _DevicePoly(pk, largest)
        d_polys = [_device_poly(p, w, pk.device) for p in polynomials]
        d_claimed = dp.empty(len(lens))
        for i, (d_f, n) in enumerate(zip(d_polys, lens)):
            dp.div(d_f, n, a, None, d_claimed[i * w:(i + 1) * w])
        claimed_limbs = d_claimed.cpu().numpy().view(np.uint64).reshape(-1, w).copy()
        gamma = derive_gamma(point, digests, claimed_limbs, hf, c, *data_transcript)
        if largest == 1:        # the folded quotient is empty: Commit errors in the reference
            raise ErrInvalidPolynomialSize("invalid polynomial size (larger than SRS or == 0)")
        d_fold = dp.empty(largest)
        dp.fold(d_polys, lens, _fr_encode([gamma], r)[0], d_fold, largest)
        d_h, d_fa = dp.empty(largest - 1), dp.empty(1)
        dp.div(d_fold, largest, a, d_h, d_fa)
        jac = pk._bases.MultiExpDevice(d_h, largest - 1, stream=dp.stream)
    return BatchOpeningProof(H=_digest(jac, pk.words), ClaimedValues=claimed_limbs)


def FoldProof(digests, proof: BatchOpeningProof, point: np.ndarray, hf, curve: str, *data_transcript: bytes):
    """kzg.FoldProof (kzg.go:341-380) -> (OpeningProof, folded digest): the claimed values are folded with [1, gamma, ...] on the
    host, the digests with one MultiExp (`fold`, kzg.go:506-528 -- the reference calls MultiExp for it too)."""
    from .multiexp import curve_package

    c = curve.split("_")[0]
    cp = CURVE_PARAMS[c]
    claimed = np.ascontiguousarray(proof.ClaimedValues, dtype=np.uint64).reshape(-1, cp.fr_words)
    if len(digests) != claimed.shape[0]:
        raise ErrInvalidNbDigests("number of digests is not the same as the number of polynomials")
    r = cp.r
    gamma = derive_gamma(point, digests, claimed, hf, c, *data_transcript)
    gam = [1]
    for _ in range(1, len(digests)):
        gam.append(gam[-1] * gamma % r)
    vals = _fr_decode(claimed, r)
    folded_eval = sum(v * g for v, g in zip(vals, gam)) % r
    aff_cls = curve_package(c)[0]
    pts = np.ascontiguousarray(np.stack([np.asarray(d, dtype=np.uint64).reshape(-1) for d in digests]))
    folded_digest = aff_cls().MultiExp(pts, _fr_encode(gam, r), MultiExpConfig()).limbs
    return OpeningProof(H=np.array(proof.H, dtype=np.uint64), ClaimedValue=_fr_encode([folded_eval], r)[0]), folded_digest


def decode_g1_points(curve: str, data: bytes, n: int, raw: bool = False, check_on_curve: bool = True) -> np.ndarray:
    """bulk G1Affine.SetBytes on the GPU (gmsm_g1_decode, csrc/decode.cu): n points of a homogeneous stream -> (n, words) uint64
    in Go memory layout.  Raises MultiExpError with the reference's message and the index of the first invalid point."""
    from . import _native

    cname = curve + "_g1" if not curve.endswith("_g1") else curve
    words = 2 * _words(CURVES[cname])
    per = 8 * words if raw else 4 * words
    if len(data) < n * per:
        raise EOFError("short buffer")      # io.ErrShortBuffer
    buf = np.frombuffer(data, dtype=np.uint8, count=n * per)
    out = np.zeros((n, words), dtype=np.uint64)
    rc = _native.lib().gmsm_g1_decode(CURVES[cname], buf.ctypes.data, n, 1 if raw else 0, 1 if check_on_curve else 0, out.ctypes.data)
    if rc != 0:
        raise MultiExpError(_native.last_error())
    return out


def ToLagrangeG1(coeffs, curve: str, device: int = 0):
    """kzg.ToLagrangeG1 (utils.go:25-64): the Lagrange form [L_i(tau)]G of a canonical SRS [tau^i]G, by an inverse FFT over G1
    points on the GPU (gmsm_g1_to_lagrange, csrc/lagrange_kernels.cuh).  `coeffs`: (n, 2 * fp.Limbs) uint64 array of G1Affine in Go
    memory layout, n a power of two; returns a new array in the affine normal form.  A torch CUDA int64 tensor in the same layout is
    transformed on its own device, on the current stream, into a new tensor (the input is left unmodified, nothing visits the
    host).  ProvingKey(curve, ToLagrangeG1(srs, curve)) is the Lagrange-form key: Commit of evaluations on the domain of size n
    with it equals CommitLagrange with the canonical key.  Errors are MultiExpError with the reference's texts."""
    cname = curve if curve.endswith(("_g1", "_g2")) else curve + "_g1"
    if cname not in CURVES:
        raise MultiExpError("unknown curve %r" % curve)
    cid = CURVES[cname]
    words = 2 * _words(cid)
    L = _native.lib()
    if _is_device(coeffs):
        import torch

        if not coeffs.is_cuda or coeffs.dtype != torch.int64 or not coeffs.is_contiguous() or coeffs.numel() % words:
            raise ValueError("device points must be a contiguous torch.int64 CUDA tensor of (n, %d) words" % words)
        n = coeffs.numel() // words
        out = torch.empty_like(coeffs)
        with torch.cuda.device(coeffs.device):
            ws = int(L.gmsm_g1_to_lagrange_workspace_bytes(cid, n))
            work = torch.empty(max(ws // 8, 1), dtype=torch.int64, device=coeffs.device)
            st = torch.cuda.current_stream(coeffs.device).cuda_stream
            _check(L.gmsm_g1_to_lagrange_device(cid, coeffs.data_ptr(), n, out.data_ptr(), work.data_ptr(), st))
        return out
    pts = np.ascontiguousarray(coeffs, dtype=np.uint64).reshape(-1, words)
    out = np.empty_like(pts)
    _check(L.gmsm_g1_to_lagrange(cid, pts.ctypes.data, pts.shape[0], device, out.ctypes.data))
    return out


def CommitLagrange(evals, pk: ProvingKey, domain) -> np.ndarray:
    """Digest of the polynomial given by its values on `domain` (fft.Domain of this package): the evaluations go to the device
    once, FFTInverse(DIF) + BitReverse (fft.go:111-190, bitreverse.go:17-42) run there and their output -- the coefficients,
    still in device memory, Montgomery form -- feeds the MultiExp directly (gmsm_bases_multiexp_device): the canonical-form
    coefficients never visit the host.  Equals Commit(FFTInverse(evals), pk)."""
    import torch

    from .fft import DIF

    ev = np.ascontiguousarray(evals, dtype=np.uint64).reshape(-1, _params(pk.curve).fr_words)
    if ev.shape[0] != domain.Cardinality:
        raise MultiExpError("len(a) must equal the domain cardinality")
    if ev.shape[0] == 0 or ev.shape[0] > pk.G1.shape[0]:
        raise ErrInvalidPolynomialSize("invalid polynomial size (larger than SRS or == 0)")
    dev = torch.device("cuda", domain.device)
    d = torch.from_numpy(ev.view(np.int64).reshape(-1).copy()).to(dev)
    st = torch.cuda.current_stream(dev).cuda_stream
    domain.fft_device(d, True, DIF, False, st)          # natural in, bit-reversed out
    domain.bit_reverse_device(d, st)
    jac = pk._bases.MultiExpDevice(d, ev.shape[0], stream=st)
    w = pk.words
    return jac[:w].copy() if jac[w:].any() else np.zeros(w, dtype=np.uint64)
