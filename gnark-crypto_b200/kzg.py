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
from .curves import CURVE_PARAMS, CurveParams  # noqa: F401  (kzg's names for the curve table)
from .curves import CURVES, GROUPS, _challenge, _curve, _fr_decode, _fr_encode, _fr_marshal, _g1_name, _params, _reduced
from .multiexp import BatchScalarMultiplication, MultiExpConfig, MultiExpError, ResidentBases, _check
from .transcript import Transcript

MARKER = 0xDEADBEEF  # utils/unsafe/dump_slice.go:78


class ErrInvalidPolynomialSize(MultiExpError):
    """kzg.ErrInvalidPolynomialSize (kzg.go:24)"""


def _check_size(n: int, n_min: int, n_max: int) -> None:
    """the refusal of kzg.Commit (kzg.go:160-162) of a polynomial that is empty or larger than the SRS, with the caller's bounds"""
    if not n_min <= n <= n_max:
        raise ErrInvalidPolynomialSize("invalid polynomial size (larger than SRS or == 0)")


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
        self.curve = _g1_name(curve)
        self.words = 2 * GROUPS[self.curve].words
        self.G1 = np.ascontiguousarray(g1_points, dtype=np.uint64).reshape(-1, self.words)
        self.device = device       # -1: sharded over GMSM_DEVICES (host scalars only)
        self._bases = ResidentBases(self.curve, self.G1, device)
        if window_tables:          # the SRS is static: trade W x the device memory for faster commitments
            self._bases.Precompute()

    @classmethod
    def from_dump(cls, curve: str, r, max_pk_points: int = 0, device: int = 0):
        """the marker + slice tail of SRS.ReadDump (marshal.go:98-115); `r` positioned at the marker"""
        read_marker(r)
        pts = read_slice(r, 2 * GROUPS[_g1_name(curve)].words, max_pk_points)
        return cls(curve, pts, device)

    @classmethod
    def from_bytes(cls, curve: str, data: bytes, n: int, raw: bool = False, check_on_curve: bool = True, device: int = 0):
        """n G1 points in the standard encoding (Encoder.Encode of a []G1Affine without its length prefix: Bytes() each, or
        RawBytes() each with RawEncoding, marshal.go:560-640) decoded on the device into resident bases"""
        return cls(curve, decode_g1_points(curve, data, n, raw, check_on_curve), device)

    def close(self):
        self._bases.close()

    def WriteTo(self, w) -> int:
        """ProvingKey.WriteTo (kzg/marshal.go:16-33): pk.G1 as a compressed []G1Affine slice, encoded on the GPU.  Returns the
        bytes written."""
        return write_points(w, self.curve, self.G1, raw=False)

    def WriteRawTo(self, w) -> int:
        """ProvingKey.WriteRawTo: the same without point compression (RawEncoding)"""
        return write_points(w, self.curve, self.G1, raw=True)

    @classmethod
    def UnsafeReadFrom(cls, curve: str, r, device: int = 0):
        """ProvingKey.UnsafeReadFrom (kzg/marshal.go:140-160): a []G1Affine slice decoded on the GPU without subgroup (or
        on-curve) checks -> (ProvingKey with the bases resident on `device`, bytes read)"""
        pts, nbytes = _read_points(r, _g1_name(curve), False, None)
        return cls(curve, pts, device), nbytes



def new_srs_g1(curve: str, size: int, alpha: int, generator: np.ndarray, r_modulus: int, encode_scalars) -> np.ndarray:
    """G1 side of kzg.NewSRS (kzg.go:100-135): [1, alpha, alpha^2, ...] * G via BatchScalarMultiplicationG1.
    `encode_scalars` turns Python ints into Montgomery fr limbs (the caller's fr.Element constructor)."""
    alphas, a = [], 1
    for _ in range(size):
        alphas.append(a)
        a = a * alpha % r_modulus
    return BatchScalarMultiplication(_g1_name(curve), generator, encode_scalars(alphas))


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


def _stream(device):
    """the current torch stream of `device`, which orders the work of a call"""
    import torch

    return torch.cuda.current_stream(device).cuda_stream


def _digest(jac: np.ndarray, w: int) -> np.ndarray:
    return jac[:w].copy() if jac[w:].any() else np.zeros(w, dtype=np.uint64)


class _DevicePoly:
    """the gmsm_fr_* entry points of one curve's scalar field on one device, ordered on the device's current torch stream, with a
    workspace for polynomials of up to max_len coefficients"""

    def __init__(self, curve: str, device: int, max_len: int):
        import torch

        self.torch = torch
        self.field = _params(curve).fr_id
        self.words = _params(curve).fr_words
        self.dev = torch.device("cuda", device)
        self.stream = _stream(self.dev)
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

    def permutation_accumulate(self, d_t1, d_t2, n: int, eps: np.ndarray, d_z):
        """d_z = the accumulation polynomial Z of permutation.Prove in the bit-reversed Lagrange layout (n <= max_len)"""
        _check(_native.lib().gmsm_fr_permutation_accumulate_device(self.field, d_t1.data_ptr(), d_t2.data_ptr(), n, eps.ctypes.data,
                                                                   d_z.data_ptr(), None if self.work is None else self.work.data_ptr(),
                                                                   self.stream))

    def permutation_numerator(self, domain, d_lt1, d_lt2, d_lz, eps: np.ndarray, omega: np.ndarray, d_out):
        """d_out = the quotient numerator of permutation.Prove on the coset of `domain` (an fft.Domain of this field)"""
        _check(_native.lib().gmsm_fft_permutation_numerator_device(domain._h, d_lt1.data_ptr(), d_lt2.data_ptr(), d_lz.data_ptr(),
                                                                   domain.Cardinality, eps.ctypes.data, omega.ctypes.data,
                                                                   d_out.data_ptr(), self.stream))

    def sort(self, d_in, n: int, d_out):
        """d_out = d_in sorted ascending by canonical value (sort.Sort(fr.Vector)); d_out may be d_in.  Returns once the sort has
        read back which byte positions vary."""
        ws = int(_native.lib().gmsm_fr_sort_workspace_bytes(self.field, n))
        work = self.torch.empty((ws + 7) // 8, dtype=self.torch.int64, device=self.dev)
        _check(_native.lib().gmsm_fr_sort_device(self.field, d_in.data_ptr(), n, d_out.data_ptr(), work.data_ptr(), self.stream))

    def plookup_accumulate(self, d_f, d_t, d_h1, d_h2, n: int, beta: np.ndarray, gamma: np.ndarray, d_z):
        """d_z = the accumulation polynomial z of plookup.ProveLookupVector in natural order (n <= max_len)"""
        _check(_native.lib().gmsm_fr_plookup_accumulate_device(
            self.field, d_f.data_ptr(), d_t.data_ptr(), d_h1.data_ptr(), d_h2.data_ptr(), n, beta.ctypes.data, gamma.ctypes.data,
            d_z.data_ptr(), None if self.work is None else self.work.data_ptr(), self.stream))

    def plookup_numerator(self, domain, d_lz, d_lh1, d_lh2, d_lt, d_lf, beta: np.ndarray, gamma: np.ndarray, alpha: np.ndarray, d_out):
        """d_out = the quotient of plookup.ProveLookupVector before its inverse FFT, on the coset of `domain` (the big domain)"""
        _check(_native.lib().gmsm_fft_plookup_numerator_device(
            domain._h, d_lz.data_ptr(), d_lh1.data_ptr(), d_lh2.data_ptr(), d_lt.data_ptr(), d_lf.data_ptr(), domain.Cardinality,
            beta.ctypes.data, gamma.ctypes.data, alpha.ctypes.data, d_out.data_ptr(), self.stream))

    def bit_reverse(self, d_a, n: int):
        """fft.BitReverse of d_a in place (n a power of two)"""
        _check(_native.lib().gmsm_fr_bit_reverse_device(self.field, d_a.data_ptr(), n, self.stream))

    # the iop package (iop.py): every call takes the workspace of gmsm_fr_iop_workspace_bytes for n elements, allocated once per size
    def _iop_work(self, n: int):
        ws = int(_native.lib().gmsm_fr_iop_workspace_bytes(self.field, n))
        if getattr(self, "_iop_ws", None) is None or self._iop_ws.numel() * 8 < ws:
            self._iop_ws = self.torch.empty((ws + 7) // 8, dtype=self.torch.int64, device=self.dev)
        return self._iop_ws

    def iop_ratio_shuffled(self, d_num, num_bitrev, d_den, den_bitrev, n: int, beta: np.ndarray, d_z):
        """d_z = the accumulating ratio of BuildRatioShuffledVectors in Lagrange Regular form (inputs already in Lagrange form)"""
        k = len(d_num)
        num = (ctypes.c_void_p * k)(*[d.data_ptr() for d in d_num])
        den = (ctypes.c_void_p * k)(*[d.data_ptr() for d in d_den])
        nb, db = (ctypes.c_int * k)(*num_bitrev), (ctypes.c_int * k)(*den_bitrev)
        work = self._iop_work(n)
        _check(_native.lib().gmsm_fr_iop_ratio_shuffled_device(self.field, num, nb, den, db, k, n, beta.ctypes.data, d_z.data_ptr(),
                                                               work.data_ptr(), self.stream))

    def iop_ratio_copy(self, domain, d_cols, bitrev, d_sigma, beta: np.ndarray, gamma: np.ndarray, d_z):
        """d_z = the accumulating ratio of BuildRatioCopyConstraint in Lagrange Regular form; d_sigma: int64 tensor of k n entries.
        Returns once the permutation has been checked."""
        k, n = len(d_cols), domain.Cardinality
        cols = (ctypes.c_void_p * k)(*[d.data_ptr() for d in d_cols])
        br = (ctypes.c_int * k)(*bitrev)
        work = self._iop_work(n)
        _check(_native.lib().gmsm_fft_iop_ratio_copy_device(domain._h, cols, br, k, n, d_sigma.data_ptr(), beta.ctypes.data, gamma.ctypes.data,
                                                            d_z.data_ptr(), work.data_ptr(), self.stream))

    def iop_lagrange_eval(self, domain, d_c, bitrev: bool, x: np.ndarray, d_out):
        """d_out = evalLagrange of d_c (Lagrange basis on `domain`) at x"""
        work = self._iop_work(domain.Cardinality)
        _check(_native.lib().gmsm_fft_iop_lagrange_eval_device(domain._h, d_c.data_ptr(), domain.Cardinality, 1 if bitrev else 0, x.ctypes.data,
                                                               d_out.data_ptr(), work.data_ptr(), self.stream))

    def iop_evaluate(self, code: np.ndarray, out_reg: int, consts: np.ndarray, d_inputs, offsets, bitrev, n: int, out_bitrev: bool, d_r):
        """d_r = the straight-line program `code` over the inputs, one value per position (iop.Evaluate)"""
        m = len(d_inputs)
        ins = (ctypes.c_void_p * max(m, 1))(*[d.data_ptr() for d in d_inputs])
        off = np.array(list(offsets) or [0], dtype=np.uint64)
        br = (ctypes.c_int * max(m, 1))(*(list(bitrev) or [0]))
        code = np.ascontiguousarray(code, dtype=np.uint32)
        consts = np.ascontiguousarray(consts, dtype=np.uint64)
        _check(_native.lib().gmsm_fr_iop_evaluate_device(self.field, code.ctypes.data, code.shape[0], out_reg, consts.ctypes.data,
                                                         consts.shape[0], ins, off.ctypes.data, br, m, n, 1 if out_bitrev else 0,
                                                         d_r.data_ptr(), self.stream))

    def iop_divide_by_xn_minus_one(self, d_a, n: int, offset: int, bitrev: bool, inv: np.ndarray, d_out):
        """d_out[rev(i)] = a.GetCoeff(i) inv[i mod rho] (DivideByXMinusOne before its inverse FFT)"""
        inv = np.ascontiguousarray(inv, dtype=np.uint64)
        _check(_native.lib().gmsm_fr_iop_divide_by_xn_minus_one_device(self.field, d_a.data_ptr(), n, offset, 1 if bitrev else 0,
                                                                       inv.ctypes.data, inv.shape[0], d_out.data_ptr(), self.stream))


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
        _check_size(n, 2, pk.G1.shape[0])
        import torch

        with torch.cuda.device(pk.device):
            dp = _DevicePoly(pk.curve, pk.device, n)
            d_f = _device_poly(p, cp.fr_words, pk.device)
            d_h, d_fa = dp.empty(n - 1), dp.empty(1)
            dp.div(d_f, n, _reduced(point, r), d_h, d_fa)
            jac = pk._bases.MultiExpDevice(d_h, n - 1, stream=dp.stream)
            fa = d_fa.cpu().numpy().view(np.uint64)
        return OpeningProof(H=_digest(jac, pk.words), ClaimedValue=fa.copy())
    p = _host_poly(p, cp.fr_words)
    _check_size(p.shape[0], 1, pk.G1.shape[0])
    coeffs = _fr_decode(p, r)
    a = _fr_decode(point, r)[0]
    fa = _eval(coeffs, a, r)
    h = _divide_by_x_minus_a(coeffs, fa, a, r)
    # Commit(h, pk) errors on an empty h as in the reference (kzg.go:160-162): a constant polynomial cannot be opened
    H = Commit(_fr_encode(h, r), pk)
    return OpeningProof(H=H.reshape(pk.words), ClaimedValue=_fr_encode([fa], r)[0])


def Commit(p, pk: ProvingKey, *nbTasks: int) -> np.ndarray:
    """kzg.Commit (kzg.go:159-176): Digest = MultiExp(pk.G1[:len(p)], p) as an affine point.  A device polynomial (torch tensor)
    goes straight to the MultiExp on a single-device proving key."""
    words = _params(pk.curve).fr_words
    cfg = MultiExpConfig(NbTasks=nbTasks[0] if nbTasks else 0)
    if _is_device(p) and pk.device >= 0:
        n = _poly_len(p, words)
        _check_size(n, 1, pk.G1.shape[0])
        import torch

        with torch.cuda.device(pk.device):
            d = _device_poly(p, words, pk.device)
            jac = pk._bases.MultiExpDevice(d, n, cfg, stream=_stream(d.device))
        return _digest(jac, pk.words)
    p = _host_poly(p, words)
    _check_size(p.shape[0], 1, pk.G1.shape[0])
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
# batched openings at one point (kzg.go:246-420) and the verifiers
# ----------------------------------------------------------------------------------------------------------------
class ErrInvalidNbDigests(MultiExpError):
    """kzg.ErrInvalidNbDigests (kzg.go:23)"""


class ErrZeroNbDigests(MultiExpError):
    """kzg.ErrZeroNbDigests (kzg.go:24)"""


class ErrVerifyOpeningProof(MultiExpError):
    """kzg.ErrVerifyOpeningProof (kzg.go:26)"""


@dataclass
class BatchOpeningProof:
    """kzg.BatchOpeningProof{H G1Affine, ClaimedValues []fr.Element} (kzg.go:66-77)"""

    H: np.ndarray
    ClaimedValues: np.ndarray


def derive_gamma(point, digests, claimed_values, hf, curve: str, *data_transcript: bytes) -> int:
    """deriveGamma (kzg.go:531-563) over fiatshamir.Transcript (fiat-shamir/transcript.go:61-131) with the single challenge
    "gamma": H("gamma" || point || digests (RawBytes) || claimed values || extra data), read big-endian and reduced mod r
    (fr.SetBytes, fr/element.go:880-903).  `hf` is a hashlib constructor (e.g. hashlib.sha256)."""
    cp = _params(curve)
    r = cp.r
    fs = Transcript(hf, "gamma")
    fs.Bind("gamma", _fr_marshal(point, r))
    for d in digests:
        fs.Bind("gamma", g1_raw_bytes(d, curve))
    for v in np.ascontiguousarray(claimed_values, dtype=np.uint64).reshape(-1, cp.fr_words):
        fs.Bind("gamma", _fr_marshal(v, r))
    for b in data_transcript:
        fs.Bind("gamma", b)
    return _challenge(fs, "gamma", r)


def BatchOpenSinglePoint(polynomials, digests, point: np.ndarray, hf, pk: ProvingKey, *data_transcript: bytes) -> BatchOpeningProof:
    """kzg.BatchOpenSinglePoint (kzg.go:246-331): ClaimedValues[i] = f_i(point); gamma by Fiat-Shamir; the folded polynomial
    sum_i gamma^i f_i is divided by (X - point) and committed with ONE MultiExp over the resident bases.  On a single-device
    proving key the evaluations, the fold and the division run on the device: the claimed values come back in one copy for
    the transcript, the folded polynomial and its quotient never leave the device."""
    if len(digests) != len(polynomials):
        raise ErrInvalidNbDigests("number of digests is not the same as the number of polynomials")
    cp = _params(pk.curve)
    r = cp.r
    if pk.device >= 0:
        return _batch_open_device(polynomials, digests, point, hf, pk, *data_transcript)
    polys = []
    for p in polynomials:
        p = _host_poly(p, cp.fr_words)
        _check_size(p.shape[0], 1, pk.G1.shape[0])
        polys.append(_fr_decode(p, r))
    a = _fr_decode(point, r)[0]
    claimed = [_eval(f, a, r) for f in polys]
    claimed_limbs = _fr_encode(claimed, r)
    gamma = derive_gamma(point, digests, claimed_limbs, hf, pk.curve, *data_transcript)
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
    H = Commit(_fr_encode(h, r), pk)          # errors on an empty h, as in the reference
    return BatchOpeningProof(H=H.reshape(pk.words), ClaimedValues=claimed_limbs)


def _batch_open_device(polynomials, digests, point, hf, pk: ProvingKey, *data_transcript: bytes) -> BatchOpeningProof:
    import torch

    cp = _params(pk.curve)
    r, w = cp.r, cp.fr_words
    lens = []
    for p in polynomials:
        n = _poly_len(p, w)
        _check_size(n, 1, pk.G1.shape[0])
        lens.append(n)
    largest = max(lens)
    a = _reduced(point, r)
    with torch.cuda.device(pk.device):
        dp = _DevicePoly(pk.curve, pk.device, largest)
        d_polys = [_device_poly(p, w, pk.device) for p in polynomials]
        d_claimed = dp.empty(len(lens))
        for i, (d_f, n) in enumerate(zip(d_polys, lens)):
            dp.div(d_f, n, a, None, d_claimed[i * w:(i + 1) * w])
        claimed_limbs = d_claimed.cpu().numpy().view(np.uint64).reshape(-1, w).copy()
        gamma = derive_gamma(point, digests, claimed_limbs, hf, pk.curve, *data_transcript)
        _check_size(largest, 2, pk.G1.shape[0])     # the folded quotient is empty: Commit errors in the reference
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

    cp = _params(curve)
    claimed = np.ascontiguousarray(proof.ClaimedValues, dtype=np.uint64).reshape(-1, cp.fr_words)
    if len(digests) != claimed.shape[0]:
        raise ErrInvalidNbDigests("number of digests is not the same as the number of polynomials")
    r = cp.r
    gamma = derive_gamma(point, digests, claimed, hf, curve, *data_transcript)
    gam = [1]
    for _ in range(1, len(digests)):
        gam.append(gam[-1] * gamma % r)
    vals = _fr_decode(claimed, r)
    folded_eval = sum(v * g for v, g in zip(vals, gam)) % r
    aff_cls = curve_package(_curve(curve))[0]
    pts = np.ascontiguousarray(np.stack([np.asarray(d, dtype=np.uint64).reshape(-1) for d in digests]))
    folded_digest = aff_cls().MultiExp(pts, _fr_encode(gam, r), MultiExpConfig()).limbs
    return OpeningProof(H=np.array(proof.H, dtype=np.uint64), ClaimedValue=_fr_encode([folded_eval], r)[0]), folded_digest


def decode_g1_points(curve: str, data: bytes, n: int, raw: bool = False, check_on_curve: bool = True) -> np.ndarray:
    """bulk G1Affine.SetBytes on the GPU (gmsm_g1_decode, csrc/decode.cu): n points of a homogeneous stream -> (n, words) uint64
    in Go memory layout.  Raises MultiExpError with the reference's message and the index of the first invalid point."""
    g = GROUPS[_g1_name(curve)]
    words = 2 * g.words
    per = 8 * words if raw else 4 * words
    if len(data) < n * per:
        raise EOFError("short buffer")      # io.ErrShortBuffer
    buf = np.frombuffer(data, dtype=np.uint8, count=n * per)
    out = np.zeros((n, words), dtype=np.uint64)
    _check(_native.lib().gmsm_g1_decode(g.id, buf.ctypes.data, n, 1 if raw else 0, 1 if check_on_curve else 0, out.ctypes.data))
    return out


# ----------------------------------------------------------------------------------------------------------------
# bulk point (de)serialisation on the GPU (csrc/decode.cu): G2Affine.setBytes, and G1Affine / G2Affine Bytes and RawBytes
# (marshal.go:801-846, :1051-1216), with the slice framing of Encoder / Decoder (a big-endian uint32 count, then the points,
# marshal.go:220-350, :533-580)
# ----------------------------------------------------------------------------------------------------------------
def _g2_group(curve: str):
    """the Group of a curve's G2 (named with or without "_g2"); ValueError for the bls24 curves, whose G2 is over Fp4"""
    name = curve if curve.endswith("_g2") else curve + "_g2"
    if _curve(name) not in CURVE_PARAMS:
        raise ValueError("unknown pairing curve %r" % curve)
    if name not in GROUPS:
        raise ValueError("%s has no G2 in this engine (its G2 is over Fp4)" % _curve(name))
    return GROUPS[name]


def _point_group(group: str):
    """the Group of a G1 or G2 group name of a pairing curve ("bn254_g1", "bls12381_g2", ...)"""
    if group.endswith("_g2"):
        return _g2_group(group)
    if _curve(group) not in CURVE_PARAMS:
        raise ValueError("not a pairing curve: %r" % group)
    return GROUPS[_g1_name(group)]


def _point_bytes(g, raw: bool) -> int:
    """bytes of one encoded point: a coordinate (Bytes) or two (RawBytes)"""
    return (2 if raw else 1) * 8 * g.words


def _decode(fn_host: str, fn_dev: str, g, data, n: int, raw: bool, check_on_curve: bool):
    words = 2 * g.words
    per = _point_bytes(g, raw)
    L = _native.lib()
    if _is_device(data):
        import torch

        if not data.is_cuda or data.dtype != torch.uint8 or not data.is_contiguous():
            raise ValueError("device bytes must be a contiguous torch.uint8 CUDA tensor")
        if data.numel() < n * per:
            raise EOFError("short buffer")
        out = torch.empty(n * words, dtype=torch.int64, device=data.device)
        err = torch.empty(1, dtype=torch.int64, device=data.device)
        with torch.cuda.device(data.device):
            _check(getattr(L, fn_dev)(g.id, data.data_ptr(), n, 1 if raw else 0, 1 if check_on_curve else 0, out.data_ptr(),
                                      err.data_ptr(), _stream(data.device)))
            first = int(err.cpu().numpy().view(np.uint64)[0])
        if first != (1 << 64) - 1:
            raise MultiExpError("point %d: %s" % (first >> 8, _DECODE_MESSAGES.get(first & 0xFF, "decode error")))
        return out.view(n, words)
    if len(data) < n * per:
        raise EOFError("short buffer")      # io.ErrShortBuffer
    buf = np.frombuffer(data, dtype=np.uint8, count=n * per)
    out = np.zeros((n, words), dtype=np.uint64)
    _check(getattr(L, fn_host)(g.id, buf.ctypes.data, n, 1 if raw else 0, 1 if check_on_curve else 0, out.ctypes.data))
    return out


# the decoder's error codes (decode_kernels.cuh) -> the reference's messages, for the device entry's first-error word
_DECODE_MESSAGES = {1: "invalid infinity point encoding", 2: "invalid fp.Element encoding",
                    3: "invalid compressed coordinate: square root doesn't exist", 4: "invalid point: subgroup check failed",
                    5: "invalid point encoding"}


def decode_g2_points(curve: str, data, n: int, raw: bool = False, check_on_curve: bool = True):
    """bulk G2Affine.setBytes without the subgroup check on the GPU (gmsm_g2_decode): n points of a homogeneous stream -> (n,
    words) uint64 in Go memory layout ({A0, A1} per Fp2 coordinate).  `data` may be a contiguous torch.uint8 CUDA tensor: the
    points are then decoded on its device, on the current stream, into a torch.int64 tensor (n, words).  Raises MultiExpError
    with the reference's message and the index of the first invalid point; ValueError for bls24-315 / bls24-317."""
    g = _g2_group(curve)
    return _decode("gmsm_g2_decode", "gmsm_g2_decode_device", g, data, n, raw, check_on_curve)


def _encode(g, points, raw: bool):
    words = 2 * g.words
    per = _point_bytes(g, raw)
    L = _native.lib()
    if _is_device(points):
        import torch

        if not points.is_cuda or points.dtype != torch.int64 or not points.is_contiguous() or points.numel() % words:
            raise ValueError("device points must be a contiguous torch.int64 CUDA tensor of (n, %d) words" % words)
        n = points.numel() // words
        out = torch.empty(max(n * per, 4), dtype=torch.uint8, device=points.device)
        with torch.cuda.device(points.device):
            _check(L.gmsm_points_encode_device(g.id, points.data_ptr(), n, 1 if raw else 0, out.data_ptr(), _stream(points.device)))
        return out[:n * per]
    pts = np.ascontiguousarray(points, dtype=np.uint64).reshape(-1, words)
    out = np.empty(max(pts.shape[0] * per, 1), dtype=np.uint8)
    _check(L.gmsm_points_encode(g.id, pts.ctypes.data, pts.shape[0], 1 if raw else 0, out.ctypes.data))
    return out[:pts.shape[0] * per].tobytes()


def encode_g1_points(curve: str, points, raw: bool = False):
    """G1Affine.Bytes (raw=False) or RawBytes (raw=True) of every point, on the GPU (gmsm_points_encode): (n, words) uint64 in Go
    memory layout -> the n encodings back to back (what Encoder writes after the slice length).  A torch.int64 CUDA tensor is
    encoded on its device, on the current stream, into a torch.uint8 tensor."""
    return _encode(_point_group(_g1_name(curve)), points, raw)


def encode_g2_points(curve: str, points, raw: bool = False):
    """the G2 twin of encode_g1_points (wire order X.A1 || X.A0 (|| Y.A1 || Y.A0)); ValueError for bls24-315 / bls24-317"""
    return _encode(_g2_group(curve), points, raw)


def write_points(w, group: str, points, raw: bool = False) -> int:
    """Encoder.Encode of a []G1Affine / []G2Affine (RawEncoding when raw): big-endian uint32 count, then the encoded points.
    `group`: "<curve>_g1" or "<curve>_g2".  Returns the bytes written."""
    g = _point_group(group)
    words = 2 * g.words
    n = (points.numel() if _is_device(points) else np.asarray(points).size) // words
    if n >= 1 << 32:
        raise ValueError("too many points for a uint32 slice length")
    body = _encode(g, points, raw)
    if _is_device(body):
        body = body.cpu().numpy().tobytes()
    w.write(struct.pack(">I", n))
    w.write(body)
    return 4 + len(body)


def read_points(r, group: str, check_on_curve: bool = False, device=None):
    """Decoder.Decode of a []G1Affine / []G2Affine with NoSubgroupChecks: a big-endian uint32 count, then the points, whose
    kind (Bytes or RawBytes) is read from the first point's flags; the stream must be homogeneous (a point of the other kind is
    "invalid point encoding").  check_on_curve=True also checks raw points against the curve equation, which the reference's
    NoSubgroupChecks path skips.  -> (n, words) uint64 in Go memory layout (device=None), else decoded on cuda:device into a
    torch.int64 tensor (the bytes are uploaded once)."""
    return _read_points(r, group, check_on_curve, device)[0]


def _read_points(r, group: str, check_on_curve: bool, device):
    """read_points -> (points, bytes read)"""
    g = _point_group(group)
    hdr = r.read(4)
    if len(hdr) != 4:
        raise EOFError("unexpected EOF")
    (n,) = struct.unpack(">I", hdr)
    if n == 0:
        if device is not None:
            import torch

            return torch.empty((0, 2 * g.words), dtype=torch.int64, device=torch.device("cuda", device)), 4
        return np.zeros((0, 2 * g.words), dtype=np.uint64), 4
    first = r.read(1)
    if len(first) != 1:
        raise EOFError("unexpected EOF")
    f = _params(g.curve).flags

    def is_raw(byte: int) -> bool:       # !isCompressed (marshal.go:409-418)
        m = byte & f["mask"]
        return m == f["unc"] or (f["unc_inf"] is not None and m == f["unc_inf"])

    raw = is_raw(first[0])
    per = _point_bytes(g, raw)
    rest = r.read(n * per - 1)
    data = first + rest
    if len(data) != n * per:
        # a raw stream holding compressed points is shorter than n raw strides: name the first point of the other kind, as the
        # decoder does for a stream of the right length, before calling the stream short
        for i in range(len(data) // per):
            if is_raw(data[i * per]) != raw:
                raise MultiExpError("point %d: invalid point encoding" % i)
        raise EOFError("unexpected EOF")
    fns = ("gmsm_g2_decode", "gmsm_g2_decode_device") if group.endswith("_g2") else ("gmsm_g1_decode", "gmsm_g1_decode_device")
    if device is not None:
        import torch

        data = torch.frombuffer(bytearray(data), dtype=torch.uint8).to(torch.device("cuda", device))
    return _decode(fns[0], fns[1], g, data, n, raw, check_on_curve), 4 + n * per


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
    words = 2 * GROUPS[cname].words
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
            _check(L.gmsm_g1_to_lagrange_device(cid, coeffs.data_ptr(), n, out.data_ptr(), work.data_ptr(), _stream(coeffs.device)))
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
    from .fft import DIF

    words = _params(pk.curve).fr_words
    ev = np.ascontiguousarray(evals, dtype=np.uint64).reshape(-1, words)      # host evaluations only
    if ev.shape[0] != domain.Cardinality:
        raise MultiExpError("len(a) must equal the domain cardinality")
    _check_size(ev.shape[0], 1, pk.G1.shape[0])
    d = _device_poly(ev, words, domain.device)          # a fresh upload: transformed in place below
    st = _stream(domain.device)
    domain.fft_device(d, True, DIF, False, st)          # natural in, bit-reversed out
    domain.bit_reverse_device(d, st)
    return _digest(pk._bases.MultiExpDevice(d, ev.shape[0], stream=st), pk.words)


# ----------------------------------------------------------------------------------------------------------------
# verifiers (kzg.go:207-240, 385-500) on the GPU pairing (pairing.py).  The reference checks with PairingCheckFixedQ on the
# precomputed lines of vk.G2; the general PairingCheck used here gives the same accept / reject for any input, because the two
# Miller loops differ only by factors that the final exponentiation removes.
# ----------------------------------------------------------------------------------------------------------------
@dataclass
class VerifyingKey:
    """kzg.VerifyingKey (kzg.go:53-58): G2[0] the G2 generator, G2[1] = [alpha]G2, G1 the G1 generator (Go memory layout)"""

    curve: str
    G2: np.ndarray
    G1: np.ndarray


def _g1_msm(curve: str, points, scalars: list) -> np.ndarray:
    """one affine G1 point: the MultiExp of `points` by the integers `scalars` (mod r)"""
    from .multiexp import curve_package

    cp = _params(curve)
    pts = np.ascontiguousarray(np.stack([np.asarray(p, dtype=np.uint64).reshape(-1) for p in points]))
    return curve_package(_curve(curve))[0]().MultiExp(pts, _fr_encode([k % cp.r for k in scalars], cp.r), MultiExpConfig()).limbs


def _pairing_check(vk: VerifyingKey, a: np.ndarray, b: np.ndarray) -> bool:
    """e(a, G2[0]) e(b, G2[1]) == 1"""
    from . import pairing

    g2 = np.ascontiguousarray(vk.G2, dtype=np.uint64).reshape(2, -1)
    P = np.ascontiguousarray(np.stack([np.asarray(a, dtype=np.uint64).reshape(-1), np.asarray(b, dtype=np.uint64).reshape(-1)]))
    return pairing.PairingCheck(_curve(vk.curve), P, g2)


def Verify(commitment, proof: OpeningProof, point, vk: VerifyingKey) -> None:
    """kzg.Verify (kzg.go:207-240): e([f(a) - a H(alpha) - f(alpha)]G1, G2) e([H(alpha)]G1, [alpha]G2) == 1, else
    ErrVerifyOpeningProof.  The G1 combination is one MultiExp."""
    r = _params(vk.curve).r
    fa = _fr_decode(proof.ClaimedValue, r)[0]
    a = _fr_decode(point, r)[0]
    total = _g1_msm(vk.curve, [vk.G1, proof.H, commitment], [fa, -a, -1])
    if not _pairing_check(vk, total, proof.H):
        raise ErrVerifyOpeningProof("can't verify opening proof")


def BatchVerifySinglePoint(digests, proof: BatchOpeningProof, point, hf, vk: VerifyingKey, *data_transcript: bytes) -> None:
    """kzg.BatchVerifySinglePoint (kzg.go:385-400): FoldProof, then Verify of the folded proof"""
    folded_proof, folded_digest = FoldProof(digests, proof, point, hf, vk.curve, *data_transcript)
    Verify(folded_digest, folded_proof, point, vk)


def BatchVerifyMultiPoints(digests, proofs, points, vk: VerifyingKey) -> None:
    """kzg.BatchVerifyMultiPoints (kzg.go:405-500): with lambda_0 = 1 and random lambda_i (secrets), checks
    e(sum lambda_i (C_i - [f_i(a_i)]G1 + [a_i]H_i), G2) e(-sum lambda_i H_i, [alpha]G2) == 1.  Each G1 side is one MultiExp."""
    import secrets

    if len(digests) != len(proofs) or len(digests) != len(points):
        raise ErrInvalidNbDigests("number of digests is not the same as the number of polynomials")
    if len(digests) == 0:
        raise ErrZeroNbDigests("number of digests is zero")
    if len(digests) == 1:
        return Verify(digests[0], proofs[0], points[0], vk)
    r = _params(vk.curve).r
    lam = [1] + [secrets.randbelow(r) for _ in range(len(digests) - 1)]
    evals = [_fr_decode(p.ClaimedValue, r)[0] for p in proofs]
    a = [_fr_decode(x, r)[0] for x in points]
    hs = [p.H for p in proofs]
    folded_eval = sum(l * e for l, e in zip(lam, evals)) % r
    folded_digests = _g1_msm(vk.curve, list(digests) + hs + [vk.G1], lam + [l * x for l, x in zip(lam, a)] + [-folded_eval])
    folded_quotients = _g1_msm(vk.curve, hs, [-l for l in lam])
    if not _pairing_check(vk, folded_digests, folded_quotients):
        raise ErrVerifyOpeningProof("can't verify opening proof")
