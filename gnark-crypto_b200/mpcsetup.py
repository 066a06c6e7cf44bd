"""mpcsetup (ecc/bn254/mpcsetup/mpcsetup.go; the mpcsetup packages of the other pairing curves are the same generated code): the
point updates of a trusted-setup contribution and the linear combinations that check one, for the seven pairing curves.

  * UpdateMonomialsG1 / UpdateMonomialsG2 (mpcsetup.go:365-381): A[i] <- [r^i] A[i], in place;
  * ScaleG1 / ScaleG2: A[i] <- [c r^i] A[i], in place -- the slice loop of UpdateValues (:64-81) for r = 1 and the alpha tau^i /
    beta tau^i slices of a powers-of-tau contribution for c = alpha (beta);
  * LinearCombinationsG1 / LinearCombinationsG2 (linearCombinationsG1 / G2, :396-447, :489-540): (truncated, shifted) of
    SameRatioMany, whose final pairing check stays with the caller.
The updates run on the GPU, one variable-base scalar multiplication per point (gmsm_scale_powers, csrc/mpc_kernels.cuh); the
linear combinations are the reference's two MultiExps, the large one on the device.

Groups: G1 of bn254, bls12-381, bls12-377, bls24-315, bls24-317, bw6-633 and bw6-761, and G2 of all but bls24-315 / bls24-317 (their
G2 is over Fp4, which the engine does not have: the G2 functions raise ValueError for them).  Points are (n, 2 * words) uint64
numpy arrays in the reference's memory layout (Montgomery limbs, infinity = zeroes), or contiguous torch.int64 CUDA tensors in the
same layout, which are updated on their own device, on its current stream.  Scalars are fr.Elements: fr.Limbs uint64 Montgomery
limbs, reduced (an unreduced one raises MultiExpError).  Results are in the affine normal form of BatchJacobianToAffineG1."""
from __future__ import annotations

import numpy as np

from . import _native
from .curves import GROUPS, _fr_decode, _fr_encode
from .kzg import _is_device, _stream
from .multiexp import Engine, _check

PAIRING_CURVES = ("bn254", "bls12381", "bls12377", "bls24315", "bls24317", "bw6633", "bw6761")


def _group(curve: str, g: str):
    """(name, Group) of G1 or G2 of a pairing curve"""
    if curve not in PAIRING_CURVES:
        raise ValueError("unknown pairing curve %r" % curve)
    name = "%s_%s" % (curve, g)
    if name not in GROUPS:
        raise ValueError("%s has no %s in this engine (its G2 is over Fp4)" % (curve, g.upper()))
    return name, GROUPS[name]


def _scalar(grp, x, what: str) -> np.ndarray:
    a = np.ascontiguousarray(x, dtype=np.uint64).reshape(-1)
    if a.size != grp.scalar_words:
        raise ValueError("%s: an fr.Element is %d uint64 limbs, got %d" % (what, grp.scalar_words, a.size))
    return a


def _check_points(grp, A) -> int:
    """the number of points of A, which must be updatable in place"""
    words = 2 * grp.words
    if _is_device(A):
        import torch

        if not A.is_cuda or A.dtype != torch.int64 or not A.is_contiguous() or A.numel() % words:
            raise ValueError("device points must be a contiguous torch.int64 CUDA tensor of (n, %d) words" % words)
        return A.numel() // words
    if not isinstance(A, np.ndarray) or A.dtype != np.uint64 or not A.flags.c_contiguous or not A.flags.writeable or A.size % words:
        raise ValueError("points must be a writable C-contiguous uint64 numpy array of (n, %d) words (updated in place)" % words)
    return A.size // words


def _scale(grp, A, first: int, n: int, c: np.ndarray, r: np.ndarray, device: int) -> None:
    """A[first + i] <- [c r^i] A[first + i] for i < n, in place"""
    if n == 0:
        return
    L = _native.lib()
    off = first * 2 * grp.words * 8
    if _is_device(A):
        import torch

        with torch.cuda.device(A.device):
            p = A.data_ptr() + off
            _check(L.gmsm_scale_powers_device(grp.id, p, n, c.ctypes.data, r.ctypes.data, p, _stream(A.device)))
        return
    p = A.ctypes.data + off
    _check(L.gmsm_scale_powers(grp.id, p, n, c.ctypes.data, r.ctypes.data, device, p))


def _update_monomials(g: str, curve: str, A, r, device: int):
    _, grp = _group(curve, g)
    n = _check_points(grp, A)
    r = _scalar(grp, r, "r")
    if n < 2:
        raise IndexError("UpdateMonomials%s: len(A) = %d, at least 2 points are needed (A[1] is updated)" % (g.upper(), n))
    _scale(grp, A, 1, n - 1, r, r, device)
    return A


def UpdateMonomialsG1(curve: str, A, r, device: int = 0):
    """UpdateMonomialsG1 (mpcsetup.go:365-381): A[i] <- [r^i] A[i] for every i, in place (A[0] is left bit-identical); returns A.
    len(A) < 2 raises IndexError, where the reference panics on A[1].  `device` is the GPU of a host array."""
    return _update_monomials("g1", curve, A, r, device)


def UpdateMonomialsG2(curve: str, A, r, device: int = 0):
    """UpdateMonomialsG2 on G2 points: A[i] <- [r^i] A[i], in place, as UpdateMonomialsG1.  The reference's UpdateMonomialsG2
    (mpcsetup.go:449-465) is declared over []G1Affine, a slip of its code generator (its body is UpdateMonomialsG1's); this one
    takes G2 points, as its name says."""
    return _update_monomials("g2", curve, A, r, device)


def _scale_all(g: str, curve: str, A, c, r, device: int):
    _, grp = _group(curve, g)
    n = _check_points(grp, A)
    c = _scalar(grp, c, "c")
    r = _fr_encode([1], grp.r)[0] if r is None else _scalar(grp, r, "r")
    _scale(grp, A, 0, n, c, r, device)
    return A


def ScaleG1(curve: str, A, c, r=None, device: int = 0):
    """A[i] <- [c r^i] A[i] for every i, in place; r = None is r = 1 (every point times c: the slice loop of UpdateValues,
    mpcsetup.go:64-81).  With c = alpha and r = tau on [tau^i]G it is the alpha tau^i slice of a powers-of-tau update.  Returns A."""
    return _scale_all("g1", curve, A, c, r, device)


def ScaleG2(curve: str, A, c, r=None, device: int = 0):
    """ScaleG1 on G2 points"""
    return _scale_all("g2", curve, A, c, r, device)


def _affine(grp, jac: np.ndarray) -> np.ndarray:
    """the engine's Jacobian result (X, Y, 1) or (0, 0, 0) as an affine point"""
    w = grp.words
    return jac[: 2 * w].copy() if jac[2 * w :].any() else np.zeros(2 * w, dtype=np.uint64)


def _host_msm(grp, pts: np.ndarray, scalars: np.ndarray) -> np.ndarray:
    out = np.zeros(3 * grp.words, dtype=np.uint64)
    pts, scalars = np.ascontiguousarray(pts), np.ascontiguousarray(scalars)
    _check(_native.lib().gmsm_multiexp(grp.id, pts.ctypes.data, scalars.ctypes.data, pts.shape[0], 0, out.ctypes.data))
    return _affine(grp, out)


def _row(a, i: int) -> np.ndarray:
    """row i of a host array or a device tensor, as a host uint64 array"""
    if _is_device(a):
        return a[i].cpu().numpy().view(np.uint64).copy()
    return np.array(a[i], dtype=np.uint64)


def _linear_combinations(g: str, curve: str, A, powers, ends):
    name, grp = _group(curve, g)
    words, fw, q = 2 * grp.words, grp.scalar_words, grp.r
    dev = _is_device(A)
    if dev:
        _check_points(grp, A)
        A2 = A.reshape(-1, words)
    else:
        A2 = np.ascontiguousarray(A, dtype=np.uint64).reshape(-1, words)
    n = A2.shape[0]
    P2 = powers.reshape(-1, fw) if _is_device(powers) else np.ascontiguousarray(powers, dtype=np.uint64).reshape(-1, fw)
    ends = [int(e) for e in ends]
    if not ends or ends[-1] != n or P2.shape[0] != n:
        raise ValueError("lengths mismatch")   # mpcsetup.go:412-414
    if len(ends) == 1 and ends[0] == 2:
        return _row(A2, 0), _row(A2, 1)
    if any(not 1 <= e <= n for e in ends):
        raise IndexError("ends %r out of range [1, %d]" % (ends, n))
    zero = [e - 1 for e in ends]
    # the large MultiExp with the last coefficient of each slice zeroed, on a copy of powers (A and powers are left unmodified)
    if dev:
        import torch

        with torch.cuda.device(A.device):
            d_pow = P2.clone() if _is_device(powers) else torch.from_numpy(P2.view(np.int64).copy()).to(A.device)
            d_pow[zero] = 0
            eng = Engine(name, n, device=A.device.index)
            try:
                truncated = _affine(grp, eng.msm_host_result(A2.reshape(-1), d_pow.reshape(-1), n))
            finally:
                eng.close()
    else:
        hp = (P2.cpu().numpy().view(np.uint64) if _is_device(powers) else P2).copy()
        hp[zero] = 0
        truncated = _host_msm(grp, A2, hp)

    # the small MultiExp (mpcsetup.go:416-444) on the few entries it reads and writes, restated statement by statement (the
    # reference's in-place updates of powers and A, and its out-of-range indices, included)
    pw, pts = {i: 0 for i in zero}, {}

    def at(i, what):
        if not 0 <= i < n:
            raise IndexError("%s[%d] out of range (len %d)" % (what, i, n))
        return i

    def P(i):
        if at(i, "powers") not in pw:
            pw[i] = _fr_decode(_row(P2, i), q)[0]
        return pw[i]

    def Pt(i):
        if at(i, "A") not in pts:
            pts[i] = _row(A2, i)
        return pts[i]

    p1 = P(1)
    r_inv_neg = (-pow(p1, -1, q)) % q if p1 else 0   # fr.Element.Inverse(0) = 0
    prev = 0
    for i, e in enumerate(ends):
        pw[at(2 * i, "powers")] = P(prev) * r_inv_neg % q
        pw[at(2 * i + 1, "powers")] = P(e - 2)
        pts[2 * i] = Pt(prev)
        pts[2 * i + 1] = Pt(e - 1)
        prev = e
    k = 2 * len(ends)
    pw[at(k, "powers")] = (-r_inv_neg) % q
    pts[k] = truncated
    shifted = _host_msm(grp, np.stack([Pt(i) for i in range(k + 1)]), _fr_encode([P(i) for i in range(k + 1)], q))
    return truncated, shifted


def LinearCombinationsG1(curve: str, A, powers, ends):
    """linearCombinationsG1 (mpcsetup.go:396-447): (truncated, shifted) as affine points, where
        truncated = sum over the slices [s, e) of ends of  powers[j] A[j],      j = s .. e - 2
        shifted   = sum over the slices [s, e) of ends of  powers[j] A[j + 1],  j = s .. e - 2
    computed as the reference computes them: one MultiExp with powers[e - 1] zeroed for truncated, then the (2 len(ends) + 1)-term
    MultiExp with the coefficients -powers[s] / powers[1], powers[e - 2] and 1 / powers[1] (fr.Element.Inverse: 1 / 0 = 0) for
    shifted, and the shortcut (A[0], A[1]) for ends = [2].  The results are therefore the reference's whatever `powers` holds.
    Unlike the reference, A and powers are left unmodified.  A: host array or device tensor (the large MultiExp then runs on its
    device); powers: (n, fr.Limbs) fr.Elements, host or device.  Raises ValueError for mismatched lengths, IndexError where the
    reference would index out of range."""
    return _linear_combinations("g1", curve, A, powers, ends)


def LinearCombinationsG2(curve: str, A, powers, ends):
    """linearCombinationsG2 (mpcsetup.go:489-540): LinearCombinationsG1 on G2 points"""
    return _linear_combinations("g2", curve, A, powers, ends)
