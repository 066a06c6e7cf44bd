"""fflonk (ecc/bn254/fflonk/fflonk.go; the fflonk packages of the other six pairing curves are the same generated code): packs of t
polynomials committed as one interleave F = sum_{i<t} X^i p_i(X^t) (Fold, FoldAndCommit) and opened at the powers s^t of a point set
through one SHPLONK proof on the extended set {s omega^k} (BatchOpen).  On a single-device proving key the interleave is never
built for the opening: shplonk.open_packs divides the p_i themselves and interleaves their quotients (see shplonk.py)."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from . import kzg, shplonk
from .curves import _fr_decode, _fr_encode, _params
from .multiexp import MultiExpError


class ErrRootsOne(MultiExpError):
    """fflonk.ErrRootsOne (fflonk.go:20)"""


class ErrNbPolynomialsNbPoints(MultiExpError):
    """fflonk.ErrNbPolynomialsNbPoints (fflonk.go:21)"""


@dataclass
class OpeningProof:
    """fflonk.OpeningProof{SOpeningProof shplonk.OpeningProof; ClaimedValues [][][]fr.Element} (fflonk.go:31-39):
    ClaimedValues[j][i] is a (len(points[j]), fr.Limbs) array of p[j][i] on the s^t of points[j], zero for t > i >= len(p[j])"""

    SOpeningProof: shplonk.OpeningProof
    ClaimedValues: list


def _next_divisor_r_minus_one(i: int, r: int) -> int:
    """getNextDivisorRMinusOne (fflonk.go:234-252): the smallest t >= i dividing r - 1, at most 100 trials"""
    if i <= 0:
        raise ValueError("an empty pack has no divisor of r-1 (the reference divides by zero)")
    trials = 100
    while (r - 1) % i != 0 and trials > 0:
        i += 1
        trials -= 1
    if trials == 0:
        raise ValueError("did not find any divisor of r-1")
    return i


def _ith_root_one(i: int, curve: str) -> int:
    """getIthRootOne (fflonk.go:213-230): GeneratorFullMultiplicativeGroup^((r - 1) / i)"""
    cp = _params(curve)
    r = cp.r
    if (r - 1) % i != 0:
        raise ErrRootsOne("fr does not contain all the t-th roots of 1")
    return pow(cp.mult_gen, (r - 1) // i, r)


def _extend_set(points: list, t: int, curve: str) -> list:
    """extendSet (fflonk.go:255-271): [p0, omega p0, .., omega^(t-1) p0, p1, ...]"""
    r = _params(curve).r
    omega = _ith_root_one(t, curve)
    out = []
    for p in points:
        x = p
        for _ in range(t):
            out.append(x)
            x = x * omega % r
    return out


def Fold(p, curve: str) -> np.ndarray:
    """Fold (fflonk.go:52-71) on the host: F[j t + i] = p[i][j], t = getNextDivisorRMinusOne(len(p)), t * max len(p[i])
    coefficients as a (n, fr.Limbs) uint64 array"""
    cp = _params(curve)
    w = cp.fr_words
    t = _next_divisor_r_minus_one(len(p), cp.r)
    hp = [kzg._host_poly(x, w) for x in p]
    out = np.zeros((t * max(x.shape[0] for x in hp), w), dtype=np.uint64)
    for i, x in enumerate(hp):
        out[i::t][:x.shape[0]] = x
    return out


def FoldAndCommit(p, pk: kzg.ProvingKey, *nbTasks: int) -> np.ndarray:
    """FoldAndCommit (fflonk.go:43-47): kzg.Commit(Fold(p), pk).  On a single-device key the interleave is one
    gmsm_fr_poly_lincomb_device (stride t) into device memory that feeds the MultiExp."""
    cp = _params(pk.curve)
    w = cp.fr_words
    if pk.device < 0:
        return kzg.Commit(Fold(p, pk.curve), pk, *nbTasks)
    import torch

    t = _next_divisor_r_minus_one(len(p), cp.r)
    lens = [kzg._poly_len(x, w) for x in p]
    size = t * max(lens)
    kzg._check_size(size, 1, pk.G1.shape[0])
    with torch.cuda.device(pk.device):
        dp = kzg._DevicePoly(pk.curve, pk.device, 0)
        ins = [(kzg._device_poly(x, w, pk.device), n, i) for i, (x, n) in enumerate(zip(p, lens)) if n]
        d_F = dp.empty(size)
        dp.lincomb([d for d, _, _ in ins], [n for _, n, _ in ins], _fr_encode([1] * len(ins), cp.r), [t] * len(ins),
                   [i for _, _, i in ins], d_F, size)
        return kzg.Commit(d_F, pk, *nbTasks)


def BatchOpen(p, digests, points, hf, pk: kzg.ProvingKey, *dataTranscript: bytes) -> OpeningProof:
    """BatchOpen (fflonk.go:77-141): pack p[j] (a list of polynomials: numpy limbs or torch CUDA int64 tensors on the key's device,
    left unmodified) is opened on the powers s^t of points[j]; digests[j] = FoldAndCommit(p[j])."""
    if len(p) != len(points):
        raise ErrNbPolynomialsNbPoints("the number of packs of polynomials should be the same as the number of pack of points")
    cp = _params(pk.curve)
    r, w = cp.r, cp.fr_words
    ts = [_next_divisor_r_minus_one(len(pack), r) for pack in p]
    base = [shplonk._decode_points(S, r) for S in points]
    ext = [_extend_set(S, t, pk.curve) for S, t in zip(base, ts)]
    if len(digests) != len(p):
        raise shplonk.ErrInvalidNumberOfDigests("number of digests should be equal to the number of polynomials")
    if not p:
        raise ValueError("fflonk.BatchOpen needs at least one pack")
    if pk.device < 0:
        values = [[[shplonk._eval(_fr_decode(kzg._host_poly(f, w), r), pow(s, t, r), r) for s in S] for f in pack]
                  for pack, S, t in zip(p, base, ts)]
        folded = [_fr_decode(Fold(pack, pk.curve), r) for pack in p]
        W, WPrime, claimed, _, _ = shplonk.batch_open_host(folded, ext, digests, hf, pk.curve, shplonk._host_commit(pk), *dataTranscript)
    else:
        W, WPrime, claimed, values = shplonk.open_packs(p, base, ts, ext, digests, hf, pk, dataTranscript)
    sproof = shplonk.OpeningProof(W=W, WPrime=WPrime, ClaimedValues=[_fr_encode(v, r).reshape(-1, w) for v in claimed])
    outer = [[_fr_encode(v, r).reshape(-1, w) for v in vals] + [np.zeros((len(S), w), dtype=np.uint64) for _ in range(t - len(vals))]
             for vals, S, t in zip(values, base, ts)]
    return OpeningProof(SOpeningProof=sproof, ClaimedValues=outer)
