"""plookup.ProveLookupVector and ProveLookupTables (ecc/bn254/fr/plookup/vector.go:345-550 and table.go:52-166; the plookup packages
of the other six pairing curves are the same generated code): a proof that the values of f are in the table t, and its
multi-column form, with KZG commitments of the interpolations, of the accumulation polynomial z and of the quotient.

On a single-device proving key everything from the inputs to the last MultiExp stays on the device: the two sorts
(gmsm_fr_sort_device, an LSD radix sort over the canonical bytes), the FFTs (fft.Domain.fft_device), the accumulation polynomial
(gmsm_fr_plookup_accumulate_device: a tile batch inversion and the permutation's prefix product), the quotient numerator on the coset
of size 2s (gmsm_fft_plookup_numerator_device) and the commitments and openings of kzg.py on device tensors.  Only the inputs (when
they are host arrays), the digests, the opening proofs and the claimed values cross PCIe.  A proving key sharded over several GPUs
(device = -1) runs the same Fr work on the current device and commits and opens through kzg's host entry points, which gives the
same proof.  As in the reference, f is not checked to lie in t: a vector outside the table still proves (and fails to verify).
VerifyLookupVector and VerifyLookupTables need pairings and are not built."""
from __future__ import annotations

import hashlib
from dataclasses import dataclass

import numpy as np

from . import fft, kzg, permutation
from .curves import _challenge, _curve, _fr_decode, _fr_encode, _params
from .fft import DIF, DIT
from .kzg import g1_raw_bytes
from .multiexp import MultiExpError
from .transcript import Transcript


class ErrIncompatibleSize(MultiExpError):
    """plookup.ErrIncompatibleSize (table.go:23)"""


@dataclass
class ProofLookupVector:
    """plookup.ProofLookupVector (vector.go:28-44): the digests h1, h2, t, z, f, h are G1Affine limbs, g the small domain's generator
    (fr.Element limbs); BatchedProof opens h1, h2, t, z, f, h at nu, BatchedProofShifted opens h1, h2, t, z at nu g"""

    size: int
    g: np.ndarray
    h1: np.ndarray
    h2: np.ndarray
    t: np.ndarray
    z: np.ndarray
    f: np.ndarray
    h: np.ndarray
    BatchedProof: kzg.BatchOpeningProof
    BatchedProofShifted: kzg.BatchOpeningProof


@dataclass
class ProofLookupTables:
    """plookup.ProofLookupTables (table.go:29-42): the digests of the rows of f and t, the lookup proof of the folded vectors and
    the permutation proof that ties the folded t to its sorted copy"""

    fs: list
    ts: list
    foldedProof: ProofLookupVector
    permutationProof: permutation.Proof


def _empty():
    return ValueError("f and t must not be empty")


def ProveLookupVector(pk: kzg.ProvingKey, f, t) -> ProofLookupVector:
    """plookup.ProveLookupVector: f and t are numpy (n, fr.Limbs) arrays or torch CUDA int64 tensors in the same layout (on the key's
    device for a single-device key), of any lengths >= 1, left unmodified.  The work is ordered on the current stream of the
    device."""
    import torch

    w = _params(pk.curve).fr_words
    nf, nt = kzg._poly_len(f, w), kzg._poly_len(t, w)
    if nf == 0 or nt == 0:             # the reference panics on f[len(f)-1]
        raise _empty()
    dev = pk.device if pk.device >= 0 else torch.cuda.current_device()
    curve = _curve(pk.curve)
    d = fft.NewDomain(curve, nf + 1 if nt <= nf else nt, device=dev)
    try:
        with torch.cuda.device(dev):
            return _prove_vector(pk, d, f, t, nf, nt, curve, dev)
    finally:
        d.close()


def _padded(dp, src, n, s):
    """the first n elements of src followed by copies of its last one, s elements (vector.go:374-385)"""
    w = dp.words
    out = dp.empty(s)
    out[:n * w].copy_(src[:n * w])
    if s > n:
        out[n * w:].view(s - n, w).copy_(src[(n - 1) * w:n * w].view(1, w).expand(s - n, w))
    return out


def _prove_vector(pk, d, f, t, nf, nt, curve, dev):
    cp = _params(curve)
    r, w = cp.r, cp.fr_words
    s = d.Cardinality
    dp = kzg._DevicePoly(curve, dev, 2 * s)
    st = dp.stream
    sharded = pk.device < 0

    def commit(p):
        return kzg.Commit(kzg._host_poly(p, w) if sharded else p, pk)

    def coeffs(v):                         # FFTInverse(DIF) + BitReverse of a copy
        c = v.clone()
        d.fft_device(c, True, DIF, False, st)
        d.bit_reverse_device(c, st)
        return c

    lf = _padded(dp, kzg._device_poly(f, w, dev), nf, s)
    lt = _padded(dp, kzg._device_poly(t, w, dev), nt, s)
    dp.sort(lt, s, lt)
    ct, cf = coeffs(lt), coeffs(lf)
    T = commit(ct)
    F = commit(cf)
    # f sorted by t: sort(lt || lf[:s-1]) split into the overlapping h1 = [0, s) and h2 = [s-1, 2s-1)
    h = dp.empty(2 * s - 1)
    h[:s * w].copy_(lt)
    h[s * w:].copy_(lf[:(s - 1) * w])
    dp.sort(h, 2 * s - 1, h)
    lh1, lh2 = h[:s * w], h[(s - 1) * w:]
    ch1, ch2 = coeffs(lh1), coeffs(lh2)
    H1 = commit(ch1)
    H2 = commit(ch2)
    fs = Transcript(hashlib.sha256, "beta", "gamma", "alpha", "nu")
    for p in (T, F, H1, H2):
        fs.Bind("beta", g1_raw_bytes(p, curve))
    beta = _fr_encode([_challenge(fs, "beta", r)], r)[0]
    gamma = _fr_encode([_challenge(fs, "gamma", r)], r)[0]
    cz = dp.empty(s)
    dp.plookup_accumulate(lf, lt, lh1, lh2, s, beta, gamma, cz)
    del h, lh1, lh2
    d.fft_device(cz, True, DIF, False, st)
    d.bit_reverse_device(cz, st)
    Z = commit(cz)
    # the five coset evaluations on the domain of size 2s (bit-reversed), the numerator, and the quotient's coefficients
    db = fft.NewDomain(curve, 2 * s, device=dev)
    try:
        big = []
        for c in (cz, ch1, ch2, ct, cf):
            v = dp.torch.zeros(2 * s * w, dtype=dp.torch.int64, device=dp.dev)
            v[:s * w].copy_(c)
            db.fft_device(v, False, DIF, True, st)
            big.append(v)
        fs.Bind("alpha", g1_raw_bytes(Z, curve))
        alpha = _fr_encode([_challenge(fs, "alpha", r)], r)[0]
        ch = dp.empty(2 * s)
        dp.plookup_numerator(db, *big, beta, gamma, alpha, ch)
        del big
        db.fft_device(ch, True, DIT, True, st)
    finally:
        db.close()
    Hd = commit(ch)
    fs.Bind("nu", g1_raw_bytes(Hd, curve))
    nu = _challenge(fs, "nu", r)
    polys = [ch1, ch2, ct, cz, cf, ch]
    if sharded:
        polys = [kzg._host_poly(p, w) for p in polys]
    digests = [H1, H2, T, Z, F, Hd]
    batched = kzg.BatchOpenSinglePoint(polys, digests, _fr_encode([nu], r)[0], hashlib.sha256, pk)
    gen = _fr_decode(d.Generator, r)[0]
    shifted = kzg.BatchOpenSinglePoint(polys[:4], digests[:4], _fr_encode([nu * gen % r], r)[0], hashlib.sha256, pk)
    return ProofLookupVector(size=s, g=d.Generator.copy(), h1=H1, h2=H2, t=T, z=Z, f=F, h=Hd, BatchedProof=batched,
                             BatchedProofShifted=shifted)


def ProveLookupTables(pk: kzg.ProvingKey, f, t) -> ProofLookupTables:
    """plookup.ProveLookupTables: f and t are lists of rows (each as ProveLookupVector takes them); the rows of f must have one
    length and the rows of t one length.  The rows are left unmodified."""
    import torch

    w = _params(pk.curve).fr_words
    if len(f) == 0 or len(t) == 0:     # the reference panics on f[0]
        raise _empty()
    if len(f) != len(t):
        raise ErrIncompatibleSize("the tables in f and t are not of the same size")
    nf = [kzg._poly_len(row, w) for row in f]
    nt = [kzg._poly_len(row, w) for row in t]
    if any(n != nf[0] for n in nf) or any(n != nt[0] for n in nt):
        raise ErrIncompatibleSize("the tables in f and t are not of the same size")
    if nf[0] == 0 or nt[0] == 0:       # the reference panics on f[i][len(f[i])-1]
        raise _empty()
    dev = pk.device if pk.device >= 0 else torch.cuda.current_device()
    curve = _curve(pk.curve)
    d = fft.NewDomain(curve, max(nf[0] + 1, nt[0]), device=dev)
    try:
        with torch.cuda.device(dev):
            return _prove_tables(pk, d, f, t, nf[0], nt[0], curve, dev)
    finally:
        d.close()


def _prove_tables(pk, d, f, t, nf, nt, curve, dev):
    cp = _params(curve)
    r, w = cp.r, cp.fr_words
    nc = d.Cardinality
    rows = len(f)
    dp = kzg._DevicePoly(curve, dev, nc)
    st = dp.stream
    sharded = pk.device < 0
    lfs, lts, Fs, Ts = [], [], [], []
    for i in range(rows):                  # commits in the reference's order: f[0], t[0], f[1], t[1], ...
        for src, n, ls, ds in ((f[i], nf, lfs, Fs), (t[i], nt, lts, Ts)):
            lv = _padded(dp, kzg._device_poly(src, w, dev), n, nc)
            c = lv.clone()
            d.fft_device(c, True, DIF, False, st)
            d.bit_reverse_device(c, st)
            ds.append(kzg.Commit(kzg._host_poly(c, w) if sharded else c, pk))
            ls.append(lv)
    fs = Transcript(hashlib.sha256, "lambda")
    for p in Fs + Ts:
        fs.Bind("lambda", g1_raw_bytes(p, curve))
    lam = _challenge(fs, "lambda", r)
    # the Horner fold sum_j lambda^j row_j (table.go:141-150) as one linear combination with [1, lambda, lambda^2, ...]
    scalars = _fr_encode([pow(lam, j, r) for j in range(rows)], r)
    foldedf, foldedt = dp.empty(nc), dp.empty(nc)
    for rows_, out in ((lfs, foldedf), (lts, foldedt)):
        dp.lincomb(rows_, [nc] * rows, scalars, [1] * rows, [0] * rows, out, nc)
    del lfs, lts
    sorted_t = dp.empty(nc)
    dp.sort(foldedt, nc, sorted_t)
    perm = permutation.Prove(pk, foldedt, sorted_t)
    del sorted_t
    folded = ProveLookupVector(pk, foldedf[:(nc - 1) * w], foldedt)
    return ProofLookupTables(fs=Fs, ts=Ts, foldedProof=folded, permutationProof=perm)
