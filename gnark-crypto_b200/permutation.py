"""permutation.Prove (ecc/bn254/fr/permutation/permutation.go:124-262; the permutation packages of the other six pairing curves are
the same generated code): a proof that the vectors t1 and t2 are permutations of each other, with KZG commitments of their
interpolations, of the accumulation polynomial Z and of the quotient.

On a single-device proving key everything from the inputs to the last MultiExp stays on the device: the five FFTs
(fft.Domain.fft_device), the accumulation polynomial (gmsm_fr_permutation_accumulate_device: a tile batch inversion and a
multi-level prefix product), the quotient numerator on the coset (gmsm_fft_permutation_numerator_device) and the commitments and
openings of kzg.py on device tensors.  Only the inputs (when they are host arrays), the four digests, the opening proofs and the five
claimed values cross PCIe.  A proving key sharded over several GPUs (device = -1) runs the same Fr work on the current device and
commits and opens through kzg's host entry points, which gives the same proof.  Verify needs pairings and is not built."""
from __future__ import annotations

import hashlib
from dataclasses import dataclass

import numpy as np

from . import fft, kzg
from .curves import _challenge, _curve, _fr_decode, _fr_encode, _params
from .fft import DIF, DIT
from .kzg import g1_raw_bytes
from .multiexp import MultiExpError
from .transcript import Transcript


class ErrIncompatibleSize(MultiExpError):
    """permutation.ErrIncompatibleSize (permutation.go:22)"""


class ErrSize(MultiExpError):
    """permutation.ErrSize (permutation.go:23)"""


@dataclass
class Proof:
    """permutation.Proof (permutation.go:29-50): the digests t1, t2, z, q are G1Affine limbs, g the domain's generator (fr.Element
    limbs); batchedProof opens t1, t2, z, q (in that order) at eta, shiftedProof opens z at eta g"""

    size: int
    g: np.ndarray
    t1: np.ndarray
    t2: np.ndarray
    z: np.ndarray
    q: np.ndarray
    batchedProof: kzg.BatchOpeningProof
    shiftedProof: kzg.OpeningProof


def Prove(pk: kzg.ProvingKey, t1, t2) -> Proof:
    """permutation.Prove: t1 and t2 are numpy (n, fr.Limbs) arrays or torch CUDA int64 tensors in the same layout (on the key's
    device for a single-device key), left unmodified.  The work is ordered on the current stream of the device."""
    import torch

    w = _params(pk.curve).fr_words
    n = kzg._poly_len(t1, w)
    if n != kzg._poly_len(t2, w):
        raise ErrIncompatibleSize("t1 and t2 should be of the same size")
    # NewDomain(n).Cardinality != n (NextPowerOfTwo(0) = 1): refused before a domain is built
    if n == 0 or n & (n - 1):
        raise ErrSize("t1 and t2 should be of size a power of 2")
    curve = _curve(pk.curve)
    dev = pk.device if pk.device >= 0 else torch.cuda.current_device()
    d = fft.NewDomain(curve, n, device=dev)
    try:
        with torch.cuda.device(dev):
            return _prove(pk, d, t1, t2, n, curve, dev)
    finally:
        d.close()


def _prove(pk, d, t1, t2, n, curve, dev):
    cp = _params(curve)
    r, w = cp.r, cp.fr_words
    dp = kzg._DevicePoly(curve, dev, n)
    st = dp.stream
    sharded = pk.device < 0

    def commit(p):
        return kzg.Commit(kzg._host_poly(p, w) if sharded else p, pk)

    d_t1, d_t2 = (kzg._device_poly(t, w, dev) for t in (t1, t2))   # device tensors in place, host arrays uploaded once
    ct1, ct2 = d_t1.clone(), d_t2.clone()
    for ct in (ct1, ct2):                                   # coefficients: FFTInverse(DIF) + BitReverse
        d.fft_device(ct, True, DIF, False, st)
        d.bit_reverse_device(ct, st)
    T1, T2 = commit(ct1), commit(ct2)
    fs = Transcript(hashlib.sha256, "epsilon", "omega", "eta")
    for p in (T1, T2):
        fs.Bind("epsilon", g1_raw_bytes(p, curve))
    eps = _fr_encode([_challenge(fs, "epsilon", r)], r)[0]
    # Z in the bit-reversed Lagrange layout, then its coefficients by FFTInverse(DIT)
    cz = dp.empty(n)
    dp.permutation_accumulate(d_t1, d_t2, n, eps, cz)
    d.fft_device(cz, True, DIT, False, st)
    Z = commit(cz)
    # the three coset evaluations (bit-reversed), the numerator, and the quotient's coefficients
    lz, lt1, lt2 = cz.clone(), ct1.clone(), ct2.clone()
    for v in (lz, lt1, lt2):
        d.fft_device(v, False, DIF, True, st)
    fs.Bind("omega", g1_raw_bytes(Z, curve))
    omega = _fr_encode([_challenge(fs, "omega", r)], r)[0]
    qv = dp.empty(n)
    dp.permutation_numerator(d, lt1, lt2, lz, eps, omega, qv)
    del lz, lt1, lt2
    d.fft_device(qv, True, DIT, True, st)
    Q = commit(qv)
    fs.Bind("eta", g1_raw_bytes(Q, curve))
    eta = _challenge(fs, "eta", r)
    polys = [ct1, ct2, cz, qv]
    if sharded:
        polys = [kzg._host_poly(p, w) for p in polys]
    batched = kzg.BatchOpenSinglePoint(polys, [T1, T2, Z, Q], _fr_encode([eta], r)[0], hashlib.sha256, pk)
    gen = _fr_decode(d.Generator, r)[0]
    shifted = kzg.Open(polys[2], _fr_encode([eta * gen % r], r)[0], pk)
    return Proof(size=n, g=d.Generator.copy(), t1=T1, t2=T2, z=Z, q=Q, batchedProof=batched, shiftedProof=shifted)

