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

from . import _native, fft, kzg
from .fft import DIF, DIT
from .kzg import _fr_decode, _fr_encode, g1_raw_bytes
from .multiexp import MultiExpError, _check
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

    cp = kzg._params(pk.curve)
    r, w = cp.r, cp.fr_words
    n = kzg._poly_len(t1, w)
    if n != kzg._poly_len(t2, w):
        raise ErrIncompatibleSize("t1 and t2 should be of the same size")
    # NewDomain(n).Cardinality != n (NextPowerOfTwo(0) = 1): refused before a domain is built
    if n == 0 or n & (n - 1):
        raise ErrSize("t1 and t2 should be of size a power of 2")
    curve = pk.curve.split("_")[0]
    dev_id = pk.device if pk.device >= 0 else torch.cuda.current_device()
    d = fft.NewDomain(curve, n, device=dev_id)
    try:
        with torch.cuda.device(dev_id):
            return _prove(pk, d, t1, t2, n, curve, torch.device("cuda", dev_id))
    finally:
        d.close()


def _challenge(fs: Transcript, name: str, r: int) -> int:
    """fr.Element.SetBytes of the raw challenge: big-endian, reduced mod r"""
    return int.from_bytes(fs.ComputeChallenge(name), "big") % r


def _prove(pk, d, t1, t2, n, curve, dev):
    import torch

    cp = kzg._params(curve)
    r, w = cp.r, cp.fr_words
    field = fft._FIELDS[curve]
    L = _native.lib()
    st = torch.cuda.current_stream(dev).cuda_stream
    sharded = pk.device < 0

    def commit(p):
        return kzg.Commit(_host(p, w) if sharded else p, pk)

    d_t1, d_t2 = (kzg._device_poly(t, w, dev.index) for t in (t1, t2))   # device tensors in place, host arrays uploaded once
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
    cz = torch.empty(n * w, dtype=torch.int64, device=dev)
    ws = int(L.gmsm_fr_permutation_workspace_bytes(field, n))
    work = torch.empty(ws // 8, dtype=torch.int64, device=dev) if ws else None
    _check(L.gmsm_fr_permutation_accumulate_device(field, d_t1.data_ptr(), d_t2.data_ptr(), n, eps.ctypes.data,
                                                   cz.data_ptr(), None if work is None else work.data_ptr(), st))
    d.fft_device(cz, True, DIT, False, st)
    Z = commit(cz)
    # the three coset evaluations (bit-reversed), the numerator, and the quotient's coefficients
    lz, lt1, lt2 = cz.clone(), ct1.clone(), ct2.clone()
    for v in (lz, lt1, lt2):
        d.fft_device(v, False, DIF, True, st)
    fs.Bind("omega", g1_raw_bytes(Z, curve))
    omega = _fr_encode([_challenge(fs, "omega", r)], r)[0]
    qv = torch.empty(n * w, dtype=torch.int64, device=dev)
    _check(L.gmsm_fft_permutation_numerator_device(d._h, lt1.data_ptr(), lt2.data_ptr(), lz.data_ptr(), n, eps.ctypes.data,
                                                   omega.ctypes.data, qv.data_ptr(), st))
    del lz, lt1, lt2
    d.fft_device(qv, True, DIT, True, st)
    Q = commit(qv)
    fs.Bind("eta", g1_raw_bytes(Q, curve))
    eta = _challenge(fs, "eta", r)
    polys = [ct1, ct2, cz, qv]
    if sharded:
        polys = [_host(p, w) for p in polys]
    batched = kzg.BatchOpenSinglePoint(polys, [T1, T2, Z, Q], _fr_encode([eta], r)[0], hashlib.sha256, pk)
    gen = _fr_decode(d.Generator, r)[0]
    shifted = kzg.Open(polys[2], _fr_encode([eta * gen % r], r)[0], pk)
    return Proof(size=n, g=d.Generator.copy(), t1=T1, t2=T2, z=Z, q=Q, batchedProof=batched, shiftedProof=shifted)


def _host(p, w):
    return kzg._host_poly(p, w)

