"""Next-row N3: host-side mirror of gnark-crypto's fft package over the C ABI.

Reference: ecc/bn254/fr/fft (domain.go:24-110 `Domain`, `NewDomain`; fft.go:18-190 `Decimation`, `FFT`,
`FFTInverse`, option `OnCoset`; bitreverse.go:17-42 `BitReverse`) and the same package of bls12-381, bls12-377, bls24-315,
bls24-317, bw6-633 and bw6-761.  Vectors are numpy (n, words) uint64 arrays = []fr.Element memory (Montgomery limbs;
words = fr.Limbs: 4, 5 for bw6-633, 6 for bw6-761), transformed in place."""
from __future__ import annotations

import numpy as np

from . import _native
from .multiexp import MultiExpError

DIT, DIF = 0, 1  # fft.Decimation
_FIELDS = {"bn254": 0, "bls12381": 1, "bls12377": 2, "bls24315": 3, "bls24317": 4, "bw6633": 5, "bw6761": 6}


class Domain:
    """fft.Domain; `NewDomain(curve, m, shift=None)`"""

    def __init__(self, curve: str, m: int, shift: np.ndarray = None, device: int = 0):
        L = _native.lib()
        if curve not in _FIELDS:
            raise MultiExpError("unknown curve %r (FFT over Fr: %s)" % (curve, ", ".join(_FIELDS)))
        self.words = int(L.gmsm_fft_fr_bytes(_FIELDS[curve])) // 8
        sp = None
        if shift is not None:
            shift = np.ascontiguousarray(shift, dtype=np.uint64).reshape(self.words)
            sp = shift.ctypes.data
        self._h = L.gmsm_fft_domain_create(_FIELDS[curve], int(m), sp, device)
        if not self._h:
            raise MultiExpError(_native.last_error())
        self.device = device
        self.Cardinality = int(L.gmsm_fft_domain_cardinality(self._h))
        c = np.zeros(5 * self.words, dtype=np.uint64)
        L.gmsm_fft_domain_constants(self._h, c.ctypes.data)
        c = c.reshape(5, self.words)
        self.Generator, self.GeneratorInv, self.CardinalityInv, self.FrMultiplicativeGen, self.FrMultiplicativeGenInv = (
            c[0].copy(), c[1].copy(), c[2].copy(), c[3].copy(), c[4].copy())

    def _vec(self, a):
        if not (isinstance(a, np.ndarray) and a.dtype == np.uint64 and a.flags["C_CONTIGUOUS"]):
            raise ValueError("a must be a C-contiguous numpy uint64 array (transformed in place)")
        if a.size != self.words * self.Cardinality:
            raise MultiExpError("len(a) must equal the domain cardinality")
        return a

    def FFT(self, a: np.ndarray, decimation: int, OnCoset: bool = False):
        a = self._vec(a)
        rc = _native.lib().gmsm_fft(self._h, a.ctypes.data, self.Cardinality, int(decimation), 1 if OnCoset else 0)
        if rc:
            raise MultiExpError(_native.last_error())
        return a

    def FFTInverse(self, a: np.ndarray, decimation: int, OnCoset: bool = False):
        a = self._vec(a)
        rc = _native.lib().gmsm_fft_inverse(self._h, a.ctypes.data, self.Cardinality, int(decimation), 1 if OnCoset else 0)
        if rc:
            raise MultiExpError(_native.last_error())
        return a

    # device tensors (torch int64 views of the same layout)
    def fft_device(self, d_a, inverse: bool, decimation: int, coset: bool = False, stream=None):
        rc = _native.lib().gmsm_fft_device(self._h, d_a.data_ptr(), self.Cardinality, 1 if inverse else 0, int(decimation),
                                           1 if coset else 0, stream)
        if rc:
            raise MultiExpError(_native.last_error())
        return d_a

    def bit_reverse_device(self, d_a, stream=None):
        rc = _native.lib().gmsm_fft_bit_reverse_device(self._h, d_a.data_ptr(), self.Cardinality, stream)
        if rc:
            raise MultiExpError(_native.last_error())
        return d_a

    def close(self):
        if self._h:
            _native.lib().gmsm_fft_domain_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def NewDomain(curve: str, m: int, shift=None, device: int = 0) -> Domain:
    return Domain(curve, m, shift, device)
