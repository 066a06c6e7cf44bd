"""Next-row N3: host-side mirror of gnark-crypto's fft package over the C ABI.

Reference: ecc/bn254/fr/fft (domain.go:24-110 `Domain`, `NewDomain`; fft.go:18-190 `Decimation`, `FFT`,
`FFTInverse`, option `OnCoset`; bitreverse.go:17-42 `BitReverse`) and the same package of bls12-381, bls12-377, bls24-315,
bls24-317, bw6-633 and bw6-761.  Vectors are numpy (n, words) uint64 arrays = []fr.Element memory (Montgomery limbs;
words = fr.Limbs: 4, 5 for bw6-633, 6 for bw6-761), transformed in place."""
from __future__ import annotations

import numpy as np

from . import _native
from .curves import CURVE_PARAMS
from .multiexp import MultiExpError, _check, _handle

DIT, DIF = 0, 1  # fft.Decimation


class Domain:
    """fft.Domain; `NewDomain(curve, m, shift=None)`"""

    def __init__(self, curve: str, m: int, shift: np.ndarray = None, device: int = 0):
        L = _native.lib()
        if curve not in CURVE_PARAMS:
            raise MultiExpError("unknown curve %r (FFT over Fr: %s)" % (curve, ", ".join(CURVE_PARAMS)))
        fr_id = CURVE_PARAMS[curve].fr_id
        self.curve = curve
        self.words = int(L.gmsm_fft_fr_bytes(fr_id)) // 8
        sp = None
        if shift is not None:
            shift = np.ascontiguousarray(shift, dtype=np.uint64).reshape(self.words)
            sp = shift.ctypes.data
        self._h = _handle(L.gmsm_fft_domain_create(fr_id, int(m), sp, device))
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
        _check(_native.lib().gmsm_fft(self._h, a.ctypes.data, self.Cardinality, int(decimation), 1 if OnCoset else 0))
        return a

    def FFTInverse(self, a: np.ndarray, decimation: int, OnCoset: bool = False):
        a = self._vec(a)
        _check(_native.lib().gmsm_fft_inverse(self._h, a.ctypes.data, self.Cardinality, int(decimation), 1 if OnCoset else 0))
        return a

    # device tensors (torch int64 views of the same layout)
    def fft_device(self, d_a, inverse: bool, decimation: int, coset: bool = False, stream=None):
        _check(_native.lib().gmsm_fft_device(self._h, d_a.data_ptr(), self.Cardinality, 1 if inverse else 0, int(decimation),
                                             1 if coset else 0, stream))
        return d_a

    def bit_reverse_device(self, d_a, stream=None):
        _check(_native.lib().gmsm_fft_bit_reverse_device(self._h, d_a.data_ptr(), self.Cardinality, stream))
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
