"""gnark-crypto_b200: H100-native multi-scalar multiplication behind gnark-crypto's MultiExp.

Layout:
  csrc/        sm_90a CUDA kernels + the C ABI (include/gmsm.h) -> libgmsm.so (built in-tree)
  _native.py   ctypes loader of libgmsm.so (fails loudly when the library or a GPU is missing)
  curves.py    the one curve table: the thirteen MultiExp groups, the seven pairing curves of the prover, the fr.Element codec
  multiexp.py  host-side mirror of the reference interface for this path:
               G1Affine/G1Jac/G2Affine/G2Jac .MultiExp(points, scalars, MultiExpConfig)
               (ecc/bn254/multiexp.go:20,32,345,357; ecc/ecc.go:107-110) + the device-level Engine
  dist.py      multi-GPU: one process per GPU, shard points/scalars, all-gather the per-window partials
  fft.py, kzg.py, shplonk.py, fflonk.py, permutation.py, plookup.py, transcript.py: the Fr FFT and the KZG provers; kzg._DevicePoly is
               the one caller of the library's device Fr polynomial entry points
  iop.py       the Fr layer of a PLONK prover (ecc/<curve>/fr/iop): Polynomial and its forms, Evaluate of a traced expression, the
               accumulating ratios BuildRatioShuffledVectors / BuildRatioCopyConstraint and DivideByXMinusOne, all on the device
  pairing.py   MillerLoop / FinalExponentiation / Pair / PairingCheck of bn254 and bls12-381 on the device
  mpcsetup.py  the point updates of a trusted-setup contribution (UpdateMonomialsG1/G2, ScaleG1/G2) and the linear combinations of
               SameRatioMany (LinearCombinationsG1/G2)
"""
from . import _native  # noqa: F401
from .multiexp import (  # noqa: F401
    BatchScalarMultiplication,
    CURVES,
    Engine,
    G1Affine,
    G1Jac,
    G2Affine,
    G2Jac,
    MultiExpConfig,
    MultiExpError,
    curve_package,
)

__all__ = ["BatchScalarMultiplication", "CURVES", "Engine", "G1Affine", "G1Jac", "G2Affine", "G2Jac", "MultiExpConfig", "MultiExpError", "curve_package"]
