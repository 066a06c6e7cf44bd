"""The argument checks of kzg.BatchVerifyMultiPoints (kzg.go:405-415) and of pairing.py that run before any device work.
CPU only."""
from importlib import import_module

import numpy as np
import pytest


def test_batch_verify_multi_points_sizes():
    kzg = import_module("gnark-crypto_b200.kzg")
    vk = kzg.VerifyingKey("bn254", np.zeros((2, 16), dtype=np.uint64), np.zeros(8, dtype=np.uint64))
    d = [np.zeros(8, dtype=np.uint64)] * 2
    p = [kzg.OpeningProof(H=np.zeros(8, dtype=np.uint64), ClaimedValue=np.zeros(4, dtype=np.uint64))] * 2
    x = [np.zeros(4, dtype=np.uint64)] * 2
    with pytest.raises(kzg.ErrInvalidNbDigests, match="number of digests is not the same"):
        kzg.BatchVerifyMultiPoints(d, p[:1], x, vk)
    with pytest.raises(kzg.ErrInvalidNbDigests):
        kzg.BatchVerifyMultiPoints(d, p, x[:1], vk)
    with pytest.raises(kzg.ErrZeroNbDigests, match="number of digests is zero"):
        kzg.BatchVerifyMultiPoints([], [], [], vk)


def test_pairing_argument_checks():
    pr = import_module("gnark-crypto_b200.pairing")
    P = np.zeros((2, 8), dtype=np.uint64)
    Q = np.zeros((2, 16), dtype=np.uint64)
    with pytest.raises(ValueError, match="invalid inputs sizes"):
        pr.MillerLoop("bn254", P[:0], Q[:0])
    with pytest.raises(ValueError, match="invalid inputs sizes"):
        pr.Pair("bn254", P, Q[:1])
    with pytest.raises(ValueError, match="whole points"):
        pr.Pair("bn254", P.reshape(-1)[:-1], Q)
    for curve in ("bls12377", "bw6761", "bw6633", "bls24315", "bls24317"):
        with pytest.raises(ValueError):
            pr.Pair(curve, P, Q)
