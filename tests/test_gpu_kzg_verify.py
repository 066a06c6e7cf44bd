"""kzg.Verify, BatchVerifySinglePoint and BatchVerifyMultiPoints (ecc/<curve>/kzg/kzg.go:207-500) on the GPU pairing, for bn254
and bls12-381: proofs of kzg.Open / BatchOpenSinglePoint on a random-alpha SRS are accepted, and a tampered claimed value, H,
point or commitment is refused with ErrVerifyOpeningProof, as the reference's TestVerifySinglePoint / TestBatchVerifyMultiPoints
do (kzg_test.go)."""
import copy
import hashlib
import random
from importlib import import_module

import numpy as np
import pytest

from oracle import oracle as O

pytestmark = pytest.mark.gpu

CURVES = ["bn254", "bls12381"]


def _setup(curve, size, seed):
    kzg = import_module("gnark-crypto_b200.kzg")
    G1, G2 = O.GROUPS[curve + "_g1"], O.GROUPS[curve + "_g2"]
    r = G1.fr.q
    rng = random.Random(seed)
    alpha = rng.randrange(2, r)
    gen = G1.encode_affine([G1.gen])[0]
    pk = kzg.ProvingKey(curve, kzg.new_srs_g1(curve, size, alpha, gen, r, G1.encode_scalars))
    vk = kzg.VerifyingKey(curve, G2.encode_affine([G2.gen, G2.scalar_mul(G2.gen, alpha)]), gen)
    return kzg, G1, r, rng, pk, vk


def _poly(G1, rng, r, n):
    return G1.encode_scalars([rng.randrange(r) for _ in range(n)])


@pytest.mark.parametrize("curve", CURVES)
def test_verify(curve):
    kzg, G1, r, rng, pk, vk = _setup(curve, 64, 1)
    f = _poly(G1, rng, r, 60)
    digest = kzg.Commit(f, pk)
    point = G1.encode_scalars([rng.randrange(r)])[0]
    proof = kzg.Open(f, point, pk)
    kzg.Verify(digest, proof, point, vk)
    bad = copy.deepcopy(proof)
    bad.ClaimedValue = G1.encode_scalars([(G1.fr.from_mont(O.Field.from_limbs([int(x) for x in proof.ClaimedValue])) + 1) % r])[0]
    with pytest.raises(kzg.ErrVerifyOpeningProof):
        kzg.Verify(digest, bad, point, vk)
    bad = copy.deepcopy(proof)
    bad.H = kzg.Commit(_poly(G1, rng, r, 5), pk)
    with pytest.raises(kzg.ErrVerifyOpeningProof):
        kzg.Verify(digest, bad, point, vk)
    with pytest.raises(kzg.ErrVerifyOpeningProof):
        kzg.Verify(digest, proof, G1.encode_scalars([rng.randrange(r)])[0], vk)
    with pytest.raises(kzg.ErrVerifyOpeningProof):
        kzg.Verify(kzg.Commit(_poly(G1, rng, r, 60), pk), proof, point, vk)


@pytest.mark.parametrize("curve", CURVES)
def test_batch_verify_single_point(curve):
    kzg, G1, r, rng, pk, vk = _setup(curve, 64, 2)
    polys = [_poly(G1, rng, r, n) for n in (64, 40, 13)]
    digests = [kzg.Commit(f, pk) for f in polys]
    point = G1.encode_scalars([rng.randrange(r)])[0]
    proof = kzg.BatchOpenSinglePoint(polys, digests, point, hashlib.sha256, pk, b"data")
    kzg.BatchVerifySinglePoint(digests, proof, point, hashlib.sha256, vk, b"data")
    with pytest.raises(kzg.ErrVerifyOpeningProof):
        kzg.BatchVerifySinglePoint(digests, proof, point, hashlib.sha256, vk, b"other data")
    bad = copy.deepcopy(proof)
    bad.ClaimedValues = bad.ClaimedValues.copy()
    bad.ClaimedValues[1] = G1.encode_scalars([5])[0]
    with pytest.raises(kzg.ErrVerifyOpeningProof):
        kzg.BatchVerifySinglePoint(digests, bad, point, hashlib.sha256, vk, b"data")


@pytest.mark.parametrize("curve", CURVES)
def test_batch_verify_multi_points(curve):
    kzg, G1, r, rng, pk, vk = _setup(curve, 32, 3)
    digests, proofs, points = [], [], []
    for _ in range(17):
        f = _poly(G1, rng, r, 30)
        x = G1.encode_scalars([rng.randrange(r)])[0]
        digests.append(kzg.Commit(f, pk))
        proofs.append(kzg.Open(f, x, pk))
        points.append(x)
    for k in (1, 2, 17):
        kzg.BatchVerifyMultiPoints(digests[:k], proofs[:k], points[:k], vk)
    for bad_index in (0, 9):
        bad = [copy.deepcopy(p) for p in proofs]
        bad[bad_index].H = proofs[(bad_index + 1) % 17].H
        with pytest.raises(kzg.ErrVerifyOpeningProof):
            kzg.BatchVerifyMultiPoints(digests, bad, points, vk)
    with pytest.raises(kzg.ErrVerifyOpeningProof):
        kzg.BatchVerifyMultiPoints(digests, proofs, points[:16] + [points[0]], vk)
