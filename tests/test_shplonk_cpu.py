"""SHPLONK / FFLONK batch openings without a GPU: the identity-based algorithm of shplonk.open_packs (restated on ints in
tests/shplonk_ref.py) equals the line-by-line restatement of the reference (shplonk.batch_open_host) limb for limb on all seven
curves, over shapes with repeated points, empty point sets, short polynomials and FFLONK packs of 1, 2, 3 and 5; the proofs pass
BatchVerify in the exponent with a known-alpha SRS and the oracle's MultiExp; tampered proofs fail it; the Fiat-Shamir transcript
chains its challenges as fiat-shamir/transcript.go does."""
import hashlib
import random
from importlib import import_module

import pytest

from tests import shplonk_ref as ref

curves = import_module("gnark-crypto_b200.curves")

CURVES = ["bn254", "bls12381", "bls12377", "bls24315", "bls24317", "bw6633", "bw6761"]


def _mods():
    return import_module("gnark-crypto_b200.kzg"), import_module("gnark-crypto_b200.shplonk"), import_module("gnark-crypto_b200.fflonk")


def _shplonk_shapes(r, rng):
    """(polynomial lengths, point sets) of plain SHPLONK"""
    a, b, c = (rng.randrange(r) for _ in range(3))
    return [
        ([9, 7, 12], [[a], [a, b], [c, a, b]]),                 # points repeated across sets
        ([6, 5, 4], [[a, b], [], [c]]),                         # an empty set
        ([2, 1, 8], [[a, b, c], [b, c], [a]]),                  # len(f_i) < |S_i|
        ([2, 3], [[a, b, c, rng.randrange(r)], [b]]),           # |S_i| + 1 larger than every length
        ([7, 6], [[a, a, b], [c]]),                             # a point repeated inside one set
        ([5], [[0, 1, r - 1]]),
    ]


def _digests(srs, polys):
    return [srs.commit(p) for p in polys]


@pytest.mark.parametrize("c", CURVES)
def test_shplonk_identities_equal_reference(c):
    kzg, shplonk, _ = _mods()
    r = kzg.CURVE_PARAMS[c].r
    rng = random.Random(101 + CURVES.index(c))
    srs = ref.OracleSRS(c, 24, rng.randrange(r))
    for lens, points in _shplonk_shapes(r, rng):
        polys = [[rng.randrange(r) for _ in range(n)] for n in lens]
        digests = _digests(srs, polys)
        want = shplonk.batch_open_host(polys, points, digests, hashlib.sha256, c, srs.commit, b"data")
        got = ref.identity_open([[p] for p in polys], points, [1] * len(points), points, digests, hashlib.sha256, c, srs.commit, b"data")
        assert got[4] == want[3] and got[5] == want[4], (lens, points)             # w and w' coefficient for coefficient
        assert got[2] == want[2]                                                     # claimed values
        assert (got[0] == want[0]).all() and (got[1] == want[1]).all()
        # a point repeated inside one set makes the reference interpolate through 1/0 = 0: a deterministic proof that fails
        # BatchVerify, which the identities reproduce all the same
        distinct = all(len(set(S)) == len(S) for S in points)
        assert ref.verify_in_exponent(polys, points, want[0], want[1], want[2], digests, hashlib.sha256, c, srs.alpha, b"data") == distinct


@pytest.mark.parametrize("c", CURVES)
def test_fflonk_identities_equal_reference(c):
    """packs of 1, 2, 3 and 5 polynomials (t from getNextDivisorRMinusOne), unequal lengths, a repeated s^t inside a pack"""
    kzg, shplonk, fflonk = _mods()
    r = kzg.CURVE_PARAMS[c].r
    rng = random.Random(202 + CURVES.index(c))
    srs = ref.OracleSRS(c, 48, rng.randrange(r))
    s = [rng.randrange(r) for _ in range(3)]
    for sizes, pts in (([1, 2, 3, 5], [[s[0]], [s[1], s[0]], [s[2]], [s[1]]]), ([3, 2], [[s[0], s[1]], []])):
        packs = [[[rng.randrange(r) for _ in range(rng.randrange(1, 6))] for _ in range(k)] for k in sizes]
        ts = [fflonk._next_divisor_r_minus_one(len(pk), r) for pk in packs]
        assert all(t >= len(pk) and (r - 1) % t == 0 for t, pk in zip(ts, packs))
        ext = [fflonk._extend_set(S, t, c) for S, t in zip(pts, ts)]
        folded = [curves._fr_decode(fflonk.Fold([curves._fr_encode(p, r) for p in pk], c), r) for pk in packs]
        digests = _digests(srs, folded)
        want = shplonk.batch_open_host(folded, ext, digests, hashlib.sha256, c, srs.commit)
        got = ref.identity_open(packs, pts, ts, ext, digests, hashlib.sha256, c, srs.commit)
        assert got[4] == want[3] and got[5] == want[4] and got[2] == want[2], (sizes, ts)
        outer = [[[shplonk._eval(p, pow(x, t, r), r) for x in S] for p in pk] for pk, S, t in zip(packs, pts, ts)]
        assert got[3] == outer
        padded = [o + [[0] * len(S)] * (t - len(o)) for o, S, t in zip(outer, pts, ts)]
        assert ref.fflonk_fold_consistent(padded, want[2], pts, c)
        assert ref.verify_in_exponent(folded, ext, want[0], want[1], want[2], digests, hashlib.sha256, c, srs.alpha)
    # a pack of 3 at two points that share s^3 (s and s omega): the identities still give the reference's digests
    omega = fflonk._ith_root_one(3, c) if (r - 1) % 3 == 0 else None
    if omega is not None:
        pk3 = [[rng.randrange(r) for _ in range(4)] for _ in range(3)]
        S = [s[0], s[0] * omega % r]
        ext = [fflonk._extend_set(S, 3, c)]
        folded = [curves._fr_decode(fflonk.Fold([curves._fr_encode(p, r) for p in pk3], c), r)]
        digests = _digests(srs, folded)
        want = shplonk.batch_open_host(folded, ext, digests, hashlib.sha256, c, srs.commit)
        got = ref.identity_open([pk3], [S], [3], ext, digests, hashlib.sha256, c, srs.commit)
        assert got[4] == want[3] and got[5] == want[4] and got[2] == want[2]


def test_tampered_proofs_fail_verification():
    kzg, shplonk, _ = _mods()
    c = "bls12381"
    r = kzg.CURVE_PARAMS[c].r
    rng = random.Random(7)
    srs = ref.OracleSRS(c, 16, rng.randrange(r))
    polys = [[rng.randrange(r) for _ in range(n)] for n in (8, 5)]
    points = [[rng.randrange(r)], [rng.randrange(r), rng.randrange(r)]]
    digests = _digests(srs, polys)
    W, WPrime, claimed, _, _ = shplonk.batch_open_host(polys, points, digests, hashlib.sha256, c, srs.commit)
    assert ref.verify_in_exponent(polys, points, W, WPrime, claimed, digests, hashlib.sha256, c, srs.alpha)
    bad = [list(v) for v in claimed]
    bad[1][0] = (bad[1][0] + 1) % r
    assert not ref.verify_in_exponent(polys, points, W, WPrime, bad, digests, hashlib.sha256, c, srs.alpha)
    assert not ref.verify_in_exponent(polys, points, W, srs.mul(5), claimed, digests, hashlib.sha256, c, srs.alpha)
    assert not ref.verify_in_exponent(polys, points, W, WPrime, claimed, digests, hashlib.sha256, c, srs.alpha, b"other")


def test_transcript_chains_challenges():
    tr = import_module("gnark-crypto_b200.transcript")
    fs = tr.Transcript(hashlib.sha256, "gamma", "z")
    fs.Bind("gamma", b"ab")
    fs.Bind("gamma", b"c")
    with pytest.raises(ValueError, match="previous challenge"):
        fs.ComputeChallenge("z")
    g = fs.ComputeChallenge("gamma")
    assert g == hashlib.sha256(b"gammaabc").digest() and fs.ComputeChallenge("gamma") == g
    with pytest.raises(ValueError, match="already computed"):
        fs.Bind("gamma", b"x")
    fs.Bind("z", b"W")
    assert fs.ComputeChallenge("z") == hashlib.sha256(b"z" + g + b"W").digest()
    with pytest.raises(ValueError, match="not recorded"):
        fs.Bind("beta", b"")
    b2 = tr.Transcript(hashlib.blake2b, "gamma")
    assert b2.ComputeChallenge("gamma") == hashlib.blake2b(b"gamma").digest()
