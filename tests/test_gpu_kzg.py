"""Next-row N2 (SURVEY.md section 8f) on the GPU: batched KZG openings at one point (kzg.BatchOpenSinglePoint / FoldProof,
ecc/bn254/kzg/kzg.go:246-380) over resident bases, and bulk decoding of serialised G1 points (G1Affine.SetBytes,
marshal.go:858-950) on the device.  The reference verifies openings with pairings (out of scope); with a test SRS whose
alpha is known the same equations are checked in the exponent by the CPU oracle, like TestCommit (kzg_test.go:209-239)."""
import hashlib
from importlib import import_module

import numpy as np
import pytest

from oracle import cref
from oracle import oracle as O

pytestmark = pytest.mark.gpu


def test_batch_open_single_point_and_fold_proof():
    kzg = import_module("gnark-crypto_b200.kzg")
    g = "bn254_g1"
    G = O.GROUPS[g]
    r = G.fr.q
    size, alpha = 1500, 0x7654321FEDCBA9876543
    gen = G.encode_affine([G.gen])[0]
    srs = kzg.new_srs_g1("bn254", size, alpha, gen, r, G.encode_scalars)
    pk = kzg.ProvingKey("bn254", srs)
    rng = np.random.default_rng(11)
    polys = [[int(x) for x in rng.integers(0, 2**62, size=m)] for m in (1500, 1200, 700)]
    enc = [G.encode_scalars(p) for p in polys]
    digests = [kzg.Commit(e, pk) for e in enc]
    ev = lambda p, x: sum(c * pow(x, i, r) for i, c in enumerate(p)) % r
    for p, d in zip(polys, digests):
        assert np.array_equal(d, cref.scalar_mul(g, gen, ev(p, alpha)))
    a = 0xABCDEF0123456789
    point = G.encode_scalars([a])[0]
    extra = b"transcript-data"
    proof = kzg.BatchOpenSinglePoint(enc, digests, point, hashlib.sha256, pk, extra)
    # claimed values f_i(a)
    assert np.array_equal(proof.ClaimedValues, G.encode_scalars([ev(p, a) for p in polys]))
    # gamma: the transcript restated independently here (fiat-shamir/transcript.go:61-131, kzg.go:531-563)
    h = hashlib.sha256()
    h.update(b"gamma")
    h.update(a.to_bytes(32, "big"))
    for d in digests:
        x, y = G.decode_affine(d.reshape(1, -1))[0]
        h.update(int(x).to_bytes(32, "big") + int(y).to_bytes(32, "big"))
    for p in polys:
        h.update(ev(p, a).to_bytes(32, "big"))
    h.update(extra)
    gamma = int.from_bytes(h.digest(), "big") % r
    assert kzg.derive_gamma(point, digests, proof.ClaimedValues, hashlib.sha256, "bn254", extra) == gamma
    # H = [ (sum gamma^i f_i(alpha) - sum gamma^i f_i(a)) / (alpha - a) ] G
    fold_alpha = sum(pow(gamma, i, r) * ev(p, alpha) for i, p in enumerate(polys)) % r
    fold_a = sum(pow(gamma, i, r) * ev(p, a) for i, p in enumerate(polys)) % r
    assert np.array_equal(proof.H, cref.scalar_mul(g, gen, (fold_alpha - fold_a) * pow(alpha - a, -1, r) % r))
    # FoldProof: folded digest = sum gamma^i digest_i (one MultiExp), folded claimed value, same H
    op, folded = kzg.FoldProof(digests, proof, point, hashlib.sha256, "bn254", extra)
    assert np.array_equal(folded, cref.scalar_mul(g, gen, fold_alpha))
    assert np.array_equal(op.ClaimedValue, G.encode_scalars([fold_a])[0]) and np.array_equal(op.H, proof.H)
    with pytest.raises(kzg.ErrInvalidNbDigests):
        kzg.BatchOpenSinglePoint(enc, digests[:2], point, hashlib.sha256, pk)
    with pytest.raises(kzg.ErrInvalidPolynomialSize):
        kzg.BatchOpenSinglePoint([np.zeros((0, 4), dtype=np.uint64)], digests[:1], point, hashlib.sha256, pk)
    pk.close()


@pytest.mark.parametrize("curve,g", [("bn254", "bn254_g1"), ("bls12381", "bls12381_g1")])
def test_device_point_decoding_matches_host_set_bytes(curve, g):
    """compressed and uncompressed streams, with infinity points, through gmsm_g1_decode against the host restatement of
    SetBytes (itself round-tripped against the oracle's points in tests/test_kzg_format_cpu.py) and the original points"""
    kzg = import_module("gnark-crypto_b200.kzg")
    G = O.GROUPS[g]
    n = 3000
    base = G.encode_affine([G.gen])[0]
    pts = cref.generate_multiples(g, base, 7, n, nthreads=4)
    pts[5] = 0
    pts[n - 1] = 0
    c = curve
    comp = b"".join(kzg.g1_bytes(p, c) for p in pts)
    raw = b"".join(kzg.g1_raw_bytes(p, c) for p in pts)
    assert np.array_equal(kzg.decode_g1_points(c, comp, n, raw=False), pts)
    assert np.array_equal(kzg.decode_g1_points(c, raw, n, raw=True), pts)
    # both signs of y occur
    flags = {comp[i * len(comp) // n] >> 5 for i in range(n)}
    assert len(flags) >= 3
    # resident bases straight from the byte stream: Commit == oracle MSM
    pk = kzg.ProvingKey.from_bytes(c, comp, n)
    s = cref.random_scalars(g, n, 3)
    want, _, _, _ = cref.msm(g, pts, s, c=0, nthreads=4)
    assert np.array_equal(kzg.Commit(s, pk), want)
    pk.close()
    # error paths carry the reference's messages and the index of the first bad point
    nb = len(comp) // n
    bad = bytearray(comp)
    bad[7 * nb + nb - 1] ^= 1          # x of point 7 changed: with probability 1/2 x^3 + b is a non-residue -> try a few
    for k in range(1, 40):
        bad2 = bytearray(comp)
        bad2[7 * nb + nb - 1] = (comp[7 * nb + nb - 1] + k) & 0xFF
        try:
            kzg.decode_g1_points(c, bytes(bad2), n, raw=False)
        except kzg.MultiExpError as e:
            assert "point 7" in str(e) and "square root doesn't exist" in str(e)
            break
    else:
        raise AssertionError("no non-residue found")
    bad3 = bytearray(raw)
    bad3[9 * 2 * nb + 2 * nb - 1] ^= 1   # y of point 9 off the curve
    with pytest.raises(kzg.MultiExpError, match="point 9: invalid point"):
        kzg.decode_g1_points(c, bytes(bad3), n, raw=True)
    assert kzg.decode_g1_points(c, bytes(bad3), n, raw=True, check_on_curve=False).shape == (n, pts.shape[1])
    bad4 = bytearray(comp)
    bad4[5 * nb + 3] = 1                # infinity flag with a non-zero byte
    with pytest.raises(kzg.MultiExpError, match="point 5: invalid infinity point encoding"):
        kzg.decode_g1_points(c, bytes(bad4), n, raw=False)
    bad5 = bytearray(raw)
    bad5[3 * 2 * nb:3 * 2 * nb + nb] = bytes([~kzg.CURVE_PARAMS[c].flags["mask"] & 0xFF]) + b"\xff" * (nb - 1)   # x >= q, flag bits zero (uncompressed)
    with pytest.raises(kzg.MultiExpError, match="point 3: invalid fp.Element encoding"):
        kzg.decode_g1_points(c, bytes(bad5), n, raw=True)


def test_commit_from_lagrange_values_stays_on_the_device():
    """next-row N3 -> N2 fusion: evaluations -> FFTInverse + BitReverse on the device -> MultiExp over resident bases with the
    device-resident coefficients (gmsm_bases_multiexp_device) == Commit of the host iFFT == [f(alpha)]G"""
    kzg = import_module("gnark-crypto_b200.kzg")
    fft = import_module("gnark-crypto_b200.fft")
    g = "bn254_g1"
    G = O.GROUPS[g]
    r = G.fr.q
    size, alpha = 4096, 0xBEEF1234567
    gen = G.encode_affine([G.gen])[0]
    srs = kzg.new_srs_g1("bn254", size, alpha, gen, r, G.encode_scalars)
    pk = kzg.ProvingKey("bn254", srs)
    dom = fft.NewDomain("bn254", size)
    rng = np.random.default_rng(5)
    coeffs = [int(x) for x in rng.integers(0, 2**62, size=size)]
    evals = G.encode_scalars(coeffs)                 # take them as coefficients, move to evaluations with the host-buffer FFT
    dom.FFT(evals, fft.DIF)
    ev_nat = evals.copy()
    # bit-reverse on the host to natural order (DIF output is bit-reversed)
    idx = np.array([int(format(i, "012b")[::-1], 2) for i in range(size)])
    ev_nat = evals[idx]
    digest = kzg.CommitLagrange(ev_nat, pk, dom)
    f_alpha = sum(c * pow(alpha, i, r) for i, c in enumerate(coeffs)) % r
    assert np.array_equal(digest, cref.scalar_mul(g, gen, f_alpha))
    assert np.array_equal(digest, kzg.Commit(G.encode_scalars(coeffs), pk))
    pk.close()
    dom.close()
