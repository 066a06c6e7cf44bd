"""The KZG prover and the device SRS decoding on all seven pairing curves.  With a test SRS whose alpha is known, every
result is checked in the exponent with the CPU oracle (like TestCommit, kzg_test.go:209-239): Commit = [f(alpha)]G, Open and
BatchOpenSinglePoint / FoldProof (gamma re-derived here with the curve's fr.Bytes / fp.Bytes), CommitLagrange = Commit of the
host iFFT, and gmsm_g1_decode of both encodings = the original points, with the reference's error messages."""
import hashlib
from importlib import import_module

import numpy as np
import pytest

from oracle import cref
from oracle import oracle as O

curves = import_module("gnark-crypto_b200.curves")

pytestmark = pytest.mark.gpu
CURVES = ["bn254", "bls12381", "bls12377", "bls24315", "bls24317", "bw6633", "bw6761"]


def _ev(p, x, r):
    return sum(c * pow(x, i, r) for i, c in enumerate(p)) % r


@pytest.mark.parametrize("c", CURVES)
def test_table_multiplicative_generator(c):
    """the curve table's GeneratorFullMultiplicativeGroup is the one the library's Fr domain uses"""
    d = import_module("gnark-crypto_b200.fft").NewDomain(c, 2)
    cp = curves.CURVE_PARAMS[c]
    try:
        assert curves._fr_decode(d.FrMultiplicativeGen, cp.r) == [cp.mult_gen]
    finally:
        d.close()


@pytest.mark.parametrize("c", CURVES)
def test_commit_open_and_batch_open(c):
    kzg = import_module("gnark-crypto_b200.kzg")
    g = c + "_g1"
    G = O.GROUPS[g]
    cp = kzg.CURVE_PARAMS[c]
    r = cp.r
    size, alpha = 700, 0x7654321FEDCBA9876543 % r
    gen = G.encode_affine([G.gen])[0]
    srs = kzg.new_srs_g1(c, size, alpha, gen, r, G.encode_scalars)
    pk = kzg.ProvingKey(c, srs)
    rng = np.random.default_rng(17)
    polys = [[int(x) for x in rng.integers(0, 2**62, size=m)] for m in (700, 513, 64)]
    polys[0][5] = r - 1
    enc = [G.encode_scalars(p) for p in polys]
    assert enc[0].shape[1] == cp.fr_words
    digests = [kzg.Commit(e, pk) for e in enc]
    for p, d in zip(polys, digests):
        assert np.array_equal(d, cref.scalar_mul(g, gen, _ev(p, alpha, r)))
    a = 0xABCDEF0123456789
    point = G.encode_scalars([a])[0]
    # Open: H = [(f(alpha) - f(a)) / (alpha - a)] G
    op = kzg.Open(enc[1], point, pk)
    fa = _ev(polys[1], a, r)
    assert np.array_equal(op.ClaimedValue, G.encode_scalars([fa])[0])
    assert np.array_equal(op.H, cref.scalar_mul(g, gen, (_ev(polys[1], alpha, r) - fa) * pow(alpha - a, -1, r) % r))
    extra = b"transcript-data"
    proof = kzg.BatchOpenSinglePoint(enc, digests, point, hashlib.sha256, pk, extra)
    assert np.array_equal(proof.ClaimedValues, G.encode_scalars([_ev(p, a, r) for p in polys]))
    h = hashlib.sha256()
    h.update(b"gamma")
    h.update(a.to_bytes(cp.fr_bytes, "big"))
    for d in digests:
        x, y = G.decode_affine(d.reshape(1, -1))[0]
        h.update(int(x).to_bytes(cp.fp_bytes, "big") + int(y).to_bytes(cp.fp_bytes, "big"))
    for p in polys:
        h.update(_ev(p, a, r).to_bytes(cp.fr_bytes, "big"))
    h.update(extra)
    gamma = int.from_bytes(h.digest(), "big") % r
    assert kzg.derive_gamma(point, digests, proof.ClaimedValues, hashlib.sha256, c, extra) == gamma
    fold_alpha = sum(pow(gamma, i, r) * _ev(p, alpha, r) for i, p in enumerate(polys)) % r
    fold_a = sum(pow(gamma, i, r) * _ev(p, a, r) for i, p in enumerate(polys)) % r
    assert np.array_equal(proof.H, cref.scalar_mul(g, gen, (fold_alpha - fold_a) * pow(alpha - a, -1, r) % r))
    op, folded = kzg.FoldProof(digests, proof, point, hashlib.sha256, c, extra)
    assert np.array_equal(folded, cref.scalar_mul(g, gen, fold_alpha))
    assert np.array_equal(op.ClaimedValue, G.encode_scalars([fold_a])[0]) and np.array_equal(op.H, proof.H)
    with pytest.raises(kzg.ErrInvalidPolynomialSize):
        kzg.Commit(G.encode_scalars([1] * (size + 1)), pk)
    pk.close()


@pytest.mark.parametrize("c", CURVES)
def test_commit_lagrange(c):
    """evaluations -> FFTInverse + BitReverse on the device -> MultiExp over resident bases == Commit of the host iFFT"""
    kzg = import_module("gnark-crypto_b200.kzg")
    fft = import_module("gnark-crypto_b200.fft")
    g = c + "_g1"
    G = O.GROUPS[g]
    r = kzg.CURVE_PARAMS[c].r
    size, alpha = 1024, 0xBEEF1234567
    gen = G.encode_affine([G.gen])[0]
    pk = kzg.ProvingKey(c, kzg.new_srs_g1(c, size, alpha, gen, r, G.encode_scalars))
    dom = fft.NewDomain(c, size)
    rng = np.random.default_rng(5)
    evals = G.encode_scalars([int(x) for x in rng.integers(0, 2**62, size=size)])
    coeffs = dom.FFTInverse(evals.copy(), fft.DIF)       # natural in, bit-reversed out (host buffer)
    idx = np.array([int(format(i, "010b")[::-1], 2) for i in range(size)])
    coeffs = np.ascontiguousarray(coeffs[idx])            # BitReverse on the host: natural-order coefficients
    digest = kzg.CommitLagrange(evals, pk, dom)
    assert np.array_equal(digest, kzg.Commit(coeffs, pk))
    f_alpha = _ev(curves._fr_decode(coeffs, r), alpha, r)
    assert np.array_equal(digest, cref.scalar_mul(g, gen, f_alpha))
    pk.close()
    dom.close()


@pytest.mark.parametrize("c", CURVES)
def test_device_point_decoding(c):
    """gmsm_g1_decode of compressed and raw streams (with infinity points, both signs of y) == the original points; the
    resident bases straight from the bytes commit like the oracle MSM; bad points carry the reference's message and index"""
    kzg = import_module("gnark-crypto_b200.kzg")
    g = c + "_g1"
    G = O.GROUPS[g]
    cp = kzg.CURVE_PARAMS[c]
    f = cp.flags
    n = 2000
    pts = cref.generate_multiples(g, G.encode_affine([G.gen])[0], 11, n, nthreads=4)
    pts[5] = 0
    pts[n - 1] = 0
    comp = b"".join(kzg.g1_bytes(p, c) for p in pts)
    raw = b"".join(kzg.g1_raw_bytes(p, c) for p in pts)
    nb = cp.fp_bytes
    assert {comp[i * nb] & f["mask"] for i in range(n)} == {f["small"], f["large"], f["inf"]}
    assert np.array_equal(kzg.decode_g1_points(c, comp, n, raw=False), pts)
    assert np.array_equal(kzg.decode_g1_points(c, raw, n, raw=True), pts)
    pk = kzg.ProvingKey.from_bytes(c, comp, n)
    s = cref.random_scalars(g, n, 3)
    want, _, _, _ = cref.msm(g, pts, s, c=0, nthreads=4)
    assert np.array_equal(kzg.Commit(s, pk), want)
    pk.close()
    x = 1
    while pow((x ** 3 + cp.b) % cp.q, (cp.q - 1) // 2, cp.q) != cp.q - 1:
        x += 1
    bad = bytearray(comp)
    xb = bytearray(x.to_bytes(nb, "big"))
    xb[0] |= f["small"]
    bad[7 * nb:8 * nb] = xb
    with pytest.raises(kzg.MultiExpError, match="point 7: invalid compressed coordinate: square root doesn't exist"):
        kzg.decode_g1_points(c, bytes(bad), n, raw=False)
    bad = bytearray(raw)
    bad[9 * 2 * nb + 2 * nb - 1] ^= 1                   # y of point 9 off the curve
    with pytest.raises(kzg.MultiExpError, match="point 9: invalid point"):
        kzg.decode_g1_points(c, bytes(bad), n, raw=True)
    assert kzg.decode_g1_points(c, bytes(bad), n, raw=True, check_on_curve=False).shape == pts.shape
    bad = bytearray(comp)
    bad[5 * nb + 3] = 1                                 # infinity flag with a non-zero byte
    with pytest.raises(kzg.MultiExpError, match="point 5: invalid infinity point encoding"):
        kzg.decode_g1_points(c, bytes(bad), n, raw=False)
    bad = bytearray(raw)
    bad[3 * 2 * nb:3 * 2 * nb + nb] = bytes([~f["mask"] & 0xFF]) + b"\xff" * (nb - 1)     # x >= q
    with pytest.raises(kzg.MultiExpError, match="point 3: invalid fp.Element encoding"):
        kzg.decode_g1_points(c, bytes(bad), n, raw=True)
    bad = bytearray(raw)
    bad[2 * 2 * nb] |= f["small"]                       # a compressed flag in a raw stream
    with pytest.raises(kzg.MultiExpError, match="point 2: invalid point encoding"):
        kzg.decode_g1_points(c, bytes(bad), n, raw=True)
