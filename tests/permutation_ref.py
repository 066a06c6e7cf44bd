"""Test references for permutation.py on Python ints (regular, not Montgomery), restating ecc/bn254/fr/permutation/permutation.go line
by line; the permutation packages of the other six pairing curves are the same generated code.
  * `batch_invert`, `accumulate`, `first_part`, `second_part`, `fold`: the Fr steps that the device kernels replace;
  * `prove`: Prove (:124-262) with the oracle's FFT (oracle.FFTDomain) and closed-form digests [f(alpha)]G of a known-alpha SRS, so
    that it shares neither MSM nor FFT with the code under test;
  * `verify`: Verify (:265-347) without the pairings: the Fr relation at eta, BatchVerifySinglePoint and kzg.Verify checked as
    C - [y]G = [alpha - a]H in G1, and the generator-order check."""
import hashlib
from importlib import import_module

import numpy as np

from oracle import cref
from oracle import oracle as O
from tests import fft_more_fields as M

curves = import_module("gnark-crypto_b200.curves")

DIT, DIF = O.DIT, O.DIF


def _kzg():
    return import_module("gnark-crypto_b200.kzg")


def domain(c, n):
    """the oracle's fft.Domain of n over the scalar field of c"""
    name = c + "_fr"
    return (O.FFTDomain if name in O.FFT_PARAMS else M.FFTDomain)(name, n)


def rev(i, n):
    lg = n.bit_length() - 1
    return int(bin(i)[2:].zfill(lg)[::-1], 2) if lg else 0


def batch_invert(a, r):
    """fr.BatchInvert (fr/element.go:658-687): zero -> zero"""
    res = [0] * len(a)
    acc = 1
    for i, v in enumerate(a):
        if v == 0:
            continue
        res[i] = acc
        acc = acc * v % r
    acc = pow(acc, r - 2, r)
    for i in range(len(a) - 1, -1, -1):
        if a[i] == 0:
            continue
        res[i] = res[i] * acc % r
        acc = acc * a[i] % r
    return res


def accumulate(t1, t2, eps, r):
    """evaluateAccumulationPolynomialBitReversed (permutation.go:52-75)"""
    s = len(t1)
    z, d = [0] * s, [0] * s
    z[0] = d[0] = 1
    for i in range(s - 1):
        _i, _ii = rev(i, s), rev((i + 1) % s, s)
        z[_ii] = z[_i] * (eps - t1[i]) % r
        d[i + 1] = d[i] * (eps - t2[i]) % r
    d = batch_invert(d, r)
    for i in range(s - 1):
        _ii = rev((i + 1) % s, s)
        z[_ii] = z[_ii] * d[i + 1] % r
    return z


def first_part(lt1, lt2, lz, eps, r):
    """evaluateFirstPartNumReverse (permutation.go:78-98)"""
    s = len(lt1)
    res = [0] * s
    for i in range(s):
        _i, _ii = rev(i, s), rev((i + 1) % s, s)
        a = lz[_ii] * (eps - lt2[_i]) % r
        b = lz[_i] * (eps - lt1[_i]) % r
        res[_i] = (a - b) % r
    return res


def second_part(lz, n, g, w, r):
    """evaluateSecondPartNumReverse (permutation.go:101-121): g = FrMultiplicativeGen, w = the domain's Generator"""
    tn = (pow(g, n, r) - 1) % r
    u, x = [], g
    for _ in range(n):
        u.append((x - 1) % r)
        x = x * w % r
    u = batch_invert(u, r)
    res = [0] * n
    for i in range(n):
        _i = rev(i, n)
        res[_i] = (lz[_i] - 1) * u[i] % r * tn % r
    return res


def fold(first, second, omega, n, g, r):
    """the omega-fold and the division by g^n - 1 (permutation.go:206-214)"""
    t = pow((pow(g, n, r) - 1) % r, r - 2, r)
    return [(omega * s + f) % r * t % r for f, s in zip(first, second)]


def numerator(lt1, lt2, lz, eps, omega, n, g, w, r):
    return fold(first_part(lt1, lt2, lz, eps, r), second_part(lz, n, g, w, r), omega, n, g, r)


def _ev(f, x, r):
    acc = 0
    for v in reversed(f):
        acc = (acc * x + v) % r
    return acc


class ClosedFormSRS:
    """kzg.Commit on the SRS [alpha^i]G as the closed form [f(alpha)]G (one oracle scalar multiplication), with Commit's size checks"""

    def __init__(self, curve, size, alpha):
        self.curve, self.g = curve, curve + "_g1"
        G = O.GROUPS[self.g]
        self.r = _kzg().CURVE_PARAMS[curve].r
        self.alpha, self.size = alpha % self.r, size
        self.gen = G.encode_affine([G.gen])[0]
        self.G = G

    def commit(self, coeffs):
        if len(coeffs) == 0 or len(coeffs) > self.size:
            raise _kzg().ErrInvalidPolynomialSize("invalid polynomial size (larger than SRS or == 0)")
        return self.mul(_ev(coeffs, self.alpha, self.r))

    def mul(self, k):
        return cref.scalar_mul(self.g, self.gen, k % self.r)


def _challenge(fs, name, r):
    return int.from_bytes(fs.ComputeChallenge(name), "big") % r


def _transcript():
    return import_module("gnark-crypto_b200.transcript").Transcript(hashlib.sha256, "epsilon", "omega", "eta")


def _batch_open(polys, digests, eta, srs, curve):
    """kzg.BatchOpenSinglePoint (kzg.go:246-331) -> (H, claimed values)"""
    kzg = _kzg()
    r = srs.r
    claimed = [_ev(f, eta, r) for f in polys]
    gamma = kzg.derive_gamma(curves._fr_encode([eta], r)[0], digests, curves._fr_encode(claimed, r), hashlib.sha256, curve)
    largest = max(len(f) for f in polys)
    folded, g = [0] * largest, 1
    for f in polys:
        for j, v in enumerate(f):
            folded[j] = (folded[j] + v * g) % r
        g = g * gamma % r
    fe = _ev(folded, eta, r)
    h = kzg._divide_by_x_minus_a(folded, fe, eta, r)
    return srs.commit(h), claimed


def prove(curve, t1, t2, srs):
    """Prove (permutation.go:124-262) -> dict of the proof's fields (digests as limbs, values as ints) and the intermediates"""
    kzg = _kzg()
    r = srs.r
    if len(t1) != len(t2):
        raise ValueError("t1 and t2 should be of the same size")
    d = domain(curve, len(t1))
    if d.cardinality != len(t1):
        raise ValueError("t1 and t2 should be of size a power of 2")
    s = d.cardinality
    fs = _transcript()
    ct1 = d.fft_inverse(list(t1), DIF)
    ct2 = d.fft_inverse(list(t2), DIF)
    ct1 = [ct1[rev(i, s)] for i in range(s)]                     # fft.BitReverse
    ct2 = [ct2[rev(i, s)] for i in range(s)]
    T1, T2 = srs.commit(ct1), srs.commit(ct2)
    for p in (T1, T2):
        fs.Bind("epsilon", kzg.g1_raw_bytes(p, curve))
    eps = _challenge(fs, "epsilon", r)
    cz = d.fft_inverse(accumulate(t1, t2, eps, r), DIT)
    Z = srs.commit(cz)
    lz = d.fft(cz, DIF, coset=True)
    lt1 = d.fft(ct1, DIF, coset=True)
    lt2 = d.fft(ct2, DIF, coset=True)
    fs.Bind("omega", kzg.g1_raw_bytes(Z, curve))
    omega = _challenge(fs, "omega", r)
    num = numerator(lt1, lt2, lz, eps, omega, s, d.shift, d.generator, r)
    q = d.fft_inverse(num, DIT, coset=True)
    Q = srs.commit(q)
    fs.Bind("eta", kzg.g1_raw_bytes(Q, curve))
    eta = _challenge(fs, "eta", r)
    H, claimed = _batch_open([ct1, ct2, cz, q], [T1, T2, Z, Q], eta, srs, curve)
    shifted = eta * d.generator % r
    zs = _ev(cz, shifted, r)
    Hs = srs.commit(kzg._divide_by_x_minus_a(cz, zs, shifted, r))
    return dict(size=s, g=d.generator, t1=T1, t2=T2, z=Z, q=Q, H=H, claimed=claimed, Hs=Hs, zs=zs,
                eps=eps, omega=omega, eta=eta, ct1=ct1, ct2=ct2, cz=cz, quotient=q)


def verify(curve, proof, alpha):
    """Verify (permutation.go:265-347) of a permutation.Proof with the pairings replaced by G1 identities under a known alpha"""
    kzg = _kzg()
    cp = kzg.CURVE_PARAMS[curve]
    r = cp.r
    G = O.GROUPS[curve + "_g1"]
    gen = G.encode_affine([G.gen])[0]
    fs = _transcript()
    for p in (proof.t1, proof.t2):
        fs.Bind("epsilon", kzg.g1_raw_bytes(p, curve))
    eps = _challenge(fs, "epsilon", r)
    fs.Bind("omega", kzg.g1_raw_bytes(proof.z, curve))
    omega = _challenge(fs, "omega", r)
    fs.Bind("eta", kzg.g1_raw_bytes(proof.q, curve))
    eta = _challenge(fs, "eta", r)
    cl = curves._fr_decode(proof.batchedProof.ClaimedValues, r)
    zs = curves._fr_decode(proof.shiftedProof.ClaimedValue, r)[0]
    # the relation at eta (:293-311)
    rhs = (pow(eta, proof.size, r) - 1) % r
    l0 = rhs * pow((eta - 1) % r, r - 2, r) % r
    rhs = rhs * cl[3] % r
    a = (eps - cl[1]) * zs % r
    b = (eps - cl[0]) * cl[2] % r
    lhs = ((a - b) + (cl[2] - 1) * l0 % r * omega) % r
    if lhs != rhs:
        return False
    digests = [proof.t1, proof.t2, proof.z, proof.q]

    def opening_holds(digest_terms, y, point, H):
        # e(C - [y]G + [point]H, [1]) = e(H, [alpha]): C - [y]G - [alpha - point]H = 0
        pts = np.stack([np.asarray(p, dtype=np.uint64).reshape(-1) for p, _ in digest_terms] + [gen, np.asarray(H, dtype=np.uint64)])
        sc = [k for _, k in digest_terms] + [-y % r, (point - alpha) % r]
        aff, _, _, _ = cref.msm(curve + "_g1", pts, G.encode_scalars(sc))
        return not aff.any()

    # BatchVerifySinglePoint (kzg.go:420-470): fold the digests and values with gamma
    gamma = kzg.derive_gamma(curves._fr_encode([eta], r)[0], digests, proof.batchedProof.ClaimedValues, hashlib.sha256, curve)
    gam = [pow(gamma, i, r) for i in range(4)]
    if not opening_holds(list(zip(digests, gam)), sum(g * v for g, v in zip(gam, cl)) % r, eta, proof.batchedProof.H):
        return False
    g = curves._fr_decode(proof.g, r)[0]
    if not opening_holds([(proof.z, 1)], zs, eta * g % r, proof.shiftedProof.H):
        return False
    # the generator's order (:333-344)
    c = pow(g, proof.size // 2, r)
    return c != 1 and c * c % r == 1
