"""Test references for plookup.py on Python ints (regular, not Montgomery), restating ecc/bn254/fr/plookup/vector.go and table.go line
by line; the plookup packages of the other six pairing curves are the same generated code.
  * `sort`, `accumulate`, `num_bit_reversed`, `z_starts_by_one`, `z_ends_by_one`, `overlap_h1h2`, `quotient_fold`: the Fr steps that
    the device kernels replace (`numerator` chains the last five);
  * `prove_vector` (ProveLookupVector, vector.go:345-550) and `prove_tables` (ProveLookupTables, table.go:52-166) with the oracle's
    FFT and closed-form digests [f(alpha)]G of a known-alpha SRS (permutation_ref.ClosedFormSRS), so that they share neither MSM nor
    FFT with the code under test;
  * `verify_vector` (VerifyLookupVector, vector.go:553-706) and `verify_tables` (VerifyLookupTables, table.go:169-220) without the
    pairings: the Fr relation at nu, BatchVerifySinglePoint checked as C - [y]G = [alpha - a]H in G1, the generator-order check, the
    digest fold, and permutation_ref.verify for the inner permutation proof."""
import hashlib
from importlib import import_module

import numpy as np

from oracle import cref
from oracle import oracle as O
from tests import permutation_ref as P

curves = import_module("gnark-crypto_b200.curves")

DIT, DIF = O.DIT, O.DIF
rev, domain, batch_invert, ClosedFormSRS = P.rev, P.domain, P.batch_invert, P.ClosedFormSRS


def _kzg():
    return import_module("gnark-crypto_b200.kzg")


def sort(v):
    """sort.Sort(fr.Vector): ascending by canonical value (fr.Element.Cmp)"""
    return sorted(v)


def accumulate(lf, lt, lh1, lh2, beta, gamma, r):
    """evaluateAccumulationPolynomial (vector.go:52-95), natural order"""
    n = len(lt)
    c = (1 + beta) * gamma % r
    d = [(beta * lh1[i + 1] + lh1[i] + c) * (beta * lh2[i + 1] + lh2[i] + c) % r for i in range(n - 1)]
    d = batch_invert(d, r)
    z = [0] * n
    z[0] = 1
    e = (1 + beta) % r
    for i in range(n - 1):
        a = (gamma + lf[i]) * (beta * lt[i + 1] + lt[i] + c) % r * e % r
        z[i + 1] = z[i] * a % r * d[i] % r
    return z


def _coset_points(s, shift, w, r):
    g, x = [], shift
    for _ in range(s):
        g.append(x)
        x = x * w % r
    return g


def _gg(s, w, r):
    """(w^2)^(s/2 - 1) (vector.go:124-126)"""
    return pow(w * w % r, s // 2 - 1, r)


def num_bit_reversed(lz, lh1, lh2, lt, lf, beta, gamma, s, shift, w, r):
    """evaluateNumBitReversed (vector.go:106-162); s = the big domain's cardinality, w its generator"""
    opb = (1 + beta) % r
    gopb = opb * gamma % r
    g = _coset_points(s, shift, w, r)
    gg = _gg(s, w, r)
    num = [0] * s
    for i in range(s):
        _i, _is = rev(i, s), rev((i + 2) % s, s)
        m = opb * lz[_i] % r * ((gamma + lf[_i]) % r) % r * ((beta * lt[_is] + lt[_i] + gopb) % r) % r
        n = (beta * lh1[_is] + lh1[_i] + gopb) * (beta * lh2[_is] + lh2[_i] + gopb) % r * lz[_is] % r
        num[_i] = (m - n) * (g[i] - gg) % r
    return num


def xn_minus_one(s, shift, r):
    """evaluateXnMinusOneDomainBig (vector.go:165-181)"""
    sh = pow(shift, s // 2, r)
    return [(sh - 1) % r, -(sh + 1) % r]


def z_starts_by_one(lz, s, shift, w, r):
    """evaluateZStartsByOneBitReversed (vector.go:234-253)"""
    xn = xn_minus_one(s, shift, r)
    den = batch_invert([(x - 1) % r for x in _coset_points(s, shift, w, r)], r)
    res = [0] * s
    for i in range(s):
        _i = rev(i, s)
        res[_i] = (lz[_i] - 1) * xn[i % 2] % r * den[i] % r
    return res


def _den_ln(s, shift, w, r):
    gg = _gg(s, w, r)
    return batch_invert([(x - gg) % r for x in _coset_points(s, shift, w, r)], r)


def z_ends_by_one(lz, s, shift, w, r):
    """evaluateZEndsByOneBitReversed (vector.go:256-274)"""
    xn, den = xn_minus_one(s, shift, r), _den_ln(s, shift, w, r)
    res = [0] * s
    for i in range(s):
        _i = rev(i, s)
        res[_i] = (lz[_i] - 1) * xn[i % 2] % r * den[i] % r
    return res


def overlap_h1h2(lh1, lh2, s, shift, w, r):
    """evaluateOverlapH1h2BitReversed (vector.go:277-299)"""
    xn, den = xn_minus_one(s, shift, r), _den_ln(s, shift, w, r)
    res = [0] * s
    for i in range(s):
        _i, _is = rev(i, s), rev((i + 2) % s, s)
        res[_i] = (lh1[_i] - lh2[_is]) * xn[i % 2] % r * den[i] % r
    return res


def quotient_fold(alpha, lh, lh0, lhn, lh1h2, s, shift, r):
    """computeQuotientCanonical (vector.go:306-335) up to its FFTInverse"""
    inv = [pow(v, r - 2, r) for v in xn_minus_one(s, shift, r)]
    res = [0] * s
    for i in range(s):
        _i = rev(i, s)
        res[_i] = (((lh1h2[_i] * alpha + lhn[_i]) * alpha + lh0[_i]) * alpha + lh[_i]) % r * inv[i % 2] % r
    return res


def numerator(lz, lh1, lh2, lt, lf, beta, gamma, alpha, s, shift, w, r):
    lh = num_bit_reversed(lz, lh1, lh2, lt, lf, beta, gamma, s, shift, w, r)
    return quotient_fold(alpha, lh, z_starts_by_one(lz, s, shift, w, r), z_ends_by_one(lz, s, shift, w, r),
                         overlap_h1h2(lh1, lh2, s, shift, w, r), s, shift, r)


def _transcript(*names):
    return import_module("gnark-crypto_b200.transcript").Transcript(hashlib.sha256, *names)


def _challenge(fs, name, curve, r, *digests):
    kzg = _kzg()
    for p in digests:
        fs.Bind(name, kzg.g1_raw_bytes(p, curve))
    return int.from_bytes(fs.ComputeChallenge(name), "big") % r


def _coeffs(d, v):
    """FFTInverse(DIF) + BitReverse"""
    c = d.fft_inverse(list(v), DIF)
    return [c[rev(i, len(c))] for i in range(len(c))]


def prove_vector(curve, f, t, srs):
    """ProveLookupVector (vector.go:345-550) -> dict of the proof's fields (digests as limbs, values as ints)"""
    r = srs.r
    if not f or not t:
        raise ValueError("f and t must not be empty")
    fs = _transcript("beta", "gamma", "alpha", "nu")
    d = domain(curve, len(f) + 1 if len(t) <= len(f) else len(t))
    s = d.cardinality
    lf = list(f) + [f[-1]] * (s - len(f))
    lt = sort(list(t) + [t[-1]] * (s - len(t)))
    ct, cf = _coeffs(d, lt), _coeffs(d, lf)
    T, F = srs.commit(ct), srs.commit(cf)
    h = sort(lt + lf[:s - 1])
    lh1, lh2 = h[:s], h[s - 1:]
    ch1, ch2 = _coeffs(d, lh1), _coeffs(d, lh2)
    H1, H2 = srs.commit(ch1), srs.commit(ch2)
    beta = _challenge(fs, "beta", curve, r, T, F, H1, H2)
    gamma = _challenge(fs, "gamma", curve, r)
    lz = accumulate(lf, lt, lh1, lh2, beta, gamma, r)
    cz = _coeffs(d, lz)
    Z = srs.commit(cz)
    db = domain(curve, 2 * s)
    big = [db.fft(c + [0] * s, DIF, coset=True) for c in (cz, ch1, ch2, ct, cf)]
    alpha = _challenge(fs, "alpha", curve, r, Z)
    num = numerator(*big, beta, gamma, alpha, 2 * s, db.shift, db.generator, r)
    ch = db.fft_inverse(num, DIT, coset=True)
    Hd = srs.commit(ch)
    nu = _challenge(fs, "nu", curve, r, Hd)
    Hb, claimed = P._batch_open([ch1, ch2, ct, cz, cf, ch], [H1, H2, T, Z, F, Hd], nu, srs, curve)
    nus = nu * d.generator % r
    Hs, claimed_s = P._batch_open([ch1, ch2, ct, cz], [H1, H2, T, Z], nus, srs, curve)
    return dict(size=s, g=d.generator, h1=H1, h2=H2, t=T, z=Z, f=F, h=Hd, H=Hb, claimed=claimed, Hs=Hs, claimed_s=claimed_s,
                beta=beta, gamma=gamma, alpha=alpha, nu=nu, lt=lt, lh1=lh1, lh2=lh2, lz=lz)


def prove_tables(curve, f, t, srs):
    """ProveLookupTables (table.go:52-166) -> dict: fs, ts (digests), folded (prove_vector's dict), permutation (permutation_ref's)"""
    r = srs.r
    if not f or not t or not all(f) or not all(t):
        raise ValueError("f and t must not be empty")
    if len(f) != len(t) or any(len(row) != len(f[0]) for row in f) or any(len(row) != len(t[0]) for row in t):
        raise ValueError("the tables in f and t are not of the same size")
    fs = _transcript("lambda")
    d = domain(curve, max(len(f[0]) + 1, len(t[0])))
    nc = d.cardinality
    lfs = [list(row) + [row[-1]] * (nc - len(row)) for row in f]
    lts = [list(row) + [row[-1]] * (nc - len(row)) for row in t]
    Fs, Ts = [], []
    for lf, lt in zip(lfs, lts):
        Fs.append(srs.commit(_coeffs(d, lf)))
        Ts.append(srs.commit(_coeffs(d, lt)))
    lam = _challenge(fs, "lambda", curve, r, *Fs, *Ts)
    foldedf, foldedt = [0] * nc, [0] * nc
    for i in range(nc):
        for j in range(len(f) - 1, -1, -1):
            foldedf[i] = (foldedf[i] * lam + lfs[j][i]) % r
            foldedt[i] = (foldedt[i] * lam + lts[j][i]) % r
    perm = P.prove(curve, foldedt, sort(foldedt), srs)
    folded = prove_vector(curve, foldedf[:-1], foldedt, srs)
    return dict(fs=Fs, ts=Ts, folded=folded, permutation=perm, lam=lam)


def _opening_holds(curve, digest_terms, y, point, H, alpha):
    """e(C - [y]G + [point]H, [1]) = e(H, [alpha]) as C - [y]G - [alpha - point]H = 0 in G1"""
    G = O.GROUPS[curve + "_g1"]
    r = _kzg().CURVE_PARAMS[curve].r
    gen = G.encode_affine([G.gen])[0]
    pts = np.stack([np.asarray(p, dtype=np.uint64).reshape(-1) for p, _ in digest_terms] + [gen, np.asarray(H, dtype=np.uint64).reshape(-1)])
    sc = [k for _, k in digest_terms] + [-y % r, (point - alpha) % r]
    aff, _, _, _ = cref.msm(curve + "_g1", pts, G.encode_scalars(sc))
    return not aff.any()


def _batch_verify(curve, digests, proof, point, alpha):
    """kzg.BatchVerifySinglePoint (kzg.go:420-470) without the pairing"""
    kzg = _kzg()
    r = kzg.CURVE_PARAMS[curve].r
    cl = curves._fr_decode(proof.ClaimedValues, r)
    gamma = kzg.derive_gamma(curves._fr_encode([point], r)[0], digests, proof.ClaimedValues, hashlib.sha256, curve)
    gam = [pow(gamma, i, r) for i in range(len(digests))]
    return _opening_holds(curve, list(zip(digests, gam)), sum(g * v for g, v in zip(gam, cl)) % r, point, proof.H, alpha)


def verify_vector(curve, proof, alpha):
    """VerifyLookupVector (vector.go:553-706) of a plookup.ProofLookupVector with the pairings replaced by G1 identities"""
    r = _kzg().CURVE_PARAMS[curve].r
    fs = _transcript("beta", "gamma", "alpha", "nu")
    beta = _challenge(fs, "beta", curve, r, proof.t, proof.f, proof.h1, proof.h2)
    gamma = _challenge(fs, "gamma", curve, r)
    alph = _challenge(fs, "alpha", curve, r, proof.z)
    nu = _challenge(fs, "nu", curve, r, proof.h)
    if not _batch_verify(curve, [proof.h1, proof.h2, proof.t, proof.z, proof.f, proof.h], proof.BatchedProof, nu, alpha):
        return False
    g = curves._fr_decode(proof.g, r)[0]
    if not _batch_verify(curve, [proof.h1, proof.h2, proof.t, proof.z], proof.BatchedProofShifted, nu * g % r, alpha):
        return False
    c = pow(g, proof.size // 2, r)
    if c == 1 or c * c % r != 1:
        return False
    cv = curves._fr_decode(proof.BatchedProof.ClaimedValues, r)
    cs = curves._fr_decode(proof.BatchedProofShifted.ClaimedValues, r)
    gn = pow(g, proof.size - 1, r)
    v = (1 + beta) % r
    w = v * gamma % r
    lhs = (nu - gn) * cv[3] % r * v % r * ((gamma + cv[4]) % r) % r * ((beta * cs[2] + cv[2] + w) % r) % r
    rhs = (nu - gn) * cs[3] % r * ((beta * cs[0] + cv[0] + w) % r) % r * ((beta * cs[1] + cv[1] + w) % r) % r
    lhs = (lhs - rhs) % r
    l0 = (pow(nu, proof.size, r) - 1) % r
    ln = l0 * pow((nu - gn) % r, r - 2, r) % r
    l0 = l0 * pow((nu - 1) % r, r - 2, r) % r
    l0z = (cv[3] - 1) * l0 % r
    lnz = (cv[3] - 1) * ln % r
    lnh1h2 = (cv[0] - cs[1]) * ln % r
    lnh1h2 = (((lnh1h2 * alph + lnz) * alph + l0z) * alph + lhs) % r
    return lnh1h2 == (pow(nu, proof.size, r) - 1) * cv[5] % r


def verify_tables(curve, proof, alpha):
    """VerifyLookupTables (table.go:169-220) without the pairings"""
    r = _kzg().CURVE_PARAMS[curve].r
    if len(proof.fs) != len(proof.ts):
        return False
    lam = _challenge(_transcript("lambda"), "lambda", curve, r, *proof.fs, *proof.ts)
    G = O.GROUPS[curve + "_g1"]
    lams = G.encode_scalars([pow(lam, i, r) for i in range(len(proof.fs))])
    comf, _, _, _ = cref.msm(curve + "_g1", np.stack([np.asarray(p, dtype=np.uint64).reshape(-1) for p in proof.fs]), lams)
    if not np.array_equal(np.asarray(comf, dtype=np.uint64).reshape(-1), np.asarray(proof.foldedProof.f, dtype=np.uint64).reshape(-1)):
        return False
    if not P.verify(curve, proof.permutationProof, alpha):
        return False
    return verify_vector(curve, proof.foldedProof, alpha)
