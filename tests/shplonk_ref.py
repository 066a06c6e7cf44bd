"""Test references for shplonk.py / fflonk.py on Python ints:
  * `identity_open`: the device algorithm of shplonk.open_packs (chained divisions by (X - a), Newton coefficients, strided linear
    combinations, one division by (X - z)), so that the CPU tests can hold it against the line-by-line restatement of the reference
    (shplonk.batch_open_host) without a GPU;
  * a known-alpha SRS and its commitments from the oracle ([alpha^i]G by cref.scalar_mul, Commit by cref.msm);
  * BatchVerify in the exponent: with alpha known, e(F + z W', [1]) = e(W', [alpha]) is the G1 identity F = (alpha - z) W', with
    F = sum_i c_i D_i - [sum_i c_i r_i(z)] G - Z_T(z) W and c_i = gamma^i Z_{T\\S_i}(z) (shplonk.go:179-274), and fflonk's
    fold-consistency check (fflonk.go:153-193)."""
from importlib import import_module

import numpy as np

from oracle import cref
from oracle import oracle as O

curves = import_module("gnark-crypto_b200.curves")


def _mods():
    return import_module("gnark-crypto_b200.kzg"), import_module("gnark-crypto_b200.shplonk"), import_module("gnark-crypto_b200.fflonk")


def _div_x_minus_a(f, a, r):
    """(f(a), quotient of f by (X - a)) -- what one gmsm_fr_poly_div_x_minus_a_device call returns"""
    b, q = 0, [0] * max(len(f) - 1, 0)
    for i in range(len(f) - 1, -1, -1):
        b = (f[i] + a * b) % r
        if i:
            q[i - 1] = b
    return b, q


def _lincomb(terms, out_len, r):
    out = [0] * out_len
    for p, s, st, off in terms:
        for m, v in enumerate(p):
            if m * st + off < out_len:
                out[m * st + off] = (out[m * st + off] + s * v) % r
    return out


def identity_open(packs, base_points, ts, ext_points, digests, hf, curve, commit, *data):
    """shplonk.open_packs with Python ints for the device work -> (W, W', claimed, outer values, w, w')"""
    kzg, shplonk, _ = _mods()
    r = kzg.CURVE_PARAMS[curve].r
    max_size, nb_points = shplonk._sizes([t * max((len(p) for p in pack), default=0) for pack, t in zip(packs, ts)], ext_points)
    fs = shplonk._transcript(hf, ext_points, digests, curve, data)
    gamma = curves._challenge(fs, "gamma", r)
    terms, values = [], []
    for j, (pack, S, t) in enumerate(zip(packs, base_points, ts)):
        ys = [pow(s, t, r) for s in S]
        vals = []
        for i, f in enumerate(pack):
            cur, newton = list(f), []
            for a in ys:
                if cur:
                    fa, cur = _div_x_minus_a(cur, a, r)
                else:
                    fa = 0
                newton.append(fa)
            terms.append((cur, pow(gamma, j, r), t, i))
            row = []
            for m, ym in enumerate(ys):
                acc, basis = 0, 1
                for l in range(m + 1):
                    acc = (acc + newton[l] * basis) % r
                    basis = basis * (ym - ys[l]) % r
                row.append(acc)
            vals.append(row)
        values.append(vals)
    w = _lincomb(terms, max_size, r)
    W = commit(w)
    fs.Bind("z", kzg.g1_raw_bytes(W, curve))
    z = curves._challenge(fs, "z", r)
    zt_z = 1
    for S in ext_points:
        for x in S:
            zt_z = zt_z * (z - x) % r
    lterms = []
    for j, (pack, t) in enumerate(zip(packs, ts)):
        cj = pow(gamma, j, r)
        for k, S in enumerate(ext_points):
            if k != j:
                for x in S:
                    cj = cj * (z - x) % r
        lterms += [(f, cj, t, i) for i, f in enumerate(pack)]
    lterms.append((w, -zt_z % r, 1, 0))
    _, wprime = _div_x_minus_a(_lincomb(lterms, max_size, r), z, r)
    wprime += [0] * (max_size + nb_points - 1 - len(wprime))        # the reference's length: zeros past maxSizePolys - 1
    WPrime = commit(wprime)
    claimed = []
    for vals, t, S in zip(values, ts, ext_points):
        claimed.append([sum(pow(x, i, r) * row[idx // t] for i, row in enumerate(vals)) % r for idx, x in enumerate(S)])
    return W, WPrime, claimed, values, w, wprime


class OracleSRS:
    """[alpha^i]G, i < n, for curve's G1 and kzg.Commit on it through the oracle's MultiExp (with Commit's size checks)"""

    def __init__(self, curve, n, alpha):
        kzg, _, _ = _mods()
        self.curve, self.g = curve, curve + "_g1"
        G = O.GROUPS[self.g]
        self.r = kzg.CURVE_PARAMS[curve].r
        self.alpha = alpha % self.r
        self.gen = G.encode_affine([G.gen])[0]
        self.G = G
        self.points = np.stack([cref.scalar_mul(self.g, self.gen, pow(self.alpha, i, self.r)) for i in range(n)])

    def commit(self, coeffs):
        kzg, _, _ = _mods()
        if len(coeffs) == 0 or len(coeffs) > self.points.shape[0]:
            raise kzg.ErrInvalidPolynomialSize("invalid polynomial size (larger than SRS or == 0)")
        aff, _, _, _ = cref.msm(self.g, self.points[:len(coeffs)], self.G.encode_scalars(list(coeffs)))
        return aff

    def mul(self, k):
        return cref.scalar_mul(self.g, self.gen, k % self.r)


def _ev(f, x, r):
    acc = 0
    for v in reversed(f):
        acc = (acc * x + v) % r
    return acc


def verify_in_exponent(polys, points, proof_W, proof_WPrime, claimed, digests, hf, curve, alpha, *data):
    """shplonk.BatchVerify with a known alpha: True when F = (alpha - z) W' in G1.  The digests are the commitments [f_i(alpha)]G, so
    sum_i c_i D_i = [sum_i c_i f_i(alpha)]G and every term is a multiple of G: compare the scalars of F and (alpha - z) W' by
    building both points from their discrete logarithms, where W and W' enter as the points of the proof (their logarithms are
    w(alpha) and w'(alpha) only if the proof is honest, so the check is on the points, not on assumed logarithms)."""
    kzg, shplonk, _ = _mods()
    cp = kzg.CURVE_PARAMS[curve]
    r = cp.r
    g = curve + "_g1"
    G = O.GROUPS[g]
    fs = shplonk._transcript(hf, points, digests, curve, data)
    gamma = curves._challenge(fs, "gamma", r)
    fs.Bind("z", kzg.g1_raw_bytes(proof_W, curve))
    z = curves._challenge(fs, "z", r)
    gen = G.encode_affine([G.gen])[0]
    acc, sum_cr, coeffs = 1, 0, []
    for i in range(len(points)):
        ci = acc * shplonk._eval(shplonk._zt_minus_si(points, i, r), z, r) % r
        ri = shplonk._interpolate(points[i], claimed[i], r)
        sum_cr = (sum_cr + ci * shplonk._eval(ri, z, r)) % r
        coeffs.append(ci)
        acc = acc * gamma % r
    ztz = shplonk._eval(shplonk._vanishing([x for S in points for x in S], r), z, r)
    # F = sum c_i D_i - [sum c_i r_i(z)] G - Z_T(z) W ; check F + z W' - alpha W' = 0 as one MultiExp over the proof's points
    pts = np.stack([np.asarray(d, dtype=np.uint64).reshape(-1) for d in digests] + [gen, proof_W, proof_WPrime])
    sc = coeffs + [-sum_cr % r, -ztz % r, (z - alpha) % r]
    aff, _, _, _ = cref.msm(g, pts, G.encode_scalars(sc))
    return not aff.any()


def fflonk_fold_consistent(outer, inner, points, curve):
    """fflonk.BatchVerify's step 0 and 1 (fflonk.go:153-193) on ints: outer[j][k][m], inner[j][m t + l]"""
    kzg, _, fflonk = _mods()
    r = kzg.CURVE_PARAMS[curve].r
    for j, vals in enumerate(outer):
        t = len(vals)
        size = len(vals[0])
        if any(len(v) != size for v in vals) or size * t != len(inner[j]):
            return False
        omega = fflonk._ith_root_one(t, curve)
        for m in range(size):
            x = points[j][m]
            for l in range(t):
                if _ev([v[m] for v in vals], x, r) != inner[j][m * t + l]:
                    return False
                x = x * omega % r
    return True
