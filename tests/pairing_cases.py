"""Shared inputs of the pairing tests: random pairs, infinity patterns and off-subgroup bn254 G2 points, as restatement values
(tests/pairing_ref.py) and the reference's memory layout."""
import random

import numpy as np

from tests import pairing_ref as PR


def random_pairs(curve: str, n: int, seed: int):
    T = PR.tower(curve)
    rng = random.Random(seed)
    P = [T.G1.scalar_mul(T.G1.gen, rng.randrange(1, T.r)) for _ in range(n)]
    Q = [T.G2.scalar_mul(T.G2.gen, rng.randrange(1, T.r)) for _ in range(n)]
    return P, Q


def encode_pairs(curve: str, P, Q):
    T = PR.tower(curve)
    return np.ascontiguousarray(T.G1.encode_affine(P)), np.ascontiguousarray(T.G2.encode_affine(Q))


def off_subgroup_g2(n: int, seed: int):
    """bn254 twist points outside the r-torsion: random x until x^3 + b' is a square in Fp2, kept when [r]Q is not infinity"""
    T = PR.tower("bn254")
    q = T.q
    rng = random.Random(seed)
    out = []
    while len(out) < n:
        x = (rng.randrange(q), rng.randrange(q))
        rhs = T.e2_add(T.e2_mul(T.e2_sqr(x), x), T.btwist)
        y = _e2_sqrt(T, rhs)
        if y is None:
            continue
        pt = (x, y)
        if T.G2.scalar_mul(pt, T.r) != T.G2.aff_inf():
            out.append(pt)
    return out


def _e2_sqrt(T, a):
    """a square root in Fp2 (q = 3 mod 4), or None"""
    q = T.q
    nrm = (a[0] * a[0] + a[1] * a[1]) % q
    if pow(nrm, (q - 1) // 2, q) not in (0, 1):
        return None
    # complex method: y = sqrt((a0 + sqrt(nrm)) / 2) + a1 / (2 y) u
    s = pow(nrm, (q + 1) // 4, q)
    for cand in ((a[0] + s) % q, (a[0] - s) % q):
        t = cand * pow(2, -1, q) % q
        y0 = pow(t, (q + 1) // 4, q)
        if y0 * y0 % q != t or y0 == 0:
            continue
        y1 = a[1] * pow(2 * y0, -1, q) % q
        y = (y0, y1)
        if T.e2_sqr(y) == (a[0] % q, a[1] % q):
            return y
    return None
