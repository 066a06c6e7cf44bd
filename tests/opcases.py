"""Shared op-level test vectors: element-wise field / point operations checked against the oracle.
Used by tests/test_hostcheck.py (CPU build of the arithmetic headers) and tests/test_gpu_ops.py
(the same operations executed by the sm_90a device code)."""
import random

import numpy as np

from oracle import oracle as O

OPS = dict(FMUL=0, FADD=1, FSUB=2, FSQR=3, FNEG=4, FDBL=5, FINV=6, ADD_MIXED=7, SUB_MIXED=8, ADD=9, DOUBLE=10, TO_AFFINE=11,
           FR_FROM_MONT=12, FDOT2=13)


def u32(a):
    return np.ascontiguousarray(a, dtype=np.uint64).view(np.uint32).reshape(a.shape[0], -1)


def enc_f(G, vals):
    return np.array([G.K.encode(v) for v in vals], dtype=np.uint64)


def dec_f(G, arr):
    arr = np.ascontiguousarray(arr, dtype=np.uint32).view(np.uint64)
    return [G.K.decode([int(x) for x in r]) for r in arr]


def enc_xyzz(G, pts):
    return np.array([sum((G.K.encode(c) for c in p), []) for p in pts], dtype=np.uint64)


def dec_xyzz(G, arr):
    arr = np.ascontiguousarray(arr, dtype=np.uint32).view(np.uint64)
    w = G.K.words
    return [[G.K.decode([int(x) for x in r[i * w : (i + 1) * w]]) for i in range(4)] for r in arr]


def field_values(G, rng, n):
    q = G.K.q
    f = G.K.f
    specials = [0, 1, q - 1, q - 2, f.Rmod, f.R2, (q - 1) // 2, (1 << (f.bits - 1)) % q, 0xFFFFFFFF, 1 << 32, (1 << 64) - 1]
    vals = specials + [rng.randrange(q) for _ in range(n)]
    if G.K.ext == 1:
        return vals
    return [(a, b) for a, b in zip(vals, reversed(vals))] + [(0, 0), (1, 0), (0, 1), (q - 1, q - 1)]


def random_xyzz(G, rng, k):
    """a non-trivial extended-Jacobian representation of [k]G: (x z^2, y z^3, z^2, z^3)"""
    K = G.K
    a = G.scalar_mul(G.gen, k)
    if G.aff_is_inf(a):
        return G.xyzz_inf()
    z = K.from_int(rng.randrange(1, K.q)) if K.ext == 1 else (rng.randrange(1, K.q), rng.randrange(K.q))
    zz = K.sqr(z)
    zzz = K.mul(zz, z)
    return [K.mul(a[0], zz), K.mul(a[1], zzz), zz, zzz]


def check_field_ops(G, run):
    """run(op, a_u32, b_u32 or None, out_words) -> u32 array"""
    K = G.K
    rng = random.Random(11)
    a = field_values(G, rng, 40)
    b = list(reversed(a))
    A, B = u32(enc_f(G, a)), u32(enc_f(G, b))
    w32 = 2 * K.words
    assert dec_f(G, run(OPS["FMUL"], A, B, w32)) == [K.mul(x, y) for x, y in zip(a, b)]
    assert dec_f(G, run(OPS["FADD"], A, B, w32)) == [K.add(x, y) for x, y in zip(a, b)]
    assert dec_f(G, run(OPS["FSUB"], A, B, w32)) == [K.sub(x, y) for x, y in zip(a, b)]
    assert dec_f(G, run(OPS["FSQR"], A, None, w32)) == [K.sqr(x) for x in a]
    assert dec_f(G, run(OPS["FNEG"], A, None, w32)) == [K.neg(x) for x in a]
    assert dec_f(G, run(OPS["FDBL"], A, None, w32)) == [K.dbl(x) for x in a]
    assert dec_f(G, run(OPS["FINV"], A[:12], None, w32)) == [K.inv(x) for x in a[:12]]
    # outputs are fully reduced Montgomery limbs: re-encoding the decoded value reproduces the bytes
    out = run(OPS["FMUL"], A, B, w32)
    assert np.array_equal(u32(enc_f(G, dec_f(G, out))), out)


def check_fr_from_mont(G, run):
    fr = G.fr
    rng = random.Random(5)
    vals = [0, 1, fr.q - 1, fr.Rmod] + [rng.randrange(fr.q) for _ in range(30)]
    A = u32(np.array([fr.to_limbs(v) for v in vals], dtype=np.uint64))
    out = run(OPS["FR_FROM_MONT"], A, None, 2 * fr.limbs)
    got = [O.Field.from_limbs([int(x) for x in r]) for r in np.ascontiguousarray(out).view(np.uint64)]
    assert got == [fr.from_mont(v) for v in vals]


def check_point_ops(G, run):
    K = G.K
    rng = random.Random(23)
    w32 = 2 * K.words
    ks = [1, 2, 3, 5, 7, 11, 100, G.fr.q - 1, G.fr.q - 2, rng.randrange(G.fr.q), rng.randrange(G.fr.q)]
    # (p, a) pairs: generic, p = inf, a = inf, p == a (doubling), p == -a (cancellation)
    ps, as_ = [], []
    for k1 in ks[:8]:
        for k2 in (1, 2, 5, k1, (G.fr.q - k1) % G.fr.q):
            ps.append(random_xyzz(G, rng, k1))
            as_.append(G.scalar_mul(G.gen, k2))
    ps.append(G.xyzz_inf()); as_.append(G.scalar_mul(G.gen, 9))
    ps.append([K.zero, K.zero, K.zero, K.zero]); as_.append(G.scalar_mul(G.gen, 9))  # all-zero infinity (memset buckets)
    ps.append(random_xyzz(G, rng, 9)); as_.append(G.aff_inf())
    ps.append(G.xyzz_inf()); as_.append(G.aff_inf())
    P, A = u32(enc_xyzz(G, ps)), u32(G.encode_affine(as_))
    for op, neg in (("ADD_MIXED", False), ("SUB_MIXED", True)):
        got = dec_xyzz(G, run(OPS[op], P, A, 4 * w32))
        for p, a, g in zip(ps, as_, got):
            want = G.add_mixed(list(p), a, negate=neg)
            assert G.xyzz_to_affine(g) == G.xyzz_to_affine(want)
            if not K.is_zero(want[2]):
                assert g == want  # the exact coordinates of the reference's formulas (g1.go:822-930)
    # full add / double
    qs = [random_xyzz(G, rng, k) for k in (1, 2, 5)] * (len(ps) // 3 + 1)
    qs = qs[: len(ps)]
    qs[0] = list(ps[0])                     # same representation -> doubling branch
    k0 = ks[1]
    ps[1], qs[1] = random_xyzz(G, rng, k0), random_xyzz(G, rng, k0)        # same point, different z -> doubling
    ps[2], qs[2] = random_xyzz(G, rng, k0), random_xyzz(G, rng, G.fr.q - k0)  # opposite -> infinity
    qs[3] = G.xyzz_inf()
    P, Q = u32(enc_xyzz(G, ps)), u32(enc_xyzz(G, qs))
    got = dec_xyzz(G, run(OPS["ADD"], P, Q, 4 * w32))
    for p, q, g in zip(ps, qs, got):
        want = G.xyzz_add(list(p), list(q))
        assert G.xyzz_to_affine(g) == G.xyzz_to_affine(want)
        if not K.is_zero(want[2]) and not K.is_zero(p[2]):
            assert g == want
    got = dec_xyzz(G, run(OPS["DOUBLE"], P, None, 4 * w32))
    for p, g in zip(ps, got):
        assert G.xyzz_to_affine(g) == G.xyzz_to_affine(G.xyzz_double(p))
    # normalisation: byte-exact affine normal form
    got = run(OPS["TO_AFFINE"], P[:10], None, 2 * w32)
    want = u32(G.encode_affine([G.xyzz_to_affine(p) for p in ps[:10]]))
    assert np.array_equal(got, want)
