"""Operands at which hand-written carry chains break, and the checks that run them.

Shared by tests/test_gpu_arith_stress.py (the sm_90a device code through the C ABI's test hooks) and
tests/test_arith_stress_cpu.py (the same routines built for the CPU, tests/test_hostcheck.py).  Not a conftest.

Field operands are STORED values: the Montgomery limbs the device reads (an integer m < q standing for the plain value
m R^-1 mod q).  The carries of a Montgomery product, a reduction or an addition depend on the stored limbs, so the extremes
are chosen there: 0, 1, q - 1, single bits at every 32-bit limb boundary, all-ones limbs, ...  The references are the
oracle's big-int operations (FpOps / Fp2Ops: K.mul, K.add, ...) on the plain values, re-encoded.  An output must equal the
reference limb for limb, which also makes it canonical (every component < q).

Scalars are plain values (the digit recoding reads the canonical scalar), encoded in Montgomery form as the engine reads them.
Failures name the group, the op, the index and the operands as decimal stored integers, so that a device-only failure can
be replayed through the CPU builds."""
import random

import numpy as np

from oracle import cref
from oracle import oracle as O
from tests.opcases import OPS

# ------------------------------------------------------------------------------------------
# generators
# ------------------------------------------------------------------------------------------


def _dedupe(vals):
    seen, out = set(), []
    for v in vals:
        if v not in seen:
            seen.add(v)
            out.append(v)
    return out


def field_extremes(f):
    """stored values < q of the field f (oracle.Field): the specials, 2^k, 2^k - 1 and q - 2^k for k at the lowest, second
    and highest bit of every 32-bit limb (and at the modulus' top bits), all-ones limb patterns with one limb cleared and
    single all-ones limbs -- everything reduced mod q"""
    q = f.q
    L = 2 * f.limbs
    vals = [0, 1, 2, q - 1, q - 2, f.Rmod, f.R2, (q - 1) // 2, (q + 1) // 2]
    ks = sorted({k for i in range(L) for k in (32 * i, 32 * i + 1, 32 * i + 31)} | {f.bits - 2, f.bits - 1, f.bits})
    for k in ks:
        vals += [(1 << k) % q, ((1 << k) - 1) % q, (q - (1 << k)) % q]
    top = (1 << (32 * L)) - 1
    for i in range(L):
        vals.append((top ^ (0xFFFFFFFF << (32 * i))) % q)
        vals.append((0xFFFFFFFF << (32 * i)) % q)
    return _dedupe(vals)


def fp2_components(G):
    """component values for Fp2 operands: the base-field extremes plus (-beta)^-1, the stored a1 whose beta-multiple
    -beta a1 (the operand the fused Fp2 product feeds to its reduction) is q - 1"""
    f = G.K.f
    return _dedupe(field_extremes(f) + [pow(-G.K.beta, -1, f.q)])


def fp2_corners(G):
    q = G.K.q
    ib = pow(-G.K.beta, -1, q)
    return [(q - 1, q - 1), (0, q - 1), (q - 1, 0), (q - 1, ib), (ib, q - 1), (1, 1)]


def coord_extremes(G):
    """one group's extreme coordinate-field elements: base-field extremes (Fp) or corners + extreme pairs (Fp2)"""
    E = field_extremes(G.K.f)
    if G.K.ext == 1:
        return E
    return _dedupe(fp2_corners(G) + [(a, a) for a in E] + [(a, 0) for a in E] + [(0, a) for a in E])


def sample_elements(G, rng, n):
    """n coordinate-field elements drawn from the extremes (Fp2: components drawn independently)"""
    if G.K.ext == 1:
        E = field_extremes(G.K.f)
        return [rng.choice(E) for _ in range(n)]
    C = fp2_components(G)
    return [(rng.choice(C), rng.choice(C)) for _ in range(n)]


def operand_pairs(G, rng, n_sample=1 << 16, all_pairs=True):
    """(x, y) operand pairs.  Fp: every ordered pair of extremes when all_pairs, otherwise every pair with one of the
    specials (0, 1, 2, q-1, q-2, R, R^2, (q -+ 1)/2) on either side, plus n_sample random pairs.  Fp2: every ordered pair
    of corners plus n_sample pairs with independently drawn components."""
    if G.K.ext == 1:
        E = field_extremes(G.K.f)
        if all_pairs:
            return [(x, y) for x in E for y in E]
        S = E[:9]
        pairs = [(x, y) for x in S for y in E] + [(y, x) for x in S for y in E] + [(x, x) for x in E]
        return _dedupe(pairs + [(rng.choice(E), rng.choice(E)) for _ in range(n_sample)])
    K = fp2_corners(G)
    els = sample_elements(G, rng, 2 * n_sample)
    return [(x, y) for x in K for y in K] + list(zip(els[::2], els[1::2]))


def operand_quads(G, rng, n_sample=1 << 16):
    """(x, y, u, v) for x*y + u*v: n_sample random choices plus the all-equal quadruples of every extreme (Fp) / every
    4-tuple of corners (Fp2) -- among them all operands q - 1, the largest frames of the fused reductions"""
    if G.K.ext == 1:
        E = field_extremes(G.K.f)
        q = G.K.q
        fixed = [(e, e, e, e) for e in E] + [(e, q - 1, e, q - 1) for e in E] + [(q - 1, e, q - 1, e) for e in E]
    else:
        K = fp2_corners(G)
        fixed = [(a, b, c, d) for a in K for b in K for c in K for d in K]
    els = sample_elements(G, rng, 4 * n_sample)
    return fixed + [tuple(els[4 * i : 4 * i + 4]) for i in range(n_sample)]


def _clip_below(v, r, bits):
    """v restricted to bits, then its highest set bits cleared until v < r (the lower windows keep their pattern)"""
    v &= (1 << bits) - 1
    while v >= r:
        v ^= 1 << (v.bit_length() - 1)
    return v


def scalar_families(fr, c):
    """plain scalars < r that drive the signed-digit recoding at width c through its edges: every c-bit window equal to
    2^(c-1)-1, 2^(c-1) (the first borrowing digit), 2^(c-1)+1 and 2^c-1 (the borrow chain runs through all windows), the
    top window at its largest value over each of those lower patterns, 2^(bits-1), r-1, r-2, 0 and 1"""
    bits, r = fr.bits, fr.q
    W = O.compute_nb_chunks(bits, c)
    out = []
    lows = []
    for w in ((1 << (c - 1)) - 1, 1 << (c - 1), (1 << (c - 1)) + 1, (1 << c) - 1):
        v = sum(w << (c * j) for j in range(W))
        out.append(_clip_below(v, r, bits))
        lows.append(v & ((1 << (c * (W - 1))) - 1))
    # alternating windows: a borrow every other window
    out.append(_clip_below(sum(((1 << (c - 1)) if j % 2 else (1 << c) - 1) << (c * j) for j in range(W)), r, bits))
    s = c * (W - 1)
    topmax = (r - 1) >> s
    for low in [0] + lows:
        v = (topmax << s) | low
        out.append(v if v < r else ((topmax - 1) << s) | low)
    out += [1 << (bits - 1), r - 1, r - 2, 0, 1]
    return _dedupe(out)


def last_window_widths(bits):
    """the widths c at which the last window holds 1 scalar bit (bits % c == 1) or all c of them, so that its digit with
    the incoming carry needs c + 1 bits (bits % c == 0)"""
    return [c for c in range(2, 25) if bits % c in (0, 1)]


def digit_scalars(G, c, n_random, seed):
    """scalar_families at width c followed by n_random random scalars, Montgomery-encoded (n x fr.limbs u64)"""
    fam = G.encode_scalars(scalar_families(G.fr, c))
    if n_random == 0:
        return fam
    return np.concatenate([fam, cref.random_scalars(G.name, n_random, seed)])


def fft_inputs(f, n):
    """stored-value inputs for the FFT butterflies: all q-1, all -1 (plain), alternating 0 / q-1, a single q-1 spike,
    all R mod q (plain 1)"""
    q = f.q
    out = {
        "all_q-1": [q - 1] * n,
        "all_minus_one": [f.to_mont(q - 1)] * n,
        "alt_0_q-1": [0 if i % 2 == 0 else q - 1 for i in range(n)],
        "spike_q-1": [q - 1 if i == n // 2 else 0 for i in range(n)],
        "all_R": [f.Rmod] * n,
    }
    return out


# ------------------------------------------------------------------------------------------
# stored values <-> u32 limbs <-> the oracle's plain values
# ------------------------------------------------------------------------------------------


class Coord:
    """stored coordinate-field elements of one group (int for Fp, (int, int) for Fp2)"""

    def __init__(self, G):
        self.f = G.K.f
        self.ext = G.K.ext
        self.w = 2 * self.f.limbs          # u32 words per base-field element
        self.words = self.ext * self.w     # per coordinate-field element

    def _comps(self, e):
        return (e,) if self.ext == 1 else e

    def pack(self, elems):
        nb = 4 * self.w
        buf = b"".join(c.to_bytes(nb, "little") for e in elems for c in self._comps(e))
        return np.frombuffer(buf, dtype="<u4").astype(np.uint32).reshape(len(elems), self.words)

    def unpack(self, arr):
        arr = np.ascontiguousarray(arr, dtype=np.uint32)
        out = []
        for row in arr:
            b = row.tobytes()
            comps = [int.from_bytes(b[4 * self.w * k : 4 * self.w * (k + 1)], "little") for k in range(self.ext)]
            out.append(comps[0] if self.ext == 1 else tuple(comps))
        return out

    def plain(self, e):
        f = self.f
        return f.from_mont(e) if self.ext == 1 else (f.from_mont(e[0]), f.from_mont(e[1]))

    def stored(self, v):
        f = self.f
        return f.to_mont(v) if self.ext == 1 else (f.to_mont(v[0]), f.to_mont(v[1]))

    def canonical(self, e):
        return all(0 <= c < self.f.q for c in self._comps(e))


def _fail(what, i, operands, got, want, kind="stored operands (decimal Montgomery limbs)"):
    ops = ", ".join(str(o) for o in operands)
    raise AssertionError("%s: first failure at #%d, %s [%s]: got %s, want %s" % (what, i, kind, ops, got, want))


def _compare(what, C, got, operands, want):
    for i, (g, w) in enumerate(zip(got, want)):
        if g != w or not C.canonical(g):
            _fail(what + ("" if C.canonical(g) else " (non-canonical output)"), i, operands[i], g, w)
    assert len(got) == len(want)


# ------------------------------------------------------------------------------------------
# checks: run(op, a_u32, b_u32 or None, out_words) -> u32 array
# ------------------------------------------------------------------------------------------


def check_field_stress(G, run, label, n_sample=1 << 16, all_pairs=True, n_inv_random=4096, seed=1):
    """FMUL, FADD, FSUB, FSQR, FNEG, FDBL, FDOT2 and FINV of one group's coordinate field on the extremes"""
    C = Coord(G)
    K = G.K
    rng = random.Random(seed)
    pairs = operand_pairs(G, rng, n_sample, all_pairs)
    xs, ys = [p[0] for p in pairs], [p[1] for p in pairs]
    A, B = C.pack(xs), C.pack(ys)
    px, py = [C.plain(x) for x in xs], [C.plain(y) for y in ys]
    for op, fn in (("FMUL", K.mul), ("FADD", K.add), ("FSUB", K.sub)):
        got = C.unpack(run(OPS[op], A, B, C.words))
        _compare("%s %s" % (label, op), C, got, pairs, [C.stored(fn(a, b)) for a, b in zip(px, py)])
    # unary ops: every extreme, and (Fp2) the sampled elements
    us = coord_extremes(G) + ([] if K.ext == 1 else xs)
    U = C.pack(us)
    pu = [C.plain(u) for u in us]
    for op, fn in (("FSQR", K.sqr), ("FNEG", K.neg), ("FDBL", K.dbl)):
        got = C.unpack(run(OPS[op], U, None, C.words))
        _compare("%s %s" % (label, op), C, got, [(u,) for u in us], [C.stored(fn(a)) for a in pu])
    # x*y + u*v through the fused reductions
    quads = operand_quads(G, rng, n_sample)
    A2 = np.hstack([C.pack([t[0] for t in quads]), C.pack([t[2] for t in quads])])
    B2 = np.hstack([C.pack([t[1] for t in quads]), C.pack([t[3] for t in quads])])
    got = C.unpack(run(OPS["FDOT2"], A2, B2, C.words))
    want = []
    for t in quads:
        x, y, u, v = (C.plain(e) for e in t)
        want.append(C.stored(K.add(K.mul(x, y), K.mul(u, v))))
    _compare("%s FDOT2" % label, C, got, quads, want)
    # inversion: every extreme (zero maps to zero) plus random elements
    f = K.f
    inv_in = coord_extremes(G) + [rng.randrange(f.q) if K.ext == 1 else (rng.randrange(f.q), rng.randrange(f.q))
                                  for _ in range(n_inv_random)]
    got = C.unpack(run(OPS["FINV"], C.pack(inv_in), None, C.words))
    _compare("%s FINV" % label, C, got, [(e,) for e in inv_in], [C.stored(K.inv(C.plain(e))) for e in inv_in])
    zero = K.zero if K.ext == 1 else (0, 0)
    assert got[inv_in.index(zero)] == zero


def check_fr_from_mont_stress(G, run, label):
    """fromMont of the scalar field's stored extremes: the canonical value, limb for limb"""
    fr = G.fr
    vals = field_extremes(fr)
    w = 2 * fr.limbs
    A = np.frombuffer(b"".join(v.to_bytes(4 * w, "little") for v in vals), dtype="<u4").astype(np.uint32).reshape(len(vals), w)
    out = run(OPS["FR_FROM_MONT"], A, None, w)
    got = [int.from_bytes(np.ascontiguousarray(r).tobytes(), "little") for r in out]
    for i, (v, g) in enumerate(zip(vals, got)):
        if g != fr.from_mont(v):
            _fail("%s FR_FROM_MONT" % label, i, (v,), g, fr.from_mont(v))


_PLAIN = "plain coordinates (xyzz point, affine point)"


def _xyzz(G, a, z):
    """extended-Jacobian representation of the affine point a with the plain z: (x z^2, y z^3, z^2, z^3)"""
    K = G.K
    if G.aff_is_inf(a):
        return G.xyzz_inf()
    zz = K.sqr(z)
    zzz = K.mul(zz, z)
    return [K.mul(a[0], zz), K.mul(a[1], zzz), zz, zzz]


def z_values(G):
    """non-zero plain z: the extremes read as plain values (1, q-1, 2^k, ...) and as stored values"""
    C = Coord(G)
    E = [e for e in coord_extremes(G) if e not in (0, (0, 0))]
    return E + [C.plain(e) for e in E]


def check_point_stress(G, run, label, n=256):
    """ADD_MIXED, SUB_MIXED, ADD, DOUBLE and TO_AFFINE on extended-Jacobian representations of consecutive multiples with z
    drawn from the extremes: generic sums, doublings (equal points, different z), cancellations, infinity on either side.
    The affine result always, the exact coordinates where the result is finite (the reference's formulas)"""
    K = G.K
    C = Coord(G)
    zs = z_values(G)
    pts = O.consecutive_multiples(G, n + 1, start_k=2)
    ps, as_, qs = [], [], []
    for i in range(n):
        p = pts[i]
        ps.append(_xyzz(G, p, zs[i % len(zs)]))
        k = i % 8
        a = {0: p, 1: G.aff_neg(p), 2: G.aff_inf()}.get(k, pts[i + 1])
        as_.append(a)
        q = {0: _xyzz(G, p, zs[(i + 7) % len(zs)]), 1: _xyzz(G, G.aff_neg(p), zs[(i + 3) % len(zs)]), 2: G.xyzz_inf()}.get(
            k, _xyzz(G, pts[i + 1], zs[(i * 5 + 1) % len(zs)]))
        qs.append(q)
    ps[3] = G.xyzz_inf()
    ps[11] = [K.zero] * 4                        # all-zero infinity (memset buckets)
    w = C.words

    def enc_xyzz(lst):
        return np.hstack([C.pack([C.stored(p[k]) for p in lst]) for k in range(4)])

    def dec_xyzz(arr):
        return [[C.plain(c) for c in row] for row in zip(*(C.unpack(arr[:, k * w : (k + 1) * w]) for k in range(4)))]

    P = enc_xyzz(ps)
    Aff = np.hstack([C.pack([C.stored(a[0]) for a in as_]), C.pack([C.stored(a[1]) for a in as_])])
    for op, neg in (("ADD_MIXED", False), ("SUB_MIXED", True)):
        got = dec_xyzz(run(OPS[op], P, Aff, 4 * w))
        for i, (p, a, g) in enumerate(zip(ps, as_, got)):
            want = G.add_mixed(list(p), a, negate=neg)
            if G.xyzz_to_affine(g) != G.xyzz_to_affine(want) or (not K.is_zero(want[2]) and g != want):
                _fail("%s %s" % (label, op), i, (p, a), g, want, _PLAIN)
    got = dec_xyzz(run(OPS["ADD"], P, enc_xyzz(qs), 4 * w))
    for i, (p, q, g) in enumerate(zip(ps, qs, got)):
        want = G.xyzz_add(list(p), list(q))
        if G.xyzz_to_affine(g) != G.xyzz_to_affine(want) or (not K.is_zero(want[2]) and not K.is_zero(p[2]) and g != want):
            _fail("%s ADD" % label, i, (p, q), g, want, _PLAIN)
    got = dec_xyzz(run(OPS["DOUBLE"], P, None, 4 * w))
    for i, (p, g) in enumerate(zip(ps, got)):
        want = G.xyzz_double(p)
        if G.xyzz_to_affine(g) != G.xyzz_to_affine(want):
            _fail("%s DOUBLE" % label, i, (p,), g, want, _PLAIN)
    got = run(OPS["TO_AFFINE"], P, None, 2 * w)
    want = np.ascontiguousarray(G.encode_affine([G.xyzz_to_affine(p) for p in ps])).view(np.uint32).reshape(n, 2 * w)
    bad = np.nonzero((got != want).any(axis=1))[0]
    if len(bad):
        i = int(bad[0])
        _fail("%s TO_AFFINE" % label, i, (ps[i],), got[i].tolist(), want[i].tolist(), _PLAIN)
