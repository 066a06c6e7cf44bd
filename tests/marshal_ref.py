"""A plain big-int restatement of point (de)serialisation for the G2 groups of the pairing curves, and the generators of the
marshalling tests (tests/test_marshal_cpu.py on the kernel emulation, tests/test_gpu_marshal.py on the device).

  * G2Affine.setBytes without the subgroup check (ecc/bn254/marshal.go:1116-1216, ecc/bls12-381/marshal.go:1160+) over a
    homogeneous stream, with the homogeneous-stream rule of the device decoder (a point is infinity only under its own kind's
    flag), and G2Affine.Bytes / RawBytes (:1051-1100).  Square roots and cube roots are generic Tonelli-Shanks / Pohlig-Hellman
    over the field of q^D elements (D = 2 for bn254, bls12-381, bls12-377; D = 1 for the bw6 G2 curves over Fp), so nothing here
    shares a line with the complex-method square root of the device.
  * G1 encoding is kzg.g1_bytes / kzg.g1_raw_bytes.
Elements are tuples of D canonical integers (A0, A1); a point is (X, Y) or None for infinity."""
from __future__ import annotations

import importlib
import random
from dataclasses import dataclass

import numpy as np

OK, BAD_INFINITY, BAD_ELEMENT, NO_SQRT, NOT_ON_CURVE, BAD_FLAGS = 0, 1, 2, 3, 4, 5
MESSAGES = {BAD_INFINITY: "invalid infinity point encoding", BAD_ELEMENT: "invalid fp.Element encoding",
            NO_SQRT: "invalid compressed coordinate: square root doesn't exist", NOT_ON_CURVE: "invalid point: subgroup check failed",
            BAD_FLAGS: "invalid point encoding"}
PAIRING = ["bn254", "bls12381", "bls12377", "bls24315", "bls24317", "bw6633", "bw6761"]
G2_GROUPS = ["bn254_g2", "bls12381_g2", "bls12377_g2", "bw6761_g2", "bw6633_g2"]
G1_GROUPS = [c + "_g1" for c in PAIRING]
ALL_GROUPS = G1_GROUPS + G2_GROUPS


def kzg():
    return importlib.import_module("gnark-crypto_b200.kzg")


def curves():
    return importlib.import_module("gnark-crypto_b200.curves")


@dataclass
class Group:
    name: str
    id: int
    q: int
    D: int                  # base-field elements per coordinate
    beta: int               # u^2 (D = 2)
    b: tuple                # the curve's (twist's) b as a D-tuple
    fp_words: int
    flags: dict

    @property
    def nb(self) -> int:    # fp.Bytes
        return 8 * self.fp_words

    @property
    def words(self) -> int:  # uint64 words of one in-memory affine point
        return 2 * self.D * self.fp_words

    def comp_bytes(self) -> int:
        return self.D * self.nb

    # ---- field of q^D elements ----
    def add(self, a, b):
        return tuple((x + y) % self.q for x, y in zip(a, b))

    def sub(self, a, b):
        return tuple((x - y) % self.q for x, y in zip(a, b))

    def neg(self, a):
        return tuple((-x) % self.q for x in a)

    def mul(self, a, b):
        q = self.q
        if self.D == 1:
            return (a[0] * b[0] % q,)
        return ((a[0] * b[0] + self.beta * a[1] * b[1]) % q, (a[0] * b[1] + a[1] * b[0]) % q)

    def pow(self, a, e: int):
        r = self.one()
        for bit in bin(e)[2:]:
            r = self.mul(r, r)
            if bit == "1":
                r = self.mul(r, a)
        return r

    def one(self):
        return (1,) + (0,) * (self.D - 1)

    def zero(self):
        return (0,) * self.D

    def is_zero(self, a) -> bool:
        return not any(a)

    @property
    def order(self) -> int:      # of the multiplicative group
        return self.q ** self.D - 1

    def norm(self, a) -> int:
        return a[0] % self.q if self.D == 1 else (a[0] * a[0] - self.beta * a[1] * a[1]) % self.q

    def is_square(self, a) -> bool:
        """E2.Legendre (the norm's Legendre symbol) != -1"""
        return self.is_zero(a) or pow(self.norm(a), (self.q - 1) // 2, self.q) == 1

    def _non_residue(self, k: int):
        for c in range(2, 1000):
            for z in ([(c,)] if self.D == 1 else [(c, 0), (c, 1), (0, c), (1, c)]):
                if self.pow(z, self.order // k) != self.one():
                    return z
        raise AssertionError("no non-residue")

    def sqrt(self, a):
        """any root of a (Tonelli-Shanks over the group of order q^D - 1), None when there is none"""
        if self.is_zero(a):
            return self.zero()
        if not self.is_square(a):
            return None
        t, s = self.order, 0
        while t % 2 == 0:
            t //= 2
            s += 1
        c = self.pow(self._non_residue(2), t)
        x, tt, m = self.pow(a, (t + 1) // 2), self.pow(a, t), s
        while tt != self.one():
            i, t2 = 0, tt
            while t2 != self.one():
                t2 = self.mul(t2, t2)
                i += 1
            b = self.pow(c, 1 << (m - i - 1))
            x, c = self.mul(x, b), self.mul(b, b)
            tt, m = self.mul(tt, c), i
        assert self.mul(x, x) == a
        return x

    def cbrt(self, a):
        """a cube root of a (Pohlig-Hellman on the 3-Sylow part), None when there is none"""
        if self.is_zero(a):
            return self.zero()
        if self.pow(a, self.order // 3) != self.one():
            return None
        t, e = self.order, 0
        while t % 3 == 0:
            t //= 3
            e += 1
        g = self.pow(self._non_residue(3), t)            # order 3^e
        A = self.pow(a, t)
        gamma = self.pow(g, 3 ** (e - 1))
        ginv = self.pow(g, 3 ** e - 1)
        k = 0
        for i in range(e):
            h = self.pow(self.mul(A, self.pow(ginv, k)), 3 ** (e - 1 - i))
            d = [self.one(), gamma, self.mul(gamma, gamma)].index(h)
            k += d * 3 ** i
        assert k % 3 == 0
        x1 = self.pow(g, k // 3)
        alpha = pow(t, -1, 3 ** e)
        beta_ = (1 - alpha * t) // 3 ** e
        B = self.pow(a, (beta_ * 3 ** e) % self.order)
        x = self.mul(self.pow(x1, alpha), self.pow(B, pow(3, -1, t)))
        assert self.mul(self.mul(x, x), x) == a
        return x

    def rhs(self, x):
        return self.add(self.mul(self.mul(x, x), x), self.b)

    def on_curve(self, x, y) -> bool:
        return self.mul(y, y) == self.rhs(x)

    def largest(self, y) -> bool:
        """LexicographicallyLargest (E2: A1, or A0 when A1 = 0)"""
        v = y[-1] if self.D == 2 and y[1] else y[0]
        return v > (self.q - 1) // 2

    # ---- memory layout: Montgomery uint64 limbs, {A0, A1} per coordinate, infinity = zeroes ----
    def elem_limbs(self, v: int) -> list:
        L = self.fp_words
        m = (v << (64 * L)) % self.q
        return [(m >> (64 * i)) & (2 ** 64 - 1) for i in range(L)]

    def row(self, pt) -> np.ndarray:
        if pt is None:
            return np.zeros(self.words, dtype=np.uint64)
        x, y = pt
        return np.array(sum((self.elem_limbs(v) for v in (*x, *y)), []), dtype=np.uint64)

    def unrow(self, r):
        """a memory row -> (X, Y) of canonical tuples, or None for the all-zero row; limbs are taken as given (not reduced)"""
        r = [int(v) for v in np.asarray(r, dtype=np.uint64).reshape(-1)]
        if not any(r):
            return None
        L, q = self.fp_words, self.q
        rinv = pow(1 << (64 * L), -1, q)
        el = [sum(r[k * L + i] << (64 * i) for i in range(L)) * rinv % q for k in range(2 * self.D)]
        return tuple(el[:self.D]), tuple(el[self.D:])

    # ---- wire format ----
    def _wire(self, e) -> bytes:
        return b"".join(v.to_bytes(self.nb, "big") for v in reversed(e))      # A1 || A0

    def bytes_(self, pt) -> bytes:
        """G2Affine.Bytes"""
        f = self.flags
        if pt is None:
            return bytes([f["inf"]]) + bytes(self.comp_bytes() - 1)
        x, y = pt
        out = bytearray(self._wire(x))
        out[0] |= f["large"] if self.largest(y) else f["small"]
        return bytes(out)

    def raw_bytes(self, pt) -> bytes:
        """G2Affine.RawBytes"""
        f = self.flags
        if pt is None:
            return bytes([f["unc"] if f["unc_inf"] is None else f["unc_inf"]]) + bytes(2 * self.comp_bytes() - 1)
        x, y = pt
        return self._wire(x) + self._wire(y)

    def set_bytes(self, enc: bytes, raw: bool, check: bool = True):
        """one point of a homogeneous stream -> (point or None, code)"""
        f, q, nb, D = self.flags, self.q, self.nb, self.D
        m = enc[0] & f["mask"]
        size = (2 if raw else 1) * D * nb
        inf_flag = (f["unc_inf"] if raw else f["inf"])
        if inf_flag is not None and m == inf_flag:
            if (enc[0] & ~f["mask"] & 0xFF) or any(enc[1:size]):
                return None, BAD_INFINITY
            return None, OK
        if (raw and m != f["unc"]) or (not raw and m not in (f["small"], f["large"])):
            return None, BAD_FLAGS
        b = bytearray(enc[:size])
        b[0] &= ~f["mask"] & 0xFF
        vals = [int.from_bytes(b[i * nb:(i + 1) * nb], "big") for i in range(size // nb)]
        if any(v >= q for v in vals):
            return None, BAD_ELEMENT
        x = tuple(reversed(vals[:D]))
        if raw:
            y = tuple(reversed(vals[D:]))
            if check and not self.on_curve(x, y) and not (self.is_zero(x) and self.is_zero(y)):
                return None, NOT_ON_CURVE
            return (x, y), OK
        y = self.sqrt(self.rhs(x))
        if y is None:
            return None, NO_SQRT
        if self.largest(y) != (m == f["large"]):
            y = self.neg(y)
        return (x, y), OK

    def decode_stream(self, data: bytes, n: int, raw: bool, check: bool = True):
        """-> (rows (n, words), first error (index, code) or None); a bad point's row is zeroes"""
        size = (2 if raw else 1) * self.comp_bytes()
        rows = np.zeros((n, self.words), dtype=np.uint64)
        first = None
        for i in range(n):
            pt, code = self.set_bytes(data[i * size:(i + 1) * size], raw, check)
            if code:
                first = first or (i, code)
            else:
                rows[i] = self.row(pt)
        return rows, first

    def encode(self, pts, raw: bool) -> bytes:
        return b"".join(self.raw_bytes(p) if raw else self.bytes_(p) for p in pts)

    # ---- points ----
    def rand_elem(self, rng):
        return tuple(rng.randrange(self.q) for _ in range(self.D))

    def point_at(self, x, rng):
        y = self.sqrt(self.rhs(x))
        if y is None:
            return None
        return (x, y if rng.random() < 0.5 else self.neg(y))

    def random_points(self, m: int, rng) -> list:
        out = []
        while len(out) < m:
            p = self.point_at(self.rand_elem(rng), rng)
            if p is not None:
                out.append(p)
        return out

    def point_with_y(self, y):
        """a point (X, y), X a cube root of y^2 - b, or None"""
        x = self.cbrt(self.sub(self.mul(y, y), self.b))
        return None if x is None else (x, y)

    def sqrt_depth(self, a: int) -> int:
        """the number of Tonelli-Shanks rounds of Fp on a square a: log2 of the order of a^t, q - 1 = 2^s t"""
        t = self.q - 1
        while t % 2 == 0:
            t //= 2
        v, k = pow(a, t, self.q), 0
        while v != 1:
            v = v * v % self.q
            k += 1
        return k

    @property
    def two_adicity(self) -> int:
        t, s = self.q - 1, 0
        while t % 2 == 0:
            t //= 2
            s += 1
        return s


def group(name: str) -> Group:
    C = curves()
    g = C.GROUPS[name]
    cp = C.CURVE_PARAMS[g.curve]
    q = cp.q
    if name.endswith("_g1"):
        return Group(name, g.id, q, 1, 0, (cp.b,), cp.fp_words, cp.flags)
    if g.degree == 1:                                      # bw6 G2 over Fp: bTwistCurveCoeff = 4 (bw6-761), 8 (bw6-633)
        return Group(name, g.id, q, 1, 0, ({"bw6761": 4, "bw6633": 8}[g.curve],), cp.fp_words, cp.flags)
    beta = {"bn254": -1, "bls12381": -1, "bls12377": -5}[g.curve] % q
    G = Group(name, g.id, q, 2, beta, (0, 0), cp.fp_words, cp.flags)
    if g.curve == "bn254":                                 # 3 / (9 + u)
        d = (9, 1)
        inv_n = pow(G.norm(d), -1, q)
        G.b = (3 * 9 * inv_n % q, -3 * inv_n % q)
    elif g.curve == "bls12381":                            # 4 (1 + u)
        G.b = (4, 4)
    else:                                                  # 1 / u = u / beta
        G.b = (0, pow(beta, -1, q))
    return G


def encode_ref(G: Group, pts, raw: bool) -> bytes:
    """the reference's encoding of a list of points (None = infinity): G1 through kzg.g1_bytes / g1_raw_bytes"""
    if G.name.endswith("_g1"):
        K = kzg()
        c = G.name[:-3]
        return b"".join((K.g1_raw_bytes if raw else K.g1_bytes)(G.row(p), c) for p in pts)
    return G.encode(pts, raw)


# ---------------------------------------------------------------------------------------------------------------- cases
@dataclass
class Case:
    title: str
    data: bytes
    n: int
    raw: bool
    check: bool = True


def _q_values(G: Group) -> list:
    q = G.q
    top = (1 << (8 * G.nb - (3 if G.flags["unc_inf"] is not None else 2))) - 1       # every value bit below the flags
    return [q, q + 1, q + (1 << 64), top]


def decode_cases(G: Group, seed: int = 1) -> list:
    """the decoder's families for one group; every case's expectation is G.decode_stream"""
    rng = random.Random(seed)
    f, D, nb = G.flags, G.D, G.nb
    pts = G.random_points(12, rng)
    cases = []
    # random on-curve points with infinity, both kinds, with and without the on-curve check
    mix = pts[:5] + [None] + pts[5:9] + [None]
    for raw in (False, True):
        cases.append(Case("random+inf raw=%d" % raw, G.encode(mix, raw), len(mix), raw))
    cases.append(Case("random unchecked raw", G.encode(mix, True), len(mix), True, False))
    # X.A1 = 0 (D = 2), and x = 0
    xs = []
    while len(xs) < 3:
        p = G.point_at((rng.randrange(G.q),) + (0,) * (D - 1), rng)
        if p:
            xs.append(p)
    p0 = G.point_at(G.zero(), rng)
    xs += [p0] if p0 else []
    for raw in (False, True):
        cases.append(Case("x.A1 = 0 raw=%d" % raw, G.encode(xs, raw), len(xs), raw))
    # Y with A1 = 0 (the A0 sign branch: a1 = 0, a0 a square) and Y with A0 = 0 (a1 = 0, a0 a non-residue: the root c u)
    if D == 2:
        ys = []
        for form in (lambda v: (v, 0), lambda v: (0, v)):
            k = 0
            while k < 3:
                p = G.point_with_y(form(rng.randrange(1, G.q)))
                if p:
                    ys += [p, (p[0], G.neg(p[1]))]
                    k += 1
        for raw in (False, True):
            cases.append(Case("y.A1 = 0 / y.A0 = 0 raw=%d" % raw, G.encode(ys, raw), len(ys), raw))
    # x with no root
    bad = []
    while len(bad) < 3:
        x = G.rand_elem(rng)
        if not G.is_square(G.rhs(x)):
            for flag in ("small", "large"):
                e = bytearray(G._wire(x))
                e[0] |= f[flag]
                bad.append(bytes(e))
    cases.append(Case("no root", b"".join(bad), len(bad), False))
    # an element equal to q or above it, in each position of both kinds
    p = pts[0]
    for raw in (False, True):
        base = G.encode([p], raw)
        for pos in range(len(base) // nb):
            for v in _q_values(G):
                e = bytearray(base)
                keep = e[0] & f["mask"] if pos == 0 else 0
                e[pos * nb:(pos + 1) * nb] = (v % (1 << (8 * nb))).to_bytes(nb, "big")
                if pos == 0:
                    e[0] = (e[0] & ~f["mask"] & 0xFF) | keep
                cases.append(Case("element %d = %#x raw=%d" % (pos, v - G.q, raw), bytes(e) + base, 2, raw))
    # every top-bit pattern of both kinds, over a valid point's payload and over zeroes
    nflag = 3 if f["unc_inf"] is not None else 2
    shift = 8 - nflag
    for raw in (False, True):
        for payload in (G.encode([p], raw), bytes(len(G.encode([p], raw)))):
            for pat in range(1 << nflag):
                e = bytearray(payload)
                e[0] = (e[0] & ~f["mask"] & 0xFF) | (pat << shift)
                cases.append(Case("flags %s raw=%d" % (bin(pat), raw), G.encode([pts[1]], raw) + bytes(e) + G.encode([pts[2]], raw),
                                  3, raw))
    # a non-zero byte anywhere in an infinity encoding (and a non-zero bit below the flags)
    for raw in (False, True):
        inf = G.encode([None], raw)
        if raw and f["unc_inf"] is None:
            continue                               # bn254: the raw infinity is the all-zero point, a valid (0, 0)
        for pos in range(len(inf)):
            e = bytearray(inf)
            e[pos] |= 1
            cases.append(Case("inf byte %d raw=%d" % (pos, raw), G.encode([pts[3]], raw) + bytes(e), 2, raw))
    # two bad points: the lower index carries the higher code
    for raw in (False, True):
        good = G.encode(pts[:6], raw)
        size = len(good) // 6
        e = bytearray(good)
        e[1 * size] = (e[1 * size] & ~f["mask"] & 0xFF) | (0b011 << 5 if nflag == 3 else (f["small"] if raw else f["unc"]))   # BAD_FLAGS
        e[4 * size + 1:4 * size + nb] = b"\xff" * (nb - 1)                  # BAD_ELEMENT (first element all ones below the flags)
        e[4 * size] |= ~f["mask"] & 0xFF
        cases.append(Case("two errors raw=%d" % raw, bytes(e), 6, raw))
    return cases


def depth_points(G: Group, rng, per: int = 2) -> dict:
    """Fp2 groups: compressed points whose rhs has a norm at Tonelli-Shanks depth 0 and s - 1 (the shallowest and deepest rounds
    of the square root of the norm).  rhs = Y^2 with norm(Y) = v, v = w^(2^s) (depth 0) or z w^(2^s), z a non-residue (the
    norm v^2 then has depth s - 1)."""
    q, s = G.q, G.two_adicity
    z = next(c for c in range(2, 100) if pow(c, (q - 1) // 2, q) == q - 1)
    out = {0: [], s - 1: []}
    for depth, zz in ((0, 1), (s - 1, z)):
        while len(out[depth]) < per:
            v = zz * pow(rng.randrange(2, q), 1 << s, q) % q
            y1 = rng.randrange(1, q)
            r = (v + G.beta * y1 * y1) % q                    # y0^2 = v + beta y1^2  (norm = y0^2 - beta y1^2)
            if pow(r, (q - 1) // 2, q) != 1:
                continue
            y0 = _fp_sqrt(r, q)
            p = G.point_with_y((y0, y1))
            if p is None:
                continue
            assert G.sqrt_depth(G.norm(G.rhs(p[0]))) == depth
            out[depth].append(p)
    return out


def encode_points(G: Group, rng) -> list:
    """random points, infinity, X.A1 = 0, Y.A1 = 0 and Y.A0 = 0 (the encoder needs no curve), and y at the sign boundary
    (q - 1) / 2, (q + 1) / 2 in the coordinate that decides"""
    q, D = G.q, G.D
    h = (q - 1) // 2
    pts = G.random_points(4, rng) + [None]
    el = lambda: G.rand_elem(rng)
    pts += [((rng.randrange(q),) + (0,) * (D - 1), el()), (el(), (rng.randrange(1, q),) + (0,) * (D - 1))]
    if D == 2:
        pts += [(el(), (0, rng.randrange(1, q))), (el(), (h, 0)), (el(), (h + 1, 0)), (el(), (rng.randrange(q), h)),
                (el(), (rng.randrange(q), h + 1)), (el(), (q - 1, 1))]
    else:
        pts += [(el(), (h,)), (el(), (h + 1,)), (el(), (q - 1,)), (el(), (1,))]
    pts += [(G.zero(), el()), (el(), G.zero())]       # one zero coordinate is no infinity
    return pts


def _fp_sqrt(a: int, q: int) -> int:
    r = kzg()._tonelli(a, q)
    assert r is not None and r * r % q == a
    return r
