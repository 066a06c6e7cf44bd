"""Generators and the reference of the G1 point decoder stress tests (k_g1_decode, decode_kernels.cuh; run on the device by
tests/test_gpu_decode_stress.py and through the CPU kernel emulation by tests/test_decode_stress_cpu.py).

The reference is a plain big-int restatement of G1Affine.setBytes without the subgroup check (marshal.go:862-950 of bn254,
:895-990 of the three-bit curves) applied to a homogeneous stream: every point of a compressed stream is fp.Bytes long and every
point of a raw one 2 * fp.Bytes, so a point is infinity only under its own kind's flag (FLAGS below).  It returns the expected
points as Montgomery limbs (oracle.py's field encoders; infinity and rejected points are zeroes) and the expected first error
(index, code).

Families (each a list of Stream):
  A. square-root depth: y = zeta * w^(2^s) with zeta a primitive 2^(k+1)-th root of unity, x = cbrt(y^2 - b), so that a = x^3 + b
     has a^t of order exactly 2^k: Tonelli-Shanks runs k rounds; every k in [0, s), plus non-residues (order 2^s);
  B. sign boundary: y = (q - 1)/2 - k and (q + 1)/2 + k, and y = h +- u 2^(32 j) (h = (q + 1)/2) so that
     lexicographically_largest is decided at 32-bit limb j;
  C. element boundary: x and raw y at and above q (q, q + 1, q + 2^(32 j), q with one limb raised), below q with one limb lowered,
     value bits above the flags, a flag-looking top byte in raw y; x = 0 and the points with y = 0;
  D. every top-bit pattern in both stream kinds with zero and non-zero payloads, every single non-zero byte of an infinity
     encoding, and the other kind's infinity flag beside a valid point, beside zeroes and at the last index;
  E. two to four errors in different blocks where the lower index carries the higher code.
"""
from __future__ import annotations

import functools
import random
from dataclasses import dataclass, field
from importlib import import_module

import numpy as np

from oracle import cref
from oracle import oracle as O

CURVES = ["bn254", "bls12381", "bls12377", "bls24315", "bls24317", "bw6633", "bw6761"]
GID = {"bn254": 0, "bls12381": 2, "bls12377": 4, "bls24315": 9, "bls24317": 10, "bw6633": 11, "bw6761": 7}
OK, BAD_INFINITY, BAD_ELEMENT, NO_SQRT, NOT_ON_CURVE, BAD_FLAGS = 0, 1, 2, 3, 4, 5
CODE_NAMES = {OK: "ok", BAD_INFINITY: "DEC_BAD_INFINITY", BAD_ELEMENT: "DEC_BAD_ELEMENT", NO_SQRT: "DEC_NO_SQRT",
              NOT_ON_CURVE: "DEC_NOT_ON_CURVE", BAD_FLAGS: "DEC_BAD_FLAGS"}
BLOCK = 128                  # threads per block of k_g1_decode

# What setBytes does with each top-bit pattern (unshifted) of a point in a homogeneous stream of either kind (marshal.go:25-34;
# isMaskInvalid rejects 001, 011 and 111 on the three-bit curves): "inf" demands a zero payload, "x" solves for y, "xy" reads
# both coordinates.  A pattern missing from its row is "invalid point encoding" -- the other kind's infinity flag included, whose
# point would have the other kind's length.
FLAGS = {
    2: {False: {0b01: "inf", 0b10: "x", 0b11: "x"}, True: {0b00: "xy"}},
    3: {False: {0b110: "inf", 0b100: "x", 0b101: "x"}, True: {0b010: "inf", 0b000: "xy"}},
}
# B's smallest k with ((q - 1)/2 - k)^2 - b a cube
SIGN_K = {"bn254": 2, "bls12381": 4, "bls12377": 1, "bls24315": 4, "bls24317": 1, "bw6633": 1, "bw6761": 3}


@dataclass(frozen=True)
class Curve:
    name: str
    q: int
    b: int
    nb: int                  # fp.Bytes
    words: int               # u64 words of one affine point
    nflag: int               # flag bits of the top byte (2 or 3)
    s: int                   # q - 1 = 2^s t, t odd
    t: int
    z_t: int                 # z^t for a quadratic non-residue z: order 2^s

    @property
    def shift(self) -> int:
        return 8 - self.nflag

    @property
    def mask(self) -> int:
        return ((1 << self.nflag) - 1) << self.shift

    @property
    def limbs32(self) -> int:
        return self.nb // 4

    def flag(self, pattern: int) -> int:
        return pattern << self.shift

    @property
    def small(self) -> int:
        return self.flag(0b10 if self.nflag == 2 else 0b100)

    @property
    def large(self) -> int:
        return self.flag(0b11 if self.nflag == 2 else 0b101)

    @property
    def inf(self) -> int:
        return self.flag(0b01 if self.nflag == 2 else 0b110)

    @property
    def unc_inf(self):
        return None if self.nflag == 2 else self.flag(0b010)


@functools.lru_cache(maxsize=None)
def curve(name: str) -> Curve:
    cp = import_module("gnark-crypto_b200.curves").CURVE_PARAMS[name]
    q = cp.q
    s, t = 0, q - 1
    while t % 2 == 0:
        t, s = t // 2, s + 1
    z = 2
    while pow(z, (q - 1) // 2, q) != q - 1:
        z += 1
    return Curve(name, q, cp.b, cp.fp_bytes, 2 * cp.fp_words, 3 if cp.flags["unc_inf"] is not None else 2, s, t, pow(z, t, q))


# ---- field helpers ----
def sqrt_mod(a: int, c: Curve):
    """a square root of a mod q (Tonelli-Shanks), None for a non-residue"""
    q = c.q
    a %= q
    if a == 0:
        return 0
    if pow(a, (q - 1) // 2, q) != 1:
        return None
    m, cc, tt, r = c.s, c.z_t, pow(a, c.t, q), pow(a, (c.t + 1) // 2, q)
    while tt != 1:
        i, t2 = 0, tt
        while t2 != 1:
            t2, i = t2 * t2 % q, i + 1
        g = pow(cc, 1 << (m - i - 1), q)
        m, cc, tt, r = i, g * g % q, tt * g * g % q, r * g % q
    assert r * r % q == a
    return r


@functools.lru_cache(maxsize=None)
def _cube_consts(q: int):
    m, e = q - 1, 0
    while m % 3 == 0:
        m, e = m // 3, e + 1
    g = 2
    while pow(g, (q - 1) // 3, q) == 1:
        g += 1
    return m, e, pow(g, m, q)


def cube_roots(a: int, q: int) -> list:
    """all x with x^3 = a mod q (q = 1 mod 3): three or none (a != 0).  x0 = a^(1/3 mod m) is off by an element of the 3-Sylow
    subgroup (order 3^e, here e <= 2), whose discrete logarithm is found by trying every exponent."""
    a %= q
    if a == 0:
        return [0]
    if pow(a, (q - 1) // 3, q) != 1:
        return []
    m, e, G = _cube_consts(q)
    x0 = pow(a, pow(3, -1, m), q)
    d = pow(x0, 3, q) * pow(a, -1, q) % q
    j = next(j for j in range(3 ** e) if pow(G, j, q) == d)
    assert j % 3 == 0
    x = x0 * pow(G, -(j // 3), q) % q
    w = pow(G, 3 ** (e - 1), q)           # a primitive cube root of unity
    roots = sorted({x, x * w % q, x * w * w % q})
    assert len(roots) == 3 and all(pow(r, 3, q) == a for r in roots)
    return roots


def sqrt_depth(a: int, c: Curve) -> int:
    """k with a^t of order 2^k: the rounds Tonelli-Shanks runs (k = s for a non-residue)"""
    v, k = pow(a, c.t, c.q), 0
    while v != 1:
        v, k = v * v % c.q, k + 1
    return k


def limbs32(v: int, c: Curve) -> list:
    return [(v >> (32 * j)) & 0xFFFFFFFF for j in range(c.limbs32)]


# ---- encodings ----
def comp(c: Curve, x: int, flag: int) -> bytes:
    """fp.Bytes big-endian x with `flag` or-ed into the top byte (x may exceed q)"""
    out = bytearray(x.to_bytes(c.nb, "big"))
    out[0] |= flag
    return bytes(out)


def raw(c: Curve, x: int, y: int, flag: int = 0) -> bytes:
    return comp(c, x, flag) + y.to_bytes(c.nb, "big")


def compress(c: Curve, x: int, y: int) -> bytes:
    return comp(c, x, c.large if y > (c.q - 1) // 2 else c.small)


# ---- the reference ----
def decode_point(c: Curve, enc: bytes, is_raw: bool, check: bool = True):
    """setBytes on one point of a homogeneous stream -> (code, (x, y) or None for infinity and errors)"""
    q = c.q
    assert len(enc) == (2 if is_raw else 1) * c.nb
    action = FLAGS[c.nflag][is_raw].get((enc[0] & c.mask) >> c.shift)
    if action is None:
        return BAD_FLAGS, None                                   # ErrInvalidEncoding
    if action == "inf":
        if (enc[0] & ~c.mask & 0xFF) or any(enc[1:]):           # isZeroed(buf[0] & ^mMask, buf[1:size])
            return BAD_INFINITY, None
        return OK, None
    x = int.from_bytes(bytes([enc[0] & ~c.mask & 0xFF]) + enc[1:c.nb], "big")
    if x >= q:                                                   # SetBytesCanonical
        return BAD_ELEMENT, None
    rhs = (x * x * x + c.b) % q
    if is_raw:
        y = int.from_bytes(enc[c.nb:], "big")
        if y >= q:
            return BAD_ELEMENT, None
        if check and (x or y) and y * y % q != rhs:              # on-curve part of the check; (0, 0) is infinity
            return NOT_ON_CURVE, None
        return OK, (x, y)
    y = sqrt_mod(rhs, c)
    if y is None:
        return NO_SQRT, None
    if (y > (q - 1) // 2) != ((enc[0] & c.mask) == c.large):    # LexicographicallyLargest, then Neg
        y = (q - y) % q
    return OK, (x, y)


def encode_point(c: Curve, xy) -> np.ndarray:
    """the in-memory G1Affine: Montgomery limbs of x then y; zeroes for infinity"""
    if xy is None:
        return np.zeros(c.words, dtype=np.uint64)
    f = O.FIELDS[c.name + "_fp"]
    return np.array(f.to_limbs(f.to_mont(xy[0])) + f.to_limbs(f.to_mont(xy[1])), dtype=np.uint64)


@dataclass
class Stream:
    """one call of the decoder: n points of one kind, each with a label, then `tail` (bytes past the stream's end)"""
    curve: str
    family: str
    case: str
    raw: bool
    points: list
    labels: list
    check: bool = True
    tail: bytes = b""
    _want: tuple = field(default=None, repr=False)

    @property
    def n(self) -> int:
        return len(self.points)

    def data(self) -> bytes:
        return b"".join(self.points) + self.tail

    def expected(self):
        """(rows (n, words) uint64, first error (index, code) or None, per-point codes)"""
        if self._want is None:
            c = curve(self.curve)
            res = [decode_point(c, p, self.raw, self.check) for p in self.points]
            rows = np.stack([encode_point(c, xy) for _, xy in res]) if res else np.zeros((0, c.words), dtype=np.uint64)
            codes = [code for code, _ in res]
            first = next(((i, k) for i, k in enumerate(codes) if k), None)
            self._want = (rows, first, codes)
        return self._want

    def title(self) -> str:
        return "%s %s %s (%s stream of %d%s)" % (self.curve, self.family, self.case, "raw" if self.raw else "compressed", self.n,
                                                "" if self.check else ", no on-curve check")


def compare(s: Stream, got_rows: np.ndarray, got_first):
    """limb-exact rows and the first error; the message names the curve, family, case and index"""
    rows, first, codes = s.expected()
    got_rows = np.asarray(got_rows, dtype=np.uint64).reshape(s.n, -1)
    bad = np.nonzero((got_rows != rows).any(axis=1))[0]
    if len(bad):
        i = int(bad[0])
        raise AssertionError("%s: index %d (%s, expected %s): %d rows differ\n got  %s\n want %s" % (
            s.title(), i, s.labels[i], CODE_NAMES[codes[i]], len(bad), got_rows[i].tolist(), rows[i].tolist()))
    fmt = lambda e: "none" if e is None else "(%d, %s)" % (e[0], CODE_NAMES.get(e[1], e[1]))
    assert got_first == first, "%s: first error %s, expected %s at %s" % (
        s.title(), fmt(got_first), fmt(first), "-" if first is None else s.labels[first[0]])


# ---- valid points ----
def subgroup_rows(name: str, m: int, seed: int):
    """m distinct subgroup points P, [2]P, ... (P = [seed-derived]G, C port): ((m, words) Montgomery rows, integer pairs)"""
    G = O.GROUPS[name + "_g1"]
    base = cref.scalar_mul(name + "_g1", G.encode_affine([G.gen])[0], random.Random(seed).randrange(2, G.fr.q))
    rows = cref.generate_multiples(name + "_g1", base, 1, m, nthreads=4)
    f = O.FIELDS[name + "_fp"]
    L = G.aff_words // 2
    rinv = f.Rinv
    return rows, [(O.Field.from_limbs(r[:L]) * rinv % f.q, O.Field.from_limbs(r[L:]) * rinv % f.q) for r in rows]


def subgroup_points(name: str, m: int, seed: int) -> list:
    return subgroup_rows(name, m, seed)[1]


def _pad(c: Curve, is_raw: bool, xy) -> bytes:
    return raw(c, *xy) if is_raw else compress(c, *xy)


def _streams(c: Curve, family: str, is_raw: bool, items, pads, check=True) -> list:
    """the accepted items of a family in one stream; every rejected item alone between two valid points, so that its code is the
    stream's first error"""
    good = [(lab, e) for lab, e in items if decode_point(c, e, is_raw, check)[0] == OK]
    out = []
    if good:
        out.append(Stream(c.name, family, "accepted points", is_raw, [e for _, e in good], [lab for lab, _ in good], check))
    for lab, e in items:
        if decode_point(c, e, is_raw, check)[0] != OK:
            out.append(Stream(c.name, family, lab, is_raw, [_pad(c, is_raw, pads[0]), e, _pad(c, is_raw, pads[1])],
                              ["valid neighbour", lab, "valid neighbour"], check))
    return out


def _both(c: Curve, lab: str, x: int, y: int) -> list:
    """(label, encoding) of (x, y) and (x, -y), each compressed and raw: -> ([compressed items], [raw items])"""
    cs, rs = [], []
    for yy, sign in ((y, "+y"), ((c.q - y) % c.q, "-y")):
        cs.append(("%s %s %s" % (lab, sign, "large" if yy > (c.q - 1) // 2 else "small"), compress(c, x, yy)))
        rs.append(("%s %s" % (lab, sign), raw(c, x, yy)))
    return cs, rs


def _family(c: Curve, fam: str, pairs, pads, extra_comp=(), extra_raw=()) -> list:
    cs, rs = list(extra_comp), list(extra_raw)
    for lab, x, y in pairs:
        a, b = _both(c, lab, x, y)
        cs += a
        rs += b
    return _streams(c, fam, False, cs, pads) + _streams(c, fam, True, rs, pads)


# ---- A: square-root depth ----
def depth_points(name: str, per_depth: int = 2, seed: int = 1):
    """[(k, x, y)] with (x^3 + b)^t of order exactly 2^k, per_depth points for every k in [0, s)"""
    c = curve(name)
    q = c.q
    rng = random.Random(seed * 1000 + GID[name])
    out = []
    for k in range(c.s):
        zeta = pow(c.z_t, 1 << (c.s - k - 1), q)       # order 2^(k+1)
        got = 0
        while got < per_depth:
            y = zeta * pow(rng.randrange(1, q), 1 << c.s, q) % q
            xs = cube_roots((y * y - c.b) % q, q)
            if not xs:
                continue
            x = xs[rng.randrange(3)]
            assert sqrt_depth((x ** 3 + c.b) % q, c) == k
            out.append((k, x, y))
            got += 1
    return out


def non_residue_xs(name: str, m: int, seed: int = 2) -> list:
    c = curve(name)
    rng = random.Random(seed * 1000 + GID[name])
    out = []
    while len(out) < m:
        x = rng.randrange(c.q)
        if pow((x ** 3 + c.b) % c.q, (c.q - 1) // 2, c.q) == c.q - 1:
            assert sqrt_depth((x ** 3 + c.b) % c.q, c) == c.s
            out.append(x)
    return out


def family_a(name: str, pads) -> list:
    c = curve(name)
    pairs = [("depth %d #%d" % (k, i % 2), x, y) for i, (k, x, y) in enumerate(depth_points(name))]
    nr = [("non-residue x #%d %s" % (i, f), comp(c, x, getattr(c, f))) for i, x in enumerate(non_residue_xs(name, 2)) for f in ("small", "large")]
    return _family(c, "A", pairs, pads, extra_comp=nr)


# ---- B: sign boundary ----
def sign_points(name: str):
    """[(label, x, y)]: y = (q - 1)/2 - k for the smallest k that has a point (with all three x), and y = h +- u 2^(32 j) for every
    32-bit limb j with the smallest u that has a point and leaves the limbs above j equal to h's"""
    c = curve(name)
    q, h = c.q, (c.q + 1) // 2
    out = []
    k = 0
    while not cube_roots(((h - 1 - k) ** 2 - c.b) % q, q):
        k += 1
    assert k == SIGN_K[name], (name, k)
    for i, x in enumerate(cube_roots(((h - 1 - k) ** 2 - c.b) % q, q)):
        out.append(("y = (q-1)/2 - %d, x #%d" % (k, i), x, h - 1 - k))
    hl = limbs32(h, c)
    rng = random.Random(GID[name])
    for j in range(c.limbs32):
        above = (h >> (32 * (j + 1))) << (32 * (j + 1))
        for sign in (1, -1):
            # limb j moved by u within its room (no carry or borrow), the limbs below h's; failing that, limb j moved by one and
            # random limbs below.  A limb with no room on one side (h's limb 0 is 1 on bls12-377) is decided on the other only.
            room = (0xFFFFFFFF - hl[j]) if sign > 0 else hl[j]
            cands = [("y = h %s %d*2^%d" % ("+" if sign > 0 else "-", u, 32 * j), h + sign * u * (1 << (32 * j)))
                     for u in range(1, min(room, 64) + 1)]
            if room:
                cands += [("y: h's limbs above %d, limb %d %s 1, random below" % (j, j, "+" if sign > 0 else "-"),
                           above + ((hl[j] + sign) << (32 * j)) + rng.randrange(1 << (32 * j)) if j else
                           above + hl[j] + sign) for _ in range(64 if j else 0)]
            for lab, y in cands:
                yl = limbs32(y, c)
                assert 0 < y < q and yl[j + 1:] == hl[j + 1:] and (yl[j] > hl[j]) == (sign > 0) and yl[j] != hl[j]
                xs = cube_roots((y * y - c.b) % q, q)
                if xs:
                    out.append((lab, xs[0], y))
                    break
    return out


def family_b(name: str, pads) -> list:
    return _family(curve(name), "B", sign_points(name), pads)


# ---- C: element boundary ----
def boundary_values(name: str):
    """(above, below): integers >= q that fit below the flag bits, and integers < q decided against q at each limb"""
    c = curve(name)
    q, top = c.q, 1 << (8 * c.nb - c.nflag)
    ql = limbs32(q, c)
    above = [("q", q), ("q+1", q + 1)] + [("q+2^%d" % (32 * j), q + (1 << (32 * j))) for j in range(c.limbs32)]
    below = [("q-1", q - 1), ("q-2", q - 2)]
    for j in range(c.limbs32):
        hi = sum(ql[i] << (32 * i) for i in range(j + 1, c.limbs32))
        if ql[j] < 0xFFFFFFFF:
            above.append(("q's limbs above %d, limb %d + 1, zeroes below" % (j, j), hi + ((ql[j] + 1) << (32 * j))))
        if ql[j] > 0 and j > 0:
            below.append(("q's limbs above %d, limb %d - 1, ones below" % (j, j), hi + ((ql[j] - 1) << (32 * j)) + (1 << (32 * j)) - 1))
    # value bits between fp.Bits and the flags
    for p in range(q.bit_length(), 8 * c.nb - c.nflag):
        above.append(("value bit %d above fp.Bits" % p, 1 << p))
        above.append(("value bit %d and x = 1" % p, (1 << p) | 1))
    above = [(lab, v) for lab, v in above if v < top]
    assert all(v >= q for _, v in above) and all(v < q for _, v in below)
    return above, below


def family_c(name: str, pads) -> list:
    c = curve(name)
    q = c.q
    above, below = boundary_values(name)
    px, py = pads[0]
    cs, rs, rs_nocheck = [], [], []
    for lab, v in above + below:
        for f in ("small", "large"):
            cs.append(("x = %s %s" % (lab, f), comp(c, v, getattr(c, f))))
        rs.append(("x = %s" % lab, raw(c, v, py)))
        rs.append(("y = %s" % lab, raw(c, px, v)))
    for p in range(1, 1 << c.nflag):         # raw y has no flags: a flag-looking top byte is a value >= q
        e = bytearray(raw(c, px, py))
        e[c.nb] |= c.flag(p)
        rs.append(("y with top bits %s" % format(p, "0%db" % c.nflag), bytes(e)))
    rs_nocheck = [(lab, e) for lab, e in rs if lab.startswith("y = ")]
    pairs = []
    sb = sqrt_mod(c.b, c)
    if sb is not None:
        pairs.append(("x = 0", 0, sb))
    for i, x in enumerate(cube_roots(-c.b % q, q)):
        pairs.append(("y = 0, x #%d" % i, x, 0))
    out = _family(c, "C", pairs, pads, extra_comp=cs, extra_raw=rs)
    return out + _streams(c, "C", True, rs_nocheck, pads, check=False)


# ---- D: flags and infinity ----
def family_d(name: str, pads) -> list:
    c = curve(name)
    (px, py), (qx, qy) = pads
    out = []
    items = {False: [], True: []}
    for is_raw in (False, True):
        size = (2 if is_raw else 1) * c.nb
        for p in range(1 << c.nflag):
            pb = format(p, "0%db" % c.nflag)
            items[is_raw].append(("top bits %s, zero payload" % pb, bytes([c.flag(p)]) + bytes(size - 1)))
            e = bytearray(raw(c, px, py) if is_raw else comp(c, px, 0))
            e[0] = (e[0] & ~c.mask & 0xFF) | c.flag(p)
            items[is_raw].append(("top bits %s, payload of a point" % pb, bytes(e)))
        infs = [c.inf] if not is_raw else ([c.unc_inf] if c.unc_inf is not None else [])
        for f in infs:
            for bit in range(c.shift):
                items[is_raw].append(("infinity %02x with byte 0 bit %d" % (f, bit), bytes([f | (1 << bit)]) + bytes(size - 1)))
            for k in range(1, size):
                e = bytearray(size)
                e[0] = f
                e[k] = 1 << (k % 8)
                items[is_raw].append(("infinity %02x with byte %d = %02x" % (f, k, e[k]), bytes(e)))
    for is_raw in (False, True):
        # every case between two valid points, whatever its verdict: an infinity must not read its neighbours
        for lab, e in items[is_raw]:
            out.append(Stream(name, "D", lab, is_raw, [_pad(c, is_raw, pads[0]), e, _pad(c, is_raw, pads[1])],
                              ["valid neighbour", lab, "valid neighbour"]))
    # the other kind's infinity flag, beside zeroes and at the last index with zeroes or a valid point's bytes past the end
    other = [(False, c.unc_inf)] if c.unc_inf is not None else []
    other.append((True, c.inf))
    for is_raw, f in other:
        size = (2 if is_raw else 1) * c.nb
        e = bytes([f]) + bytes(size - 1)
        lab = "%02x (the other kind's infinity)" % f
        v = _pad(c, is_raw, pads[0])
        out.append(Stream(name, "D", lab + " before a zero point", is_raw, [v, e, bytes(size)], ["valid", lab, "zero bytes"]))
        out.append(Stream(name, "D", lab + " before another", is_raw, [v, e, e], ["valid", lab, lab]))
        for tail, tl in ((b"", "nothing"), (bytes(size), "zero bytes"), (_pad(c, is_raw, pads[1]), "a valid point")):
            out.append(Stream(name, "D", "%s at the last index, then %s past the end" % (lab, tl), is_raw, [v, v, e],
                              ["valid", "valid", lab], tail=tail))
        if is_raw:   # X half zero, Y half garbage
            g = bytearray(e)
            g[c.nb:] = qy.to_bytes(c.nb, "big")
            out.append(Stream(name, "D", lab + " with a non-zero Y half", is_raw, [v, bytes(g), v], ["valid", lab + ", Y half set", "valid"]))
    return out


# ---- E: first-error order ----
def family_e(name: str, pts) -> list:
    """errors planted in different blocks, the lower index with the higher code; pts: >= 521 valid points"""
    c = curve(name)
    n = 4 * BLOCK + 9
    out = []
    xbad = comp(c, c.q, c.small)
    nr = comp(c, non_residue_xs(name, 1, seed=5)[0], c.large)
    plans = {
        False: [
            [(5, BAD_FLAGS), (130, BAD_INFINITY), (n - 1, BAD_ELEMENT)],
            [(7, NO_SQRT), (200, BAD_ELEMENT), (300, BAD_INFINITY)],
            [(BLOCK - 1, BAD_FLAGS), (BLOCK, NO_SQRT), (2 * BLOCK, BAD_ELEMENT), (3 * BLOCK + 1, BAD_INFINITY)],
            [(n - 2, BAD_FLAGS), (n - 1, BAD_INFINITY)],
        ],
        True: [
            [(BLOCK - 1, NOT_ON_CURVE), (BLOCK, BAD_ELEMENT), (400, BAD_INFINITY), (n - 1, BAD_FLAGS)],
            [(3, BAD_FLAGS), (2 * BLOCK + 5, NOT_ON_CURVE), (3 * BLOCK + 7, BAD_ELEMENT)],
        ],
    }
    for is_raw, ps in plans.items():
        size = (2 if is_raw else 1) * c.nb
        for plan in ps:
            if is_raw and c.unc_inf is None:          # bn254 has no raw infinity flag
                plan = [(i, k) for i, k in plan if k != BAD_INFINITY]
            enc = [_pad(c, is_raw, p) for p in pts[:n]]
            labels = ["valid"] * n
            for i, code in plan:
                if code == BAD_FLAGS:
                    e = bytearray(enc[i])
                    e[0] = (e[0] & ~c.mask & 0xFF) | c.flag(0b001 if c.nflag == 3 else (0b10 if is_raw else 0b00))
                elif code == BAD_INFINITY:
                    e = bytearray(size)
                    e[0] = c.unc_inf if is_raw else c.inf
                    e[size // 2] = 0x80
                elif code == BAD_ELEMENT:
                    e = bytearray(raw(c, pts[i][0], c.q) if is_raw else xbad)
                elif code == NO_SQRT:
                    e = bytearray(nr)
                elif code == NOT_ON_CURVE:
                    e = bytearray(raw(c, pts[i][0], (pts[i][1] + 1) % c.q))
                enc[i] = bytes(e)
                labels[i] = "planted " + CODE_NAMES[code]
            s = Stream(name, "E", "errors " + ", ".join("%s@%d" % (CODE_NAMES[k], i) for i, k in plan), is_raw, enc, labels)
            assert s.expected()[1] == plan[0], (s.title(), s.expected()[1])
            assert [i for i, k in enumerate(s.expected()[2]) if k] == [i for i, _ in plan]
            out.append(s)
    return out


def pads(name: str, seed: int = 7) -> list:
    return subgroup_points(name, 2, seed)


def families(name: str) -> dict:
    """families A to E of one curve: {letter: [Stream]}"""
    p = pads(name)
    return {"A": family_a(name, p), "B": family_b(name, p), "C": family_c(name, p), "D": family_d(name, p),
            "E": family_e(name, subgroup_points(name, 4 * BLOCK + 9, 11))}


def accepted_encodings(name: str, is_raw: bool) -> list:
    """(label, encoding) of the accepted points of families A to C, one of each distinct encoding"""
    seen, out = set(), []
    p = pads(name)
    for s in family_a(name, p) + family_b(name, p) + family_c(name, p):
        if s.raw != is_raw or not s.check:
            continue
        for lab, e, k in zip(s.labels, s.points, s.expected()[2]):
            if k == OK and e not in seen:
                seen.add(e)
                out.append(("%s %s" % (s.family, lab), e))
    return out


def production_block(name: str, is_raw: bool, m: int = 1 << 16, seed: int = 13):
    """m distinct encodings of accepted points: those of families A to C, one infinity, then distinct subgroup points ->
    (encodings as an (m, point size) uint8 array, expected (m, words) uint64 rows, labels)"""
    c = curve(name)
    size = (2 if is_raw else 1) * c.nb
    head = accepted_encodings(name, is_raw)
    head.append(("infinity", bytes([c.unc_inf if is_raw else c.inf]) + bytes(size - 1)) if (c.unc_inf is not None or not is_raw)
                else ("infinity (0, 0)", bytes(size)))
    rows, pts = subgroup_rows(name, m - len(head), seed)
    enc = [e for _, e in head] + [_pad(c, is_raw, xy) for xy in pts]
    assert len(set(enc)) == m
    want = np.concatenate([np.stack([encode_point(c, decode_point(c, e, is_raw)[1]) for _, e in head]), rows])
    labels = [lab for lab, _ in head] + ["subgroup point %d" % i for i in range(len(pts))]
    return np.frombuffer(b"".join(enc), dtype=np.uint8).reshape(m, size), want, labels
