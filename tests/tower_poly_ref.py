"""Fp12 of bn254 and bls12-381 as one plain polynomial ring, with no Fp2 / Fp6 layering: an oracle for the tower operations that
shares no formula with tests/pairing_ref.py or tower.cuh.

  bn254:     Fp[w] / (w^12 - 18 w^6 + 82)   (xi = 9 + u, u = w^6 - 9, u^2 = -1)
  bls12-381: Fp[w] / (w^12 - 2 w^6 + 2)     (xi = 1 + u, u = w^6 - 1)

The GT layout maps in by C0.B0, C0.B1, C0.B2, C1.B0, C1.B1, C1.B2 -> w^0, w^2, w^4, w^1, w^3, w^5 (v = w^2, w^2 = v, v^3 = xi = w^6),
each Fp2 coefficient a0 + a1 u expanded with u = w^6 - xi0.  A ring element is a tuple of 12 coefficients, lowest degree first.
The operations are the definitions: a product is schoolbook multiplication and reduction, the inverse is pow(q^12 - 2) (so
0 -> 0), the Frobenius map of order k is pow(q^k) and the conjugation pow(q^6)."""
from tests import pairing_ref as PR

_POS = (0, 2, 4, 1, 3, 5)   # the power of w of C0.B0, C0.B1, C0.B2, C1.B0, C1.B1, C1.B2


class PolyTower:
    def __init__(self, curve: str):
        T = PR.tower(curve)
        self.T = T
        self.q = T.q
        self.r = T.r
        self.xi0 = T.xi[0]
        assert T.xi[1] == 1
        # w^12 = 2 xi0 w^6 - (xi0^2 + 1)
        self.m6 = 2 * self.xi0 % self.q
        self.m0 = (-(self.xi0 * self.xi0 + 1)) % self.q
        self._slot = 2 * self.q.bit_length() + 8   # Kronecker packing: 12 products of two residues fit a slot

    # ---- the map from and to the GT layout ----
    def embed(self, a):
        """a GT element (pairing_ref layout) as a ring element"""
        q, c = self.q, [0] * 12
        for (x0, x1), e in zip([x for half in a for x in half], _POS):
            c[e] = (c[e] + x0 - self.xi0 * x1) % q     # (x0 + x1 u) w^e, u = w^6 - xi0
            c[e + 6] = (c[e + 6] + x1) % q
        return tuple(c)

    def unembed(self, c):
        """the inverse of embed: the coefficient of w^e (e < 6) is c_e + c_{e+6} w^6 = (c_e + xi0 c_{e+6}) + c_{e+6} u"""
        q = self.q
        e2 = [((c[e] + self.xi0 * c[e + 6]) % q, c[e + 6] % q) for e in _POS]
        return (tuple(e2[:3]), tuple(e2[3:]))

    # ---- ring operations ----
    def mul(self, a, b):
        s = self._slot
        mask = (1 << s) - 1
        pa = sum(x << (s * i) for i, x in enumerate(a))
        pb = sum(x << (s * i) for i, x in enumerate(b))
        prod = pa * pb
        c = [(prod >> (s * i)) & mask for i in range(23)]
        for d in range(22, 11, -1):      # w^d = w^(d-12) (m6 w^6 + m0)
            t = c[d] % self.q
            c[d - 6] += self.m6 * t
            c[d - 12] += self.m0 * t
        return tuple(x % self.q for x in c[:12])

    def one(self):
        return (1,) + (0,) * 11

    def pow(self, a, e):
        assert e >= 0
        r = self.one()
        for bit in bin(e)[2:]:
            r = self.mul(r, r)
            if bit == "1":
                r = self.mul(r, a)
        return r

    def inv(self, a):
        return self.pow(a, self.q ** 12 - 2)

    def frob(self, a, k):
        return self.pow(a, self.q ** k)

    def conj(self, a):
        return self.pow(a, self.q ** 6)

    # ---- exponents of the pairing (meaningful on the cyclotomic subgroup) ----
    def final_exp_exponent(self):
        """s (q^12 - 1) / r: the reference's hard part computes a multiple of the textbook exponent, s = 2 x0 (6 x0^2 + 3 x0 + 1)
        for bn254 and 3 for bls12-381 (pinned by tests/test_pairing_ref_cpu.py)"""
        x0 = self.T.x0
        s = 2 * x0 * (6 * x0 ** 2 + 3 * x0 + 1) if self.T.curve == "bn254" else 3
        return s * (self.q ** 12 - 1) // self.r

    def gt_pow(self, a, e):
        """a^e with e taken mod q^12 - 1, so that negative exponents are inverses"""
        return self.pow(a, e % (self.q ** 12 - 1))


_CACHE = {}


def poly_tower(curve: str) -> PolyTower:
    if curve not in _CACHE:
        _CACHE[curve] = PolyTower(curve)
    return _CACHE[curve]
