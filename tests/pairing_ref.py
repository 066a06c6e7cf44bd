"""Big-int restatement of the bn254 and bls12-381 pairings: the Fp6 / Fp12 towers, the projective line steps, both MillerLoops
(with their n = 1 / n = 2 special cases and the shared squarings of the multi-pair loop) and both FinalExponentiation chains.

Replaces (reference): ecc/bn254/pairing.go (Pair :26, PairingCheck :38, FinalExponentiation :52, MillerLoop :111, doubleStep,
addMixedStep, lineCompute), ecc/bls12-381/pairing.go (FinalExponentiation, MillerLoop :103-233, doubleStep, addMixedStep,
tangentLine), and the towers ecc/<curve>/internal/fptower/{e6,e12,e12_pairing,frobenius}.go.  Values are plain integers (not
Montgomery); E2 = (A0, A1), E6 = (B0, B1, B2), E12 = (C0, C1), Fp6 = Fp2[v]/(v^3 - xi), Fp12 = Fp6[w]/(w^2 - v).
In memory a GT element is 12 Montgomery fp.Elements in the order C0.B0.A0, C0.B0.A1, C0.B1.A0, ..., C1.B2.A1."""
import numpy as np

from oracle import oracle as O

CURVES = {
    # field, xi, twist kind, x0, G1 group, G2 group
    "bn254": dict(fp="bn254_fp", xi=(9, 1), twist="d", x0=4965661367192848881, g1="bn254_g1", g2="bn254_g2"),
    "bls12381": dict(fp="bls12381_fp", xi=(1, 1), twist="m", x0=-15132376222941642752, g1="bls12381_g1", g2="bls12381_g2"),
}


def naf(a):
    """ecc.NafDecomposition: least significant digit first"""
    d = []
    while a:
        if a & 1 == 0:
            d.append(0)
        elif a & 3 == 3:
            d.append(-1)
            a += 1
        else:
            d.append(1)
        a >>= 1
    return d


class Tower:
    def __init__(self, curve: str):
        c = CURVES[curve]
        self.curve = curve
        self.fp = O.FIELDS[c["fp"]]
        self.q = q = self.fp.q
        self.r = O.GROUPS[c["g1"]].fr.q
        self.xi = c["xi"]
        self.twist = c["twist"]
        self.x0 = c["x0"]
        self.G1 = O.GROUPS[c["g1"]]
        self.G2 = O.GROUPS[c["g2"]]
        self.K2 = self.G2.K
        self.btwist = self.G2.b
        if curve == "bn254":
            self.loop = naf(6 * self.x0 + 2)
        else:
            self.loop = [(-self.x0 >> i) & 1 for i in range(64)]
        # gamma[k][e] = xi^(e (p^k - 1) / 6)
        self.gamma = {k: [None] + [self.e2_pow(self.xi, e * (q ** k - 1) // 6) for e in range(1, 6)] for k in (1, 2, 3)}
        self.inv2 = pow(2, -1, q)

    # ---- E2 ----
    def e2_add(self, a, b):
        return ((a[0] + b[0]) % self.q, (a[1] + b[1]) % self.q)

    def e2_sub(self, a, b):
        return ((a[0] - b[0]) % self.q, (a[1] - b[1]) % self.q)

    def e2_neg(self, a):
        return ((-a[0]) % self.q, (-a[1]) % self.q)

    def e2_dbl(self, a):
        return self.e2_add(a, a)

    def e2_mul(self, a, b):
        q = self.q
        return ((a[0] * b[0] - a[1] * b[1]) % q, (a[0] * b[1] + a[1] * b[0]) % q)

    def e2_sqr(self, a):
        return self.e2_mul(a, a)

    def e2_inv(self, a):
        q = self.q
        n = (a[0] * a[0] + a[1] * a[1]) % q
        ni = pow(n, -1, q) if n else 0
        return (a[0] * ni % q, (-a[1] * ni) % q)

    def e2_conj(self, a):
        return (a[0], (-a[1]) % self.q)

    def e2_by_fp(self, a, s):
        return (a[0] * s % self.q, a[1] * s % self.q)

    def e2_halve(self, a):
        return self.e2_by_fp(a, self.inv2)

    def e2_nr(self, a):   # MulByNonResidue: times xi
        return self.e2_mul(a, self.xi)

    def e2_pow(self, a, e):
        r = (1, 0)
        while e:
            if e & 1:
                r = self.e2_mul(r, a)
            a = self.e2_mul(a, a)
            e >>= 1
        return r

    # ---- E6 ----
    def e6_add(self, a, b):
        return tuple(self.e2_add(x, y) for x, y in zip(a, b))

    def e6_sub(self, a, b):
        return tuple(self.e2_sub(x, y) for x, y in zip(a, b))

    def e6_neg(self, a):
        return tuple(self.e2_neg(x) for x in a)

    def e6_mul(self, a, b):
        m = self.e2_mul
        a0, a1, a2 = a
        b0, b1, b2 = b
        c0 = self.e2_add(m(a0, b0), self.e2_nr(self.e2_add(m(a1, b2), m(a2, b1))))
        c1 = self.e2_add(self.e2_add(m(a0, b1), m(a1, b0)), self.e2_nr(m(a2, b2)))
        c2 = self.e2_add(self.e2_add(m(a0, b2), m(a1, b1)), m(a2, b0))
        return (c0, c1, c2)

    def e6_nr(self, a):   # times v
        return (self.e2_nr(a[2]), a[0], a[1])

    def e6_inv(self, a):
        a0, a1, a2 = a
        m, s, sub = self.e2_mul, self.e2_sqr, self.e2_sub
        t0 = sub(s(a0), self.e2_nr(m(a1, a2)))
        t1 = sub(self.e2_nr(s(a2)), m(a0, a1))
        t2 = sub(s(a1), m(a0, a2))
        d = self.e2_add(m(a0, t0), self.e2_nr(self.e2_add(m(a2, t1), m(a1, t2))))
        di = self.e2_inv(d)
        return (m(t0, di), m(t1, di), m(t2, di))

    # ---- E12 ----
    def one(self):
        return (((1, 0), (0, 0), (0, 0)), ((0, 0), (0, 0), (0, 0)))

    def zero(self):
        return (((0, 0),) * 3, ((0, 0),) * 3)

    def mul(self, a, b):
        t0 = self.e6_mul(a[0], b[0])
        t1 = self.e6_mul(a[1], b[1])
        c1 = self.e6_sub(self.e6_sub(self.e6_mul(self.e6_add(a[0], a[1]), self.e6_add(b[0], b[1])), t0), t1)
        return (self.e6_add(t0, self.e6_nr(t1)), c1)

    def sqr(self, a):
        return self.mul(a, a)

    def conj(self, a):
        return (a[0], self.e6_neg(a[1]))

    def inv(self, a):
        t = self.e6_sub(self.e6_mul(a[0], a[0]), self.e6_nr(self.e6_mul(a[1], a[1])))
        ti = self.e6_inv(t)
        return (self.e6_mul(a[0], ti), self.e6_neg(self.e6_mul(a[1], ti)))

    def frob(self, a, k):
        """a^(p^k): coefficient of w^e (C0.B0, C0.B1, C0.B2, C1.B0, C1.B1, C1.B2 -> e = 0, 2, 4, 1, 3, 5) conjugated for odd k,
        times gamma[k][e]"""
        out = []
        for half, exps in ((a[0], (0, 2, 4)), (a[1], (1, 3, 5))):
            cs = []
            for x, e in zip(half, exps):
                y = self.e2_conj(x) if k & 1 else x
                cs.append(y if e == 0 else self.e2_mul(y, self.gamma[k][e]))
            out.append(tuple(cs))
        return tuple(out)

    def cyclo_sqr(self, x):
        """Granger-Scott squaring (e12.go CyclotomicSquare); x0..x5 = C0.B0, C1.B1, C0.B2, C1.B0, C0.B1, C1.B2"""
        a, s, sub, nr = self.e2_add, self.e2_sqr, self.e2_sub, self.e2_nr
        (b00, b01, b02), (b10, b11, b12) = x
        t0, t1 = s(b11), s(b00)
        t6 = sub(sub(s(a(b11, b00)), t0), t1)
        t2, t3 = s(b02), s(b10)
        t7 = sub(sub(s(a(b02, b10)), t2), t3)
        t4, t5 = s(b12), s(b01)
        t8 = nr(sub(sub(s(a(b12, b01)), t4), t5))
        t0 = a(nr(t0), t1)
        t2 = a(nr(t2), t3)
        t4 = a(nr(t4), t5)
        z00 = a(self.e2_dbl(sub(t0, b00)), t0)
        z01 = a(self.e2_dbl(sub(t2, b01)), t2)
        z02 = a(self.e2_dbl(sub(t4, b02)), t4)
        z10 = a(self.e2_dbl(a(t8, b10)), t8)
        z11 = a(self.e2_dbl(a(t6, b11)), t6)
        z12 = a(self.e2_dbl(a(t7, b12)), t7)
        return ((z00, z01, z02), (z10, z11, z12))

    def cyclo_sqr_compressed(self, x):
        """e12.go CyclotomicSquareCompressed: updates C0.B1, C0.B2, C1.B0, C1.B2 (the others are kept)"""
        a, s, sub, nr, d = self.e2_add, self.e2_sqr, self.e2_sub, self.e2_nr, self.e2_dbl
        (b00, b01, b02), (b10, b11, b12) = x
        t0, t1 = s(b01), s(b12)
        t2 = s(a(b01, b12))
        t5 = sub(t2, a(t0, t1))
        t3 = s(a(b10, b02))
        t2 = s(b10)
        t6 = nr(t5)
        z10 = a(d(a(t6, b10)), t6)
        t5 = a(t0, nr(t1))
        z02 = a(d(sub(t5, b02)), t5)
        t1 = s(b02)
        t5 = a(t2, nr(t1))
        z01 = a(d(sub(t5, b01)), t5)
        t5 = sub(t3, a(t2, t1))
        z12 = a(t5, d(a(t5, b12)))
        return ((b00, z01, z02), (z10, b11, z12))

    def decompress_karabina(self, x):
        """e12.go DecompressKarabina / BatchDecompressKarabina (the batch inversion gives the same values)"""
        a, s, sub, nr, d, m = self.e2_add, self.e2_sqr, self.e2_sub, self.e2_nr, self.e2_dbl, self.e2_mul
        (b00, b01, b02), (b10, b11, b12) = x
        if b12 == (0, 0):
            t0 = d(m(b01, b12))
            t1 = b02
            if t1 == (0, 0):
                return self.one()
        else:
            t0 = s(b01)
            t1 = a(d(sub(t0, b02)), t0)
            t0 = a(nr(s(b12)), t1)
            t1 = d(d(b10))
        g1 = m(t0, self.e2_inv(t1))
        t1 = m(b02, b01)
        t2 = sub(d(sub(s(g1), t1)), t1)
        t2 = a(t2, m(b10, b12))
        g0 = a(nr(t2), (1, 0))
        return ((g0, b01, b02), (b10, g1, b12))

    def nsqr(self, x, n):
        for _ in range(n):
            x = self.cyclo_sqr(x)
        return x

    def expt(self, x):
        if self.curve == "bn254":
            return self._expt_bn254(x)
        return self.cyclo_sqr(self.expt_half(x))

    def _expt_bn254(self, x):
        """e12_pairing.go Expt (bn254): x^x0 by the reference's addition chain"""
        S, M = self.cyclo_sqr, self.mul
        t3 = S(x)
        t5 = S(t3)
        result = S(t5)
        t0 = S(result)
        t2 = M(x, t0)
        t0 = M(t3, t2)
        t1 = M(x, t0)
        t4 = M(result, t2)
        t6 = S(t2)
        t1 = M(t0, t1)
        t0 = M(t3, t1)
        t6 = self.nsqr(t6, 6)
        t5 = M(t5, t6)
        t5 = M(t4, t5)
        t5 = self.nsqr(t5, 7)
        t4 = M(t4, t5)
        t4 = self.nsqr(t4, 8)
        t4 = M(t0, t4)
        t3 = M(t3, t4)
        t3 = self.nsqr(t3, 6)
        t2 = M(t2, t3)
        t2 = self.nsqr(t2, 8)
        t2 = M(t0, t2)
        t2 = self.nsqr(t2, 6)
        t2 = M(t0, t2)
        t2 = self.nsqr(t2, 10)
        t1 = M(t1, t2)
        t1 = self.nsqr(t1, 6)
        t0 = M(t0, t1)
        return M(result, t0)

    def expt_half(self, x):
        """e12_pairing.go ExptHalf (bls12-381): x^(x0 / 2), compressed squarings and Karabina decompression"""
        r = x
        for _ in range(15):
            r = self.cyclo_sqr_compressed(r)
        t0 = r
        for _ in range(32):
            r = self.cyclo_sqr_compressed(r)
        t1 = r
        b0, b1 = self.decompress_karabina(t0), self.decompress_karabina(t1)
        res = self.mul(b0, b1)
        b1 = self.nsqr(b1, 9)
        res = self.mul(res, b1)
        b1 = self.nsqr(b1, 3)
        res = self.mul(res, b1)
        b1 = self.nsqr(b1, 2)
        res = self.mul(res, b1)
        b1 = self.cyclo_sqr(b1)
        res = self.mul(res, b1)
        return self.conj(res)

    # ---- final exponentiation ----
    def final_exp(self, z, *zs):
        M, C, F = self.mul, self.conj, self.frob
        result = z
        for e in zs:
            result = M(result, e)
        t0 = M(C(result), self.inv(result))
        result = M(F(t0, 2), t0)
        if result == self.one():
            return result
        if self.curve == "bn254":
            S, E = self.cyclo_sqr, self.expt
            t0 = S(C(E(result)))
            t1 = M(t0, S(t0))
            t2 = C(E(t1))
            t3 = C(t1)
            t1 = M(t2, t3)
            t3 = S(t2)
            t4 = M(t1, E(t3))
            t3 = M(t0, t4)
            t0 = M(result, M(t2, t4))
            t0 = M(F(t3, 1), t0)
            t0 = M(F(t4, 2), t0)
            t2 = F(M(C(result), t3), 3)
            return M(t2, t0)
        S, E = self.cyclo_sqr, self.expt
        t0 = S(result)
        t1 = M(self.expt_half(t0), C(result))
        t2 = E(t1)
        t1 = M(C(t1), t2)
        t2 = E(t1)
        t1 = M(F(t1, 1), t2)
        result = M(result, t0)
        t0 = E(t1)
        t2 = E(t0)
        t0 = F(t1, 2)
        t1 = M(M(C(t1), t2), t0)
        return M(result, t1)

    # ---- line steps on g2Proj (x, y, z) ----
    def double_step(self, p):
        a, s, sub, m, d = self.e2_add, self.e2_sqr, self.e2_sub, self.e2_mul, self.e2_dbl
        x, y, z = p
        A = self.e2_halve(m(x, y))
        B = s(y)
        C = s(z)
        D = a(d(C), C)
        E = m(D, self.btwist)
        F = a(d(E), E)
        G = self.e2_halve(a(B, F))
        H = sub(s(a(y, z)), a(B, C))
        I = sub(E, B)
        J = s(x)
        EE = s(E)
        K = a(d(EE), EE)
        np_ = (m(sub(B, F), A), sub(s(G), K), m(B, H))
        if self.twist == "d":
            line = (self.e2_neg(H), a(d(J), J), I)
        else:
            line = (I, a(d(J), J), self.e2_neg(H))
        return np_, line

    def _add_line(self, p, qa):
        x, y, z = p
        O_ = self.e2_sub(y, self.e2_mul(qa[1], z))
        L = self.e2_sub(x, self.e2_mul(qa[0], z))
        J = self.e2_sub(self.e2_mul(qa[0], O_), self.e2_mul(L, qa[1]))
        if self.twist == "d":
            line = (L, self.e2_neg(O_), J)
        else:
            line = (J, self.e2_neg(O_), L)
        return O_, L, line

    def add_mixed_step(self, p, qa):
        a, s, sub, m, d = self.e2_add, self.e2_sqr, self.e2_sub, self.e2_mul, self.e2_dbl
        x, y, z = p
        O_, L, line = self._add_line(p, qa)
        C = s(O_)
        D = s(L)
        E = m(L, D)
        F = m(z, C)
        G = m(x, D)
        H = sub(a(E, F), d(G))
        t1 = m(y, E)
        np_ = (m(L, H), sub(m(sub(G, H), O_), t1), m(E, z))
        return np_, line

    def line_compute(self, p, qa):
        return self._add_line(p, qa)[2]

    def tangent_line(self, p):
        return self.double_step(p)[1]

    def scale(self, line, P):
        """bn254: r0 *= P.y, r1 *= P.x; bls12-381: r1 *= P.x, r2 *= P.y"""
        r0, r1, r2 = line
        if self.twist == "d":
            return (self.e2_by_fp(r0, P[1]), self.e2_by_fp(r1, P[0]), r2)
        return (r0, self.e2_by_fp(r1, P[0]), self.e2_by_fp(r2, P[1]))

    def sparse(self, line):
        """a line as a full E12: bn254 at positions 0, 3, 4 (C0.B0, C1.B0, C1.B1); bls12-381 at 0, 1, 4 (C0.B0, C0.B1, C1.B1)"""
        Z = (0, 0)
        if self.twist == "d":
            return ((line[0], Z, Z), (line[1], line[2], Z))
        return ((line[0], line[1], Z), (Z, line[2], Z))

    def mul_line(self, f, line):
        return self.mul(f, self.sparse(line))

    # ---- Miller loops ----
    def miller_loop(self, P, Q):
        """MillerLoop(P, Q): P affine G1 (x, y), Q affine G2 ((x0, x1), (y0, y1)); infinity = zeros, skipped"""
        if len(P) == 0 or len(P) != len(Q):
            raise ValueError("invalid inputs sizes")
        pairs = [(p, q) for p, q in zip(P, Q) if not (self.G1.aff_is_inf(p) or self.G2.aff_is_inf(q))]
        if self.curve == "bn254":
            return self._miller_bn254(pairs)
        return self._miller_bls12381(pairs)

    def _miller_bn254(self, pairs):
        n = len(pairs)
        p = [a for a, _ in pairs]
        q = [b for _, b in pairs]
        qn = [(b[0], self.e2_neg(b[1])) for b in q]
        qp = [(b[0], b[1], (1, 0)) for b in q]
        result = self.one()
        # first doubling: the n = 1 / n = 2 special cases of the reference build the same product from 1
        for k in range(n):
            qp[k], l1 = self.double_step(qp[k])
            result = self.mul_line(result, self.scale(l1, p[k]))
        result = self.sqr(result)
        for k in range(n):
            l2 = self.scale(self.line_compute(qp[k], qn[k]), p[k])
            qp[k], l1 = self.add_mixed_step(qp[k], q[k])
            result = self.mul_line(self.mul_line(result, self.scale(l1, p[k])), l2)
        for i in range(len(self.loop) - 4, -1, -1):
            result = self.sqr(result)
            for k in range(n):
                qp[k], l1 = self.double_step(qp[k])
                result = self.mul_line(result, self.scale(l1, p[k]))
                if self.loop[i] != 0:
                    qp[k], l2 = self.add_mixed_step(qp[k], q[k] if self.loop[i] == 1 else qn[k])
                    result = self.mul_line(result, self.scale(l2, p[k]))
        for k in range(n):
            X, Y = q[k]
            q1 = (self.e2_mul(self.e2_conj(X), self.gamma[1][2]), self.e2_mul(self.e2_conj(Y), self.gamma[1][3]))
            q2 = (self.e2_mul(X, self.gamma[2][2]), self.e2_neg(self.e2_mul(Y, self.gamma[2][3])))
            qp[k], l2 = self.add_mixed_step(qp[k], q1)
            l1 = self.line_compute(qp[k], q2)
            result = self.mul_line(self.mul_line(result, self.scale(l2, p[k])), self.scale(l1, p[k]))
        return result

    def _miller_bls12381(self, pairs):
        n = len(pairs)
        p = [a for a, _ in pairs]
        q = [b for _, b in pairs]
        qp = [(b[0], b[1], (1, 0)) for b in q]
        result = self.one()
        for k in range(n):
            qp[k], l1 = self.double_step(qp[k])
            qp[k], l2 = self.add_mixed_step(qp[k], q[k])
            result = self.mul_line(self.mul_line(result, self.scale(l1, p[k])), self.scale(l2, p[k]))
        for i in range(len(self.loop) - 3, 0, -1):
            result = self.sqr(result)
            for k in range(n):
                qp[k], l1 = self.double_step(qp[k])
                result = self.mul_line(result, self.scale(l1, p[k]))
                if self.loop[i] != 0:
                    qp[k], l2 = self.add_mixed_step(qp[k], q[k])
                    result = self.mul_line(result, self.scale(l2, p[k]))
        result = self.sqr(result)
        for k in range(n):
            result = self.mul_line(result, self.scale(self.tangent_line(qp[k]), p[k]))
        return self.conj(result)

    def pair(self, P, Q):
        return self.final_exp(self.miller_loop(P, Q))

    def pairing_check(self, P, Q):
        return self.pair(P, Q) == self.one()

    # ---- memory layout ----
    def flat(self, a):
        return [c for half in a for e2 in half for c in e2]

    def unflat(self, v):
        v = [int(x) % self.q for x in v]
        e2 = [(v[2 * i], v[2 * i + 1]) for i in range(6)]
        return ((e2[0], e2[1], e2[2]), (e2[3], e2[4], e2[5]))

    def encode(self, elems) -> np.ndarray:
        L = self.fp.limbs
        out = np.zeros((len(elems), 12 * L), dtype=np.uint64)
        for i, a in enumerate(elems):
            out[i] = [w for c in self.flat(a) for w in self.fp.to_limbs(self.fp.to_mont(c))]
        return out

    def decode(self, arr) -> list:
        L = self.fp.limbs
        arr = np.asarray(arr, dtype=np.uint64).reshape(-1, 12 * L)
        return [self.unflat([self.fp.from_mont(O.Field.from_limbs([int(w) for w in r[L * j: L * (j + 1)]])) for j in range(12)])
                for r in arr]

    def gt_pow(self, a, e):
        r = self.one()
        while e:
            if e & 1:
                r = self.mul(r, a)
            a = self.mul(a, a)
            e >>= 1
        return r


_TOWERS = {}


def tower(curve: str) -> Tower:
    if curve not in _TOWERS:
        _TOWERS[curve] = Tower(curve)
    return _TOWERS[curve]
