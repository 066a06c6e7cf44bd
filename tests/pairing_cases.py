"""Shared inputs of the pairing tests, as restatement values (tests/pairing_ref.py) and the reference's memory layout: random pairs,
off-subgroup and small-order points, adversarial tower operands by family, DecompressKarabina's branch inputs, and the table of
the tower test ops (gmsm_test_tower_op) with the restatement's value of each."""
import random

import numpy as np

from oracle import oracle as O
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


def off_subgroup_g2(n: int, seed: int, curve: str = "bn254"):
    """twist points outside the r-torsion: random x until x^3 + b' is a square in Fp2, kept when [r]Q is not infinity"""
    T = PR.tower(curve)
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


# ---- adversarial tower operands (the E2 / E6 / E12 tuples of tests/pairing_ref.py) ----
def edge_fp(q: int):
    """coordinates where modular arithmetic goes wrong: 0, 1, 2, q - 1, (q - 1) / 2, (q + 1) / 2"""
    return [0, 1, 2, q - 1, (q - 1) // 2, (q + 1) // 2]


def adversarial_e2(curve: str, seed: int, n_random: int = 4):
    """every pair of edge coordinates, then random values, and random values with a0 = 0 or a1 = 0"""
    T = PR.tower(curve)
    rng = random.Random(seed)
    ed = edge_fp(T.q)
    out = [(x, y) for x in ed for y in ed]
    for _ in range(n_random):
        out += [(rng.randrange(T.q), rng.randrange(T.q)), (0, rng.randrange(T.q)), (rng.randrange(T.q), 0)]
    return out


def random_e2(T, rng):
    return (rng.randrange(T.q), rng.randrange(T.q))


def random_e12(T, rng):
    return T.unflat([rng.randrange(T.q) for _ in range(12)])


def from_components(c):
    """six E2 components in memory order (C0.B0, C0.B1, C0.B2, C1.B0, C1.B1, C1.B2) as an E12"""
    return (tuple(c[:3]), tuple(c[3:]))


def components(a):
    return [x for half in a for x in half]


def cyclotomic(T, z):
    """the easy part of the final exponentiation, z^((q^6 - 1)(q^2 + 1)): an element of the cyclotomic subgroup"""
    t0 = T.mul(T.conj(z), T.inv(z))
    return T.mul(T.frob(t0, 2), t0)


def adversarial_e12(curve: str, seed: int):
    """families of E12 operands, by name: one non-zero component at each of the six positions (an edge or a random value), a
    zero C0, a zero C1, zero, one, components drawn from the edge E2 values, random elements, and genuine cyclotomic elements"""
    T = PR.tower(curve)
    rng = random.Random(seed)
    e2s = adversarial_e2(curve, seed)
    Z = (0, 0)
    fam = {}
    fam["single"] = [from_components([v if j == pos else Z for j in range(6)])
                     for pos in range(6) for v in ((1, 0), (T.q - 1, T.q - 1), (0, 1), random_e2(T, rng))]
    fam["zero_c0"] = [(((Z,) * 3), T.unflat([0] * 6 + [rng.randrange(T.q) for _ in range(6)])[1]) for _ in range(3)]
    fam["zero_c1"] = [(T.unflat([rng.randrange(T.q) for _ in range(6)] + [0] * 6)[0], (Z,) * 3) for _ in range(3)]
    fam["zero_one"] = [T.zero(), T.one()]
    fam["edge"] = [from_components([e2s[rng.randrange(len(e2s))] for _ in range(6)]) for _ in range(12)]
    fam["random"] = [random_e12(T, rng) for _ in range(6)]
    fam["cyclotomic"] = [cyclotomic(T, random_e12(T, rng)) for _ in range(4)]
    return fam


def karabina_cases(curve: str, seed: int):
    """DecompressKarabina operands in each of its branches, with the other components random and non-zero:
    'g5zero' C1.B2 = 0 with C0.B2 != 0; 'g5g2zero' C1.B2 = C0.B2 = 0 (the branch that returns one); 'g3zero' C1.B2 != 0 with
    C1.B0 = 0 (a division by zero, whose inverse is zero); 'generic' no zero component"""
    T = PR.tower(curve)
    rng = random.Random(seed)
    Z = (0, 0)
    out = {"g5zero": [], "g5g2zero": [], "g3zero": [], "generic": []}
    for _ in range(4):
        c = [random_e2(T, rng) for _ in range(6)]
        out["generic"].append(from_components(c))
        out["g5zero"].append(from_components(c[:5] + [Z]))
        out["g5g2zero"].append(from_components(c[:2] + [Z] + c[3:5] + [Z]))
        out["g3zero"].append(from_components(c[:3] + [Z] + c[4:]))
    return out


def karabina_branch(a):
    """which branch of DecompressKarabina the operand takes (the names of karabina_cases)"""
    (_, _, b02), (b10, _, b12) = a
    if b12 == (0, 0):
        return "g5g2zero" if b02 == (0, 0) else "g5zero"
    return "g3zero" if b10 == (0, 0) else "generic"


# ---- points on which the Miller loop degenerates ----
# the G2 cofactors: bn254 2q - r; bls12-381 (x^8 - 4x^7 + 5x^6 - 4x^4 + 6x^3 - 4x^2 - 4x + 13) / 9, which has the factors 13^2,
# 23^2, 2713, 11953 and 262069 below 10^6; bn254's has 10069
def g2_cofactor(curve: str) -> int:
    T = PR.tower(curve)
    if curve == "bn254":
        return 2 * T.q - T.r
    x = T.x0
    return (x ** 8 - 4 * x ** 7 + 5 * x ** 6 - 4 * x ** 4 + 6 * x ** 3 - 4 * x ** 2 - 4 * x + 13) // 9


def _random_twist_point(T, rng, x_in_fp=False):
    while True:
        x = (rng.randrange(T.q), 0 if x_in_fp else rng.randrange(T.q))
        y = _e2_sqrt(T, T.e2_add(T.e2_mul(T.e2_sqr(x), x), T.btwist))
        if y is not None:
            return (x, y)


def small_order_g2(curve: str, ell: int, n: int, seed: int):
    """n twist points of prime order ell: S = [#E'/ell^v]R for random twist points R (#E' = r times the cofactor, ell^v the
    largest power of ell dividing it), then S = [ell]S until [ell]S is infinity.  (With ell^2 | #E' the ell-torsion may be all
    of Z/ell x Z/ell, so [#E'/ell]R alone can vanish for every R.)"""
    T = PR.tower(curve)
    N = T.r * g2_cofactor(curve)
    assert N % ell == 0
    m = N
    while m % ell == 0:
        m //= ell
    rng = random.Random(seed)
    out = []
    while len(out) < n:
        pt = T.G2.scalar_mul(_random_twist_point(T, rng), m)
        if pt == T.G2.aff_inf():
            continue
        while (nxt := T.G2.scalar_mul(pt, ell)) != T.G2.aff_inf():
            pt = nxt
        out.append(pt)
    return out


def g2_x_in_fp(curve: str, n: int, seed: int):
    """twist points with X.A1 = 0 (outside the r-torsion for these seeds)"""
    T = PR.tower(curve)
    rng = random.Random(seed)
    return [_random_twist_point(T, rng, x_in_fp=True) for _ in range(n)]


def off_subgroup_g1(curve: str, n: int, seed: int):
    """G1 curve points outside the r-torsion: random x until x^3 + b is a square, the cofactor left uncleared"""
    assert curve != "bn254"   # bn254 G1 is the r-torsion
    T = PR.tower(curve)
    q = T.q
    rng = random.Random(seed)
    out = []
    while len(out) < n:
        x = rng.randrange(q)
        rhs = (x * x * x + T.G1.b) % q
        y = pow(rhs, (q + 1) // 4, q)
        if y * y % q != rhs:
            continue
        if T.G1.scalar_mul((x, y), T.r) != T.G1.aff_inf():
            out.append((x, y))
    return out


def bls12381_g1_order3():
    """(0, 2) and (0, -2) on y^2 = x^3 + 4: the 3-torsion of bls12-381 G1, off the r-torsion, with x = 0"""
    T = PR.tower("bls12381")
    return [(0, 2), (0, T.q - 2)]


# ---- the tower ops of gmsm_test_tower_op (include/gmsm.h GMSM_TOWER_OP_*) ----
# name: (op id, operand widths in E2 units (a, b), output width)
TOWER_OPS = {
    "e6_mul": (0, 3, 3, 3), "e6_inv": (1, 3, 0, 3), "e6_mul_by_01": (2, 3, 2, 3), "e6_mul_by_1": (3, 3, 1, 3),
    "e6_mul_by_12": (4, 3, 2, 3), "mul": (5, 6, 6, 6), "sqr": (6, 6, 0, 6), "inv": (7, 6, 0, 6), "conj": (8, 6, 0, 6),
    "frob1": (9, 6, 0, 6), "frob2": (10, 6, 0, 6), "frob3": (11, 6, 0, 6), "cyclo_sqr": (12, 6, 0, 6),
    "cyclo_sqr_compressed": (13, 6, 0, 6), "decompress_karabina": (14, 6, 0, 6), "expt": (15, 6, 0, 6), "expt_half": (16, 6, 0, 6),
    "mul_by_line": (17, 6, 3, 6), "line_by_line": (18, 3, 3, 5), "mul_by_two_lines": (19, 6, 5, 6), "double_step": (20, 3, 0, 6),
    "add_mixed_step": (21, 3, 2, 6), "line_compute": (22, 3, 2, 6), "final_exp": (23, 6, 0, 6), "miller_loop_one": (24, 1, 2, 6),
}


def tower_op_cases(curve: str, name: str, seed: int):
    """(family, a, b) operands of one op, a and b lists of E2 at the op's widths: every adversarial E12 family (its halves for the
    E6 ops), the DecompressKarabina branch inputs for the compressed squaring and decompression, lines and products of lines built
    from edge E2 values, G2 projective points at Z = 0, at T = Q and T = -Q and at edge coordinates, and degenerate pairs for the
    Miller loop"""
    T = PR.tower(curve)
    rng = random.Random(seed)
    _, wa, wb, _ = TOWER_OPS[name]
    e2s = adversarial_e2(curve, seed)
    pick = lambda k: [e2s[rng.randrange(len(e2s))] for _ in range(k)]
    fam = adversarial_e12(curve, seed)
    if name in ("cyclo_sqr_compressed", "decompress_karabina", "expt", "expt_half", "final_exp", "cyclo_sqr"):
        fam.update(karabina_cases(curve, seed + 1))
    if name == "final_exp":
        fam["subfield"] = [from_components([random_e2(T, rng)] + [(0, 0)] * 5), from_components([(rng.randrange(T.q), 0)] + [(0, 0)] * 5),
                           from_components([random_e2(T, rng) for _ in range(3)] + [(0, 0)] * 3),
                           from_components([(0, 0)] * 3 + [random_e2(T, rng)] + [(0, 0)] * 2)]
    flat = [(f, components(x)) for f in sorted(fam) for x in fam[f]]
    Z = (0, 0)
    out = []
    if wa == 3 and name.startswith("e6"):
        halves = [(f, c[h * 3:(h + 1) * 3]) for f, c in flat for h in (0, 1)]
        for i, (f, a) in enumerate(halves):
            b = halves[(7 * i + 3) % len(halves)][1] if wb == 3 else pick(wb)
            out.append((f, a, b))
    elif wa == 6:
        for i, (f, a) in enumerate(flat):
            if wb == 6:
                b = flat[(5 * i + 1) % len(flat)][1]
            elif wb == 3:   # a line: an edge value at each coefficient, some zero
                b = pick(3)
            elif wb == 5:
                b = pick(5)
            else:
                b = []
            out.append((f, a, b))
    elif name == "line_by_line":
        lines = [pick(3) for _ in range(40)] + [[Z, Z, Z], [(1, 0), Z, Z], [Z, (1, 0), Z], [Z, Z, (1, 0)]]
        for i, a in enumerate(lines):
            out.append(("edge" if i < 40 else "unit", a, lines[(3 * i + 1) % len(lines)]))
        out.append(("zero", [Z, Z, Z], pick(3)))
    elif name in ("double_step", "add_mixed_step", "line_compute"):
        P, Q = random_pairs(curve, 4, seed)
        small = small_order_g2(curve, 10069 if curve == "bn254" else 13, 2, seed)
        for q in Q + small:
            z = random_e2(T, rng)
            proj = [T.e2_mul(q[0], z), T.e2_mul(q[1], z), z]
            neg = (q[0], T.e2_neg(q[1]))
            out += [("t_eq_q", proj, list(q)), ("t_eq_minus_q", proj, list(neg)),
                    ("z_zero", [q[0], q[1], Z], list(q)), ("affine", [q[0], q[1], (1, 0)], list(Q[0]))]
        out += [("edge", pick(3), pick(2)) for _ in range(16)]
        out += [("zero", [Z, Z, Z], [Z, Z])]
        if wb == 0:
            out = [(f, a, []) for f, a, _ in out]
    elif name == "miller_loop_one":
        for f, P, Q in degenerate_pairs(curve, seed):
            out += [(f, [p], list(q)) for p, q in zip(P, Q)]
    else:
        raise KeyError(name)
    return out


def degenerate_pairs(curve: str, seed: int):
    """(family, P, Q) lists of pairs, none at infinity, on which the Miller loop takes degenerate paths: small-order twist points
    (T reaches -Q or infinity partway), off-subgroup points, X.A1 = 0, and bls12-381's x = 0 points of order 3"""
    P, Q = random_pairs(curve, 4, seed)
    fams = [("random", P, Q)]
    ells = [10069] if curve == "bn254" else [13, 23]
    for ell in ells:
        fams.append(("order_%d" % ell, P[:2], small_order_g2(curve, ell, 2, seed + ell)))
    fams.append(("off_subgroup_g2", P[:2], off_subgroup_g2(2, seed + 1, curve)))
    fams.append(("x_in_fp", P[:2], g2_x_in_fp(curve, 2, seed + 2)))
    if curve == "bls12381":
        fams.append(("g1_order3", bls12381_g1_order3(), Q[:2]))
        fams.append(("off_subgroup_g1", off_subgroup_g1(curve, 2, seed + 3), Q[:2]))
        fams.append(("order3_x_order13", bls12381_g1_order3(), small_order_g2(curve, 13, 2, seed + 4)))
    return fams


def two_lines_e12(curve: str, x):
    """the five E2 of a product of two lines as an E12: C0 and C1.B0, C1.B1 (bn254) or C1.B1, C1.B2 (bls12-381)"""
    Z = (0, 0)
    if curve == "bn254":
        return ((x[0], x[1], x[2]), (x[3], x[4], Z))
    return ((x[0], x[1], x[2]), (Z, x[3], x[4]))


def tower_op_ref(curve: str, name: str, a, b):
    """the restatement's value of one op: a and b are lists of E2 (the op's operands in memory order), the result likewise"""
    T = PR.tower(curve)
    e6 = lambda v: tuple(v[:3])
    e12 = lambda v: from_components(v)
    Z = (0, 0)
    if name == "e6_mul":
        return list(T.e6_mul(e6(a), e6(b)))
    if name == "e6_inv":
        return list(T.e6_inv(e6(a)))
    if name == "e6_mul_by_01":
        return list(T.e6_mul(e6(a), (b[0], b[1], Z)))
    if name == "e6_mul_by_1":
        return list(T.e6_mul(e6(a), (Z, b[0], Z)))
    if name == "e6_mul_by_12":
        return list(T.e6_mul(e6(a), (Z, b[0], b[1])))
    one = {"mul": lambda x: T.mul(x, e12(b)), "sqr": T.sqr, "inv": T.inv, "conj": T.conj, "frob1": lambda x: T.frob(x, 1),
           "frob2": lambda x: T.frob(x, 2), "frob3": lambda x: T.frob(x, 3), "cyclo_sqr": T.cyclo_sqr,
           "cyclo_sqr_compressed": T.cyclo_sqr_compressed, "decompress_karabina": T.decompress_karabina, "expt": T.expt,
           "expt_half": T.expt_half, "final_exp": T.final_exp, "mul_by_line": lambda x: T.mul_line(x, tuple(b)),
           "mul_by_two_lines": lambda x: T.mul(x, two_lines_e12(curve, b))}
    if name in one:
        return components(one[name](e12(a)))
    if name == "line_by_line":
        p = T.mul(T.sparse(tuple(a)), T.sparse(tuple(b)))
        c = components(p)
        keep = (0, 1, 2, 3, 4) if curve == "bn254" else (0, 1, 2, 4, 5)
        assert all(c[j] == Z for j in range(6) if j not in keep)
        return [c[j] for j in keep]
    if name == "double_step":
        p, line = T.double_step(tuple(a))
        return list(p) + list(line)
    if name == "add_mixed_step":
        p, line = T.add_mixed_step(tuple(a), tuple(b))
        return list(p) + list(line)
    if name == "line_compute":
        return list(a) + list(T.line_compute(tuple(a), tuple(b)))
    if name == "miller_loop_one":
        return components(T.miller_loop([a[0]], [tuple(b)]))
    raise KeyError(name)


def encode_e2s(curve: str, rows, width: int) -> np.ndarray:
    """rows of `width` E2 values as Montgomery limbs, one row per element (at least one column, for an unused operand)"""
    T = PR.tower(curve)
    fp, L = T.fp, T.fp.limbs
    out = np.zeros((len(rows), max(width, 1) * 2 * L), dtype=np.uint64)
    for i, row in enumerate(rows):
        assert len(row) == width
        out[i, :width * 2 * L] = [w for e in row for c in e for w in fp.to_limbs(fp.to_mont(c % T.q))]
    return out


def decode_e2s(curve: str, arr, width: int):
    T = PR.tower(curve)
    fp, L = T.fp, T.fp.limbs
    arr = np.asarray(arr, dtype=np.uint64).reshape(-1, width * 2 * L)
    vals = lambda r: [fp.from_mont(O.Field.from_limbs([int(w) for w in r[L * j: L * (j + 1)]])) for j in range(2 * width)]
    return [[tuple(v[2 * k: 2 * k + 2]) for k in range(width)] for v in map(vals, arr)]
