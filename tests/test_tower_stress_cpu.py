"""The pairing towers on adversarial operands, on the CPU: every tower test op (tower_testops.cuh, k_tower_op) through the kernel
emulation, limb for limb against the big-int restatement (tests/pairing_ref.py) over every operand family of tests/pairing_cases.py,
and against the plain polynomial ring of tests/tower_poly_ref.py wherever the identity holds; DecompressKarabina in each of its
branches, with the restatement pinned by the formulas of e12.go's DecompressKarabina worked by hand; and the Miller loop of
degenerate pairs (small-order and off-subgroup points, x = 0) at small forced chunks.  CPU only."""
import ctypes
import random

import numpy as np
import pytest

from tests import pairing_cases as PC
from tests import pairing_ref as PR
from tests import tower_poly_ref as TP
from tests.test_emu_pairing_cpu import IDS, _lib, emu_final_exp, emu_miller

CURVES = sorted(IDS)
# ops whose result is the ring operation on every input (the rest hold on the cyclotomic subgroup only)
RING_OPS = ("e6_mul", "e6_inv", "e6_mul_by_01", "e6_mul_by_1", "e6_mul_by_12", "mul", "sqr", "inv", "conj", "frob1", "frob2", "frob3",
            "mul_by_line", "line_by_line", "mul_by_two_lines")
POW_SAMPLE = 4   # elements per op checked by a model pow (inv, conj, frob, final_exp): each costs up to a second


def emu_tower_op(curve, name, rows_a, rows_b, threads=64):
    op, wa, wb, wo = PC.TOWER_OPS[name]
    T = PR.tower(curve)
    n = len(rows_a)
    a = PC.encode_e2s(curve, rows_a, wa)
    b = PC.encode_e2s(curve, rows_b if wb else [[]] * n, wb)
    out = np.zeros((n, wo * 2 * T.fp.limbs), dtype=np.uint64)
    rc = getattr(_lib(), "emu_tower_op_%d" % IDS[curve])(ctypes.c_int(op), ctypes.c_void_p(a.ctypes.data), ctypes.c_void_p(b.ctypes.data),
                                                        ctypes.c_void_p(out.ctypes.data), ctypes.c_uint64(n), ctypes.c_uint(threads))
    assert rc == 0
    return PC.decode_e2s(curve, out, wo)


def model_check(curve, name, a, b, got, pow_ok):
    """got (a list of E2) against the polynomial ring: True when checked, False when the op has no ring identity for this input"""
    M = TP.poly_tower(curve)
    emb = lambda x: M.embed(x)
    e6 = lambda v: PC.from_components(list(v) + [(0, 0)] * 3)
    Z = (0, 0)
    want = None
    if name == "e6_mul":
        want, g = M.mul(emb(e6(a)), emb(e6(b))), e6(got)
    elif name == "e6_inv" and pow_ok:
        want, g = M.inv(emb(e6(a))), e6(got)
    elif name in ("e6_mul_by_01", "e6_mul_by_1", "e6_mul_by_12"):
        c = [Z, b[0], Z] if name == "e6_mul_by_1" else [b[0], b[1], Z] if name == "e6_mul_by_01" else [Z, b[0], b[1]]
        want, g = M.mul(emb(e6(a)), emb(e6(c))), e6(got)
    elif name == "mul":
        want, g = M.mul(emb(PC.from_components(a)), emb(PC.from_components(b))), PC.from_components(got)
    elif name == "sqr":
        x = emb(PC.from_components(a))
        want, g = M.mul(x, x), PC.from_components(got)
    elif name in ("inv", "conj", "frob1", "frob2", "frob3") and pow_ok:
        x = emb(PC.from_components(a))
        want = {"inv": M.inv, "conj": M.conj}.get(name, lambda y: M.frob(y, int(name[-1])))(x)
        g = PC.from_components(got)
    elif name == "mul_by_line":
        want, g = M.mul(emb(PC.from_components(a)), emb(PR.tower(curve).sparse(tuple(b)))), PC.from_components(got)
    elif name == "line_by_line":
        T = PR.tower(curve)
        want, g = M.mul(emb(T.sparse(tuple(a))), emb(T.sparse(tuple(b)))), PC.two_lines_e12(curve, got)
    elif name == "mul_by_two_lines":
        want, g = M.mul(emb(PC.from_components(a)), emb(PC.two_lines_e12(curve, b))), PC.from_components(got)
    if want is None:
        return False
    assert M.unembed(want) == g, name
    return True


@pytest.mark.parametrize("curve", CURVES)
@pytest.mark.parametrize("name", sorted(PC.TOWER_OPS))
def test_tower_op_families(curve, name):
    """every operand family through k_tower_op, limb-exact against the restatement; the ring identity on the families where it
    holds; every family of the op's case list reached"""
    if curve == "bn254" and name == "expt_half":
        T = PR.tower(curve)
        z = np.zeros((1, 12 * T.fp.limbs), dtype=np.uint64)
        assert getattr(_lib(), "emu_tower_op_0")(ctypes.c_int(PC.TOWER_OPS[name][0]), ctypes.c_void_p(z.ctypes.data),
                                                 ctypes.c_void_p(z.ctypes.data), ctypes.c_void_p(z.ctypes.data), ctypes.c_uint64(1),
                                                 ctypes.c_uint(1)) == 1
        return
    cases = PC.tower_op_cases(curve, name, seed=len(name))
    if name in ("expt", "expt_half", "final_exp", "miller_loop_one"):   # the restatement's cost: a few per family
        seen = {}
        cases = [c for c in cases if seen.setdefault(c[0], []).append(1) or len(seen[c[0]]) <= 3]
    got = emu_tower_op(curve, name, [a for _, a, _ in cases], [b for _, _, b in cases], threads=7)
    hits = {}
    for (fam, a, b), g in zip(cases, got):
        assert g == PC.tower_op_ref(curve, name, a, b), (name, fam, a, b)
        hits[fam] = hits.get(fam, 0) + 1
    assert len(hits) >= 3 and min(hits.values()) >= 1, hits
    if name in RING_OPS:
        checked, pows = 0, 0
        for (fam, a, b), g in zip(cases, got):
            pow_ok = pows < POW_SAMPLE and (fam != "single" or pows == 0)
            if model_check(curve, name, a, b, g, pow_ok):
                checked += 1
                pows += name in ("e6_inv", "inv", "conj", "frob1", "frob2", "frob3")
        assert checked >= min(len(cases), POW_SAMPLE)


@pytest.mark.parametrize("curve", CURVES)
def test_cyclotomic_ops_vs_model(curve):
    """on cyclotomic elements: CyclotomicSquare is a square, k compressed squarings then DecompressKarabina are x^(2^k), Expt and
    ExptHalf are powers by x0 and x0 / 2, and FinalExponentiation is the power by s (q^12 - 1) / r"""
    T, M = PR.tower(curve), TP.poly_tower(curve)
    rng = random.Random(41)
    xs = [PC.cyclotomic(T, PC.random_e12(T, rng)) for _ in range(3)]
    rows = [PC.components(x) for x in xs]
    emb = [M.embed(x) for x in xs]
    for g, e in zip(emu_tower_op(curve, "cyclo_sqr", rows, None), emb):
        assert PC.from_components(g) == M.unembed(M.mul(e, e))
    for k in (1, 2, 15):
        r = rows
        for _ in range(k):
            r = emu_tower_op(curve, "cyclo_sqr_compressed", r, None)
        for g, e in zip(emu_tower_op(curve, "decompress_karabina", r, None), emb):
            assert PC.from_components(g) == M.unembed(M.pow(e, 1 << k)), k
    for g, e in zip(emu_tower_op(curve, "expt", rows, None), emb):
        assert PC.from_components(g) == M.unembed(M.gt_pow(e, T.x0))
    if curve == "bls12381":
        for g, e in zip(emu_tower_op(curve, "expt_half", rows, None), emb):
            assert PC.from_components(g) == M.unembed(M.gt_pow(e, T.x0 // 2))
    rnd = [PC.random_e12(T, rng) for _ in range(2)]
    for x in xs[:1] + rnd:
        g = emu_tower_op(curve, "final_exp", [PC.components(x)], None)[0]
        assert PC.from_components(g) == M.unembed(M.pow(M.embed(x), M.final_exp_exponent()))


@pytest.mark.parametrize("curve", CURVES)
def test_poly_model_is_the_tower(curve):
    """the model itself: w^12 reduces to 2 xi0 w^6 - (xi0^2 + 1), embedding is a ring homomorphism, and the model agrees with
    the restatement on random inputs"""
    T, M = PR.tower(curve), TP.poly_tower(curve)
    w = (0, 1) + (0,) * 10
    xi0 = T.xi[0]
    assert M.pow(w, 12) == ((-(xi0 * xi0 + 1)) % T.q,) + (0,) * 5 + (2 * xi0,) + (0,) * 5
    assert M.embed(((T.xi, (0, 0), (0, 0)), ((0, 0),) * 3)) == M.pow(w, 6)   # v^3 = xi = w^6
    rng = random.Random(42)
    for _ in range(4):
        a, b = PC.random_e12(T, rng), PC.random_e12(T, rng)
        assert M.unembed(M.embed(a)) == a
        assert M.embed((T.e6_add(a[0], b[0]), T.e6_add(a[1], b[1]))) == tuple(
            (x + y) % T.q for x, y in zip(M.embed(a), M.embed(b)))
        assert M.unembed(M.mul(M.embed(a), M.embed(b))) == T.mul(a, b)
    a = PC.random_e12(T, rng)
    assert M.unembed(M.inv(M.embed(a))) == T.inv(a)
    assert M.unembed(M.frob(M.embed(a), 1)) == T.frob(a, 1)
    assert M.inv(M.embed(T.zero())) == M.embed(T.zero())


def _karabina_by_hand(T, x):
    """DecompressKarabina from its stated formulas (e12.go), with g1 = C0.B1, g2 = C0.B2, g3 = C1.B0, g5 = C1.B2 and E = xi:
    when C1.B2 = 0: g4 = 2 g1 g5 / g2, or one when also C0.B2 = 0; otherwise g4 = (E g5^2 + 3 g1^2 - 2 g2) / (4 g3), an inverse of
    zero being zero; then g0 = E (2 g4^2 + g3 g5 - 3 g2 g1) + 1.  Fp2 arithmetic written out over u^2 = -1."""
    q = T.q
    mul = lambda a, b: ((a[0] * b[0] - a[1] * b[1]) % q, (a[0] * b[1] + a[1] * b[0]) % q)
    lin = lambda *terms: (sum(k * t[0] for k, t in terms) % q, sum(k * t[1] for k, t in terms) % q)
    inv = lambda a: (lambda n: (a[0] * n % q, -a[1] * n % q))(pow((a[0] ** 2 + a[1] ** 2) % q, q - 2, q))
    (g0_in, g1, g2), (g3, g4_in, g5) = x
    if g5 == (0, 0):
        if g2 == (0, 0):
            return T.one()
        g4 = mul(lin((2, mul(g1, g5))), inv(g2))
    else:
        g4 = mul(lin((1, mul(T.xi, mul(g5, g5))), (3, mul(g1, g1)), (-2, g2)), inv(lin((4, g3))))
    g0 = lin((1, mul(T.xi, lin((2, mul(g4, g4)), (1, mul(g3, g5)), (-3, mul(g2, g1))))), (1, (1, 0)))
    return ((g0, g1, g2), (g3, g4, g5))


@pytest.mark.parametrize("curve", CURVES)
def test_karabina_branches(curve):
    """every branch of DecompressKarabina reached, counted per family: the kernel limb-exact against the restatement, the
    restatement equal to the formulas worked by hand, and a hand-built input per branch with small components"""
    T = PR.tower(curve)
    cases = PC.karabina_cases(curve, seed=5)
    Z = (0, 0)
    hand = {"g5zero": [(3, 1), (5, 0), (7, 2), (11, 0), (13, 1), Z], "g5g2zero": [(3, 1), (5, 0), Z, (11, 0), (13, 1), Z],
            "g3zero": [(3, 1), (5, 0), (7, 2), Z, (13, 1), (17, 4)], "generic": [(3, 1), (5, 0), (7, 2), (11, 0), (13, 1), (17, 4)]}
    for f, c in hand.items():
        cases[f].append(PC.from_components(c))
    flat = [(f, x) for f in sorted(cases) for x in cases[f]]
    got = emu_tower_op(curve, "decompress_karabina", [PC.components(x) for _, x in flat], None, threads=3)
    counts = {}
    for (f, x), g in zip(flat, got):
        assert PC.karabina_branch(x) == f
        want = T.decompress_karabina(x)
        assert want == _karabina_by_hand(T, x), f
        assert PC.from_components(g) == want, f
        counts[f] = counts.get(f, 0) + 1
    assert counts == {"g5zero": 5, "g5g2zero": 5, "g3zero": 5, "generic": 5}
    # the branch that returns one is reached because the inputs keep C0.B1 and C1.B0 non-zero: without it C1.B1 = 0 and
    # C0.B0 = 1 but C0.B1, C1.B0 would stay
    assert all(PC.from_components(g) == T.one() for (f, _), g in zip(flat, got) if f == "g5g2zero")
    assert all(x[0][1] != Z and x[1][0] != Z for f, x in flat if f == "g5g2zero")


@pytest.mark.parametrize("curve", CURVES)
def test_emu_degenerate_pairs(curve):
    """the Miller loop of every degenerate family, alone and mixed with random pairs, at forced small chunks, against the
    restatement; then the final exponentiation of each"""
    T = PR.tower(curve)
    for fam, P, Q in PC.degenerate_pairs(curve, seed=61):
        pa, qa = PC.encode_pairs(curve, P, Q)
        want = T.miller_loop(P, Q)
        for chunk, threads in ((1, 1), (2, 2), (1 << 16, 64)):
            assert np.array_equal(emu_miller(curve, pa, qa, chunk, threads, 3), T.encode([want])), (fam, chunk)
        assert np.array_equal(emu_final_exp(curve, T.encode([want])), T.encode([T.final_exp(want)])), fam
    Pr, Qr = PC.random_pairs(curve, 3, seed=62)
    mixes = PC.degenerate_pairs(curve, seed=63)
    P = Pr + [p for _, Ps, _ in mixes for p in Ps[:1]]
    Q = Qr + [q for _, _, Qs in mixes for q in Qs[:1]]
    pa, qa = PC.encode_pairs(curve, P, Q)
    assert np.array_equal(emu_miller(curve, pa, qa, 3, 2, 5), T.encode([T.miller_loop(P, Q)]))


@pytest.mark.parametrize("curve", CURVES)
def test_emu_cancelling_and_repeated_pairs(curve):
    """(P, Q) with (P, -Q) in one chunk and in different chunks: the product's final exponentiation is one; one point repeated
    over a whole block of 64 threads"""
    T = PR.tower(curve)
    P, Q = PC.random_pairs(curve, 2, seed=64)
    negQ = [T.G2.aff_neg(q) for q in Q]
    Ps = [P[0], P[1], P[0], P[1]]
    Qs = [Q[0], Q[1], negQ[0], negQ[1]]
    pa, qa = PC.encode_pairs(curve, Ps, Qs)
    want = T.miller_loop(Ps, Qs)
    assert T.final_exp(want) == T.one()
    for chunk in (4, 2, 1):   # the partners in one chunk, then in different chunks
        got = emu_miller(curve, pa, qa, chunk, 2, 1)
        assert np.array_equal(got, T.encode([want])), chunk
        assert np.array_equal(emu_final_exp(curve, got), T.encode([T.one()]))
    Ps, Qs = [P[0]] * 65, [Q[0]] * 65
    pa, qa = PC.encode_pairs(curve, Ps, Qs)
    want = T.gt_pow(T.miller_loop([P[0]], [Q[0]]), 65)
    assert want == T.miller_loop(Ps, Qs)
    assert np.array_equal(emu_miller(curve, pa, qa, 1 << 16, 64, 0), T.encode([want]))
