"""The pairing on the H100 at its edges: every tower test op (gmsm_test_tower_op, tower_testops.cuh) over every adversarial operand
family, 4096 elements per op so that warps take mixed branches, limb-exact against the big-int restatement (tests/pairing_ref.py)
and against the polynomial ring (tests/tower_poly_ref.py) where the identity holds; MillerLoop and Pair of degenerate pairs
(small-order and off-subgroup points, x = 0); chunk boundaries of the multi-pair loop; a caller workspace of exactly the stated
size; FinalExponentiation of subfield elements and of long products with zeros; bilinearity on the device."""
import ctypes
import random

import numpy as np
import pytest

from tests import pairing_cases as PC
from tests import pairing_ref as PR
from tests import tower_poly_ref as TP
from tests.test_gpu_pairing import _check_distinct, _dev, _distinct, _host, _pkg

pytestmark = pytest.mark.gpu

CURVES = ["bn254", "bls12381"]
CID = {"bn254": 0, "bls12381": 2}
N_OPS = 4096


def _lib():
    import gnark_crypto_b200  # noqa: F401
    import importlib

    return importlib.import_module("gnark-crypto_b200._native").lib()


def tower_op(curve, name, rows_a, rows_b):
    op, wa, wb, wo = PC.TOWER_OPS[name]
    T = PR.tower(curve)
    n = len(rows_a)
    a = PC.encode_e2s(curve, rows_a, wa)
    b = PC.encode_e2s(curve, rows_b if wb else [[]] * n, wb)
    out = np.zeros((n, wo * 2 * T.fp.limbs), dtype=np.uint64)
    vp = lambda x: ctypes.c_void_p(x.ctypes.data)
    assert _lib().gmsm_test_tower_op(CID[curve], op, vp(a), vp(b), vp(out), n) == 0
    return out


@pytest.mark.parametrize("curve", CURVES)
@pytest.mark.parametrize("name", sorted(PC.TOWER_OPS))
def test_tower_op_families(curve, name):
    """the distinct cases of every family, tiled in a shuffled order to 4096 elements, limb-exact against the restatement"""
    from tests.test_tower_stress_cpu import RING_OPS, model_check

    if curve == "bn254" and name == "expt_half":
        z = np.zeros(48, dtype=np.uint64)
        vp = ctypes.c_void_p(z.ctypes.data)
        assert _lib().gmsm_test_tower_op(0, PC.TOWER_OPS[name][0], vp, vp, vp, 1) == 1
        return
    cases = PC.tower_op_cases(curve, name, seed=100 + len(name))
    want = [PC.tower_op_ref(curve, name, a, b) for _, a, b in cases]
    rng = random.Random(len(name))
    idx = [i % len(cases) for i in range(N_OPS)]
    rng.shuffle(idx)
    got = tower_op(curve, name, [cases[i][1] for i in idx], [cases[i][2] for i in idx])
    wo = PC.TOWER_OPS[name][3]
    enc_want = PC.encode_e2s(curve, want, wo)
    for j, i in enumerate(idx):
        assert np.array_equal(got[j], enc_want[i]), (name, cases[i][0], j)
    if name in RING_OPS:
        dec = PC.decode_e2s(curve, got[:len(cases)], wo)
        pows = 0
        for j in range(min(len(cases), 64)):
            fam, a, b = cases[idx[j]]
            if model_check(curve, name, a, b, dec[j], pows < 2):
                pows += name in ("e6_inv", "inv", "conj", "frob1", "frob2", "frob3")


@pytest.mark.parametrize("curve", CURVES)
def test_cyclotomic_ops_vs_model(curve):
    """compressed squarings then decompression, Expt / ExptHalf and the final exponentiation on the device, against model powers"""
    T, M = PR.tower(curve), TP.poly_tower(curve)
    rng = random.Random(7)
    xs = [PC.cyclotomic(T, PC.random_e12(T, rng)) for _ in range(2)]
    rows = [PC.components(x) for x in xs]
    dec = lambda arr: [PC.from_components(r) for r in PC.decode_e2s(curve, arr, 6)]
    r = rows
    for _ in range(15):
        r = PC.decode_e2s(curve, tower_op(curve, "cyclo_sqr_compressed", r, None), 6)
    for g, x in zip(dec(tower_op(curve, "decompress_karabina", r, None)), xs):
        assert g == M.unembed(M.pow(M.embed(x), 1 << 15))
    for g, x in zip(dec(tower_op(curve, "expt", rows, None)), xs):
        assert g == M.unembed(M.gt_pow(M.embed(x), T.x0))
    if curve == "bls12381":
        for g, x in zip(dec(tower_op(curve, "expt_half", rows, None)), xs):
            assert g == M.unembed(M.gt_pow(M.embed(x), T.x0 // 2))


@pytest.mark.parametrize("curve", CURVES)
def test_degenerate_pairs(curve):
    """MillerLoop and Pair of every degenerate family, alone and mixed with random pairs"""
    pr = _pkg()
    T = PR.tower(curve)
    fams = PC.degenerate_pairs(curve, seed=71)
    for fam, P, Q in fams:
        pa, qa = PC.encode_pairs(curve, P, Q)
        ml = T.miller_loop(P, Q)
        assert np.array_equal(pr.MillerLoop(curve, pa, qa).reshape(1, -1), T.encode([ml])), fam
        assert np.array_equal(pr.Pair(curve, pa, qa).reshape(1, -1), T.encode([T.final_exp(ml)])), fam
    Pr, Qr = PC.random_pairs(curve, 3, seed=72)
    P = Pr + [p for _, Ps, _ in fams for p in Ps]
    Q = Qr + [q for _, _, Qs in fams for q in Qs]
    pa, qa = PC.encode_pairs(curve, P, Q)
    assert np.array_equal(pr.MillerLoop(curve, pa, qa).reshape(1, -1), T.encode([T.miller_loop(P, Q)]))
    # one point over a whole 64-thread block, and a bit more
    Ps, Qs = [P[-1]] * 65, [Q[-1]] * 65
    pa, qa = PC.encode_pairs(curve, Ps, Qs)
    assert np.array_equal(pr.MillerLoop(curve, pa, qa).reshape(1, -1), T.encode([T.gt_pow(T.miller_loop([P[-1]], [Q[-1]]), 65)]))


def _pair_with_infinities(curve, n, seed, inf_ranges):
    """Pair over n distinct pairs with the pairs in inf_ranges set to infinity equals Pair(G1, [sum a_i b_i]G2) over the rest"""
    pr = _pkg()
    T = PR.tower(curve)
    a, b, pa, qa, _ = _distinct(curve, n, seed)
    pa = np.array(pa)
    for lo, hi in inf_ranges:
        pa[lo:hi] = 0
    keep = np.ones(n, dtype=bool)
    for lo, hi in inf_ranges:
        keep[lo:hi] = False
    c = sum(x * y for x, y, k in zip(a, b, keep) if k) % T.r
    got = _host(pr.Pair(curve, _dev(pa), _dev(qa)))
    q1 = T.G2.scalar_mul(T.G2.gen, c)
    assert np.array_equal(got, T.encode([T.pair([T.G1.gen], [q1])]))


@pytest.mark.parametrize("curve", CURVES)
def test_chunk_edges(curve):
    """2^16 + 1 pairs (a last chunk of one pair, no reduction), with infinities at the chunk edges"""
    C = 1 << 16
    _pair_with_infinities(curve, C + 1, 81, [(0, 1), (C - 1, C)])


def test_bn254_chunk_shapes():
    C = 1 << 16
    _check_distinct("bn254", 2 * C - 1, seed=82)
    _pair_with_infinities("bn254", 3 * C, 83, [(C, 2 * C)])        # the middle chunk all infinity
    _pair_with_infinities("bn254", 3 * C, 84, [(2 * C, 3 * C)])    # the last chunk all infinity


def test_bls12381_several_chunks():
    _check_distinct("bls12381", (1 << 17) + 3, seed=85)


@pytest.mark.parametrize("curve", CURVES)
def test_pairing_check_partners_a_chunk_apart(curve):
    """(P_i, Q_i) and (-P_i, Q_i) with the partners 2^16 apart, in different chunks; one perturbation breaks the check"""
    import gnark_crypto_b200 as pkg

    pr = _pkg()
    T = PR.tower(curve)
    half = 1 << 16
    a, _, pa, qa, _ = _distinct(curve, half, seed=86)
    g1 = T.G1.encode_affine([T.G1.gen])[0]
    neg = pkg.BatchScalarMultiplication(T.G1.name, g1, T.G1.encode_scalars([T.r - x for x in a]))
    P = np.concatenate([pa, neg])
    Q = np.concatenate([qa, qa])
    assert pr.PairingCheck(curve, _dev(P), _dev(Q))
    P[half + 777] = pkg.BatchScalarMultiplication(T.G1.name, g1, T.G1.encode_scalars([T.r - a[777] + 1]))[0]
    assert not pr.PairingCheck(curve, _dev(P), _dev(Q))


@pytest.mark.parametrize("curve", CURVES)
def test_workspace_exact_size(curve):
    """a workspace of exactly gmsm_pairing_workspace_bytes(n) filled with 0xFF, then a 4 KiB guard: the result is the
    restatement's and the guard intact; two calls on two streams with their own workspaces give their own results"""
    import torch

    L = _lib()
    T = PR.tower(curve)
    gb = 12 * 2 * T.fp.limbs * 4
    C = 1 << 16
    P, Q = PC.random_pairs(curve, 3, seed=87)
    for n in (1, 2, C, C + 1):
        Ps = [P[i % 3] for i in range(n)]
        Qs = [Q[i % 3] for i in range(n)]
        pa, qa = PC.encode_pairs(curve, Ps, Qs)
        k = [(n + 2 - i) // 3 for i in range(3)]
        want = T.mul(T.mul(T.gt_pow(T.miller_loop([P[0]], [Q[0]]), k[0]), T.gt_pow(T.miller_loop([P[1]], [Q[1]]), k[1])),
                     T.gt_pow(T.miller_loop([P[2]], [Q[2]]), k[2]))
        wsb = L.gmsm_pairing_workspace_bytes(CID[curve], n)
        assert wsb % 8 == 0
        ws = torch.full(((wsb + 4096) // 8,), -1, dtype=torch.int64, device="cuda")
        out = torch.zeros(gb // 8, dtype=torch.int64, device="cuda")
        dP, dQ = _dev(pa), _dev(qa)
        assert L.gmsm_pairing_miller_loop_device(CID[curve], dP.data_ptr(), dQ.data_ptr(), n, out.data_ptr(), ws.data_ptr(), None) == 0
        torch.cuda.synchronize()
        assert np.array_equal(_host(out), T.encode([want])), n
        assert bool((ws[wsb // 8:] == -1).all()), n
    # two streams, two workspaces
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    pairs = [PC.random_pairs(curve, 5, seed=88), PC.random_pairs(curve, 7, seed=89)]
    outs = []
    for (Ps, Qs), s in zip(pairs, (s1, s2)):
        pa, qa = PC.encode_pairs(curve, Ps, Qs)
        wsb = L.gmsm_pairing_workspace_bytes(CID[curve], len(Ps))
        with torch.cuda.stream(s):
            ws = torch.full(((wsb + 4096) // 8,), -1, dtype=torch.int64, device="cuda")
            out = torch.zeros(gb // 8, dtype=torch.int64, device="cuda")
            dP, dQ = _dev(pa), _dev(qa)
        s.synchronize()
        assert L.gmsm_pairing_miller_loop_device(CID[curve], dP.data_ptr(), dQ.data_ptr(), len(Ps), out.data_ptr(), ws.data_ptr(),
                                                 ctypes.c_void_p(s.cuda_stream)) == 0
        outs.append((out, ws, wsb, dP, dQ))
    torch.cuda.synchronize()
    for (Ps, Qs), (out, ws, wsb, _, _) in zip(pairs, outs):
        assert np.array_equal(_host(out), T.encode([T.miller_loop(Ps, Qs)]))
        assert bool((ws[wsb // 8:] == -1).all())


@pytest.mark.parametrize("curve", CURVES)
def test_final_exponentiation_edges(curve):
    """the easy-part shortcut on subfield inputs (an Fp2 value, an Fp6 value, c w), products of k elements with a zero at the
    first, middle and last position, and a long product, against the restatement; random inputs against the model's pow"""
    pr = _pkg()
    T, M = PR.tower(curve), TP.poly_tower(curve)
    rng = random.Random(91)
    Z = (0, 0)
    sub = [PC.from_components([PC.random_e2(T, rng)] + [Z] * 5), PC.from_components([PC.random_e2(T, rng) for _ in range(3)] + [Z] * 3),
           PC.from_components([Z] * 3 + [PC.random_e2(T, rng)] + [Z] * 2)]
    for x in sub:
        assert T.final_exp(x) == T.one()
        assert np.array_equal(pr.FinalExponentiation(curve, T.encode([x])[0]).reshape(1, -1), T.encode([T.one()]))
    for k in (2, 3, 64, 1000):
        zs = [PC.random_e12(T, rng) for _ in range(k)]
        want = T.final_exp(*zs)
        enc = T.encode(zs)
        assert np.array_equal(pr.FinalExponentiation(curve, *[enc[i] for i in range(k)]).reshape(1, -1), T.encode([want])), k
        if k <= 3:
            prod = M.one()
            for z in zs:
                prod = M.mul(prod, M.embed(z))
            assert M.unembed(M.pow(prod, M.final_exp_exponent())) == want
        for pos in (0, k // 2, k - 1):
            zz = list(zs)
            zz[pos] = T.zero()
            enc = T.encode(zz)
            assert np.array_equal(pr.FinalExponentiation(curve, *[enc[i] for i in range(k)]).reshape(1, -1),
                                  T.encode([T.final_exp(*zz)])), (k, pos)


@pytest.mark.parametrize("curve", CURVES)
def test_bilinearity_on_device(curve):
    """Pair([a]P, [b]Q) = Pair(P, Q)^(ab) for a, b in {1, 2, r - 1, random}, the power taken in the polynomial model"""
    pr = _pkg()
    T, M = PR.tower(curve), TP.poly_tower(curve)
    rng = random.Random(92)
    P, Q = PC.random_pairs(curve, 1, seed=93)
    pa, qa = PC.encode_pairs(curve, P, Q)
    base = M.embed(T.decode(pr.Pair(curve, pa, qa).reshape(1, -1))[0])
    for a in (1, 2, T.r - 1, rng.randrange(T.r)):
        for b in (1, 2, T.r - 1, rng.randrange(T.r)):
            pa, qa = PC.encode_pairs(curve, [T.G1.scalar_mul(P[0], a)], [T.G2.scalar_mul(Q[0], b)])
            got = T.decode(pr.Pair(curve, pa, qa).reshape(1, -1))[0]
            assert M.embed(got) == M.pow(base, a * b % T.r), (a, b)
