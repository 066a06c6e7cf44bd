"""Pairings on the H100 (pairing.cu / pairing_kernels.cuh) through the C ABI and gnark-crypto_b200/pairing.py, compared limb for
limb with the big-int restatement (tests/pairing_ref.py): random and special pairs, host and device inputs on a non-default
stream, products and checks over 2^16 distinct pairs, 2^20 distinct bn254 pairs (several chunks), and the argument errors."""
import ctypes
import random

import numpy as np
import pytest

from tests import pairing_cases as PC
from tests import pairing_ref as PR

pytestmark = pytest.mark.gpu

CURVES = ["bn254", "bls12381"]


def _pkg():
    import gnark_crypto_b200  # noqa: F401
    import importlib

    return importlib.import_module("gnark-crypto_b200.pairing")


def _dev(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a).view(np.int64).reshape(-1).copy()).cuda()


def _host(t):
    return t.cpu().numpy().view(np.uint64).reshape(1, -1)


@pytest.mark.parametrize("curve", CURVES)
def test_miller_loop_limb_exact_random(curve):
    pr = _pkg()
    T = PR.tower(curve)
    P, Q = PC.random_pairs(curve, 300, seed=21)
    pa, qa = PC.encode_pairs(curve, P, Q)
    got = pr.MillerLoop(curve, pa, qa).reshape(1, -1)
    assert np.array_equal(got, T.encode([T.miller_loop(P, Q)]))
    # one pair: MillerLoop and Pair against the restatement, host and device inputs
    for k in range(3):
        want_ml = T.miller_loop([P[k]], [Q[k]])
        assert np.array_equal(pr.MillerLoop(curve, pa[k:k + 1], qa[k:k + 1]).reshape(1, -1), T.encode([want_ml]))
        assert np.array_equal(_host(pr.Pair(curve, _dev(pa[k:k + 1]), _dev(qa[k:k + 1]))), T.encode([T.final_exp(want_ml)]))


@pytest.mark.parametrize("curve", CURVES)
def test_special_pairs(curve):
    import torch

    pr = _pkg()
    T = PR.tower(curve)
    P, Q = PC.random_pairs(curve, 4, seed=22)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for i in range(4):
            for side in (0, 1):
                P2, Q2 = list(P), list(Q)
                if side == 0:
                    P2[i] = T.G1.aff_inf()
                else:
                    Q2[i] = T.G2.aff_inf()
                pa, qa = PC.encode_pairs(curve, P2, Q2)
                want = T.miller_loop(P2, Q2)
                assert np.array_equal(_host(pr.MillerLoop(curve, _dev(pa), _dev(qa))), T.encode([want]))
        pa, qa = PC.encode_pairs(curve, [T.G1.aff_inf()] * 3, Q[:3])
        one = T.encode([T.one()])
        assert np.array_equal(pr.MillerLoop(curve, pa, qa).reshape(1, -1), one)
        assert np.array_equal(pr.Pair(curve, pa, qa).reshape(1, -1), one)
        dP, dQ = [P[0]] * 3 + [P[1]], [Q[0]] * 3 + [Q[1]]
        pa, qa = PC.encode_pairs(curve, dP, dQ)
        assert np.array_equal(pr.MillerLoop(curve, pa, qa).reshape(1, -1), T.encode([T.miller_loop(dP, dQ)]))
    s.synchronize()


def test_bn254_off_subgroup_g2():
    pr = _pkg()
    T = PR.tower("bn254")
    Q = PC.off_subgroup_g2(3, seed=23)
    P, _ = PC.random_pairs("bn254", 3, seed=24)
    pa, qa = PC.encode_pairs("bn254", P, Q)
    ml = T.miller_loop(P, Q)
    assert np.array_equal(pr.MillerLoop("bn254", pa, qa).reshape(1, -1), T.encode([ml]))
    assert np.array_equal(pr.Pair("bn254", pa, qa).reshape(1, -1), T.encode([T.final_exp(ml)]))


@pytest.mark.parametrize("curve", CURVES)
def test_final_exponentiation(curve):
    pr = _pkg()
    T = PR.tower(curve)
    rng = random.Random(25)
    cases = [[T.one()], [T.unflat([5] + [0] * 11)], [T.zero()], [T.unflat([rng.randrange(T.q) for _ in range(12)]) for _ in range(3)]]
    for zs in cases:
        enc = T.encode(zs)
        want = T.encode([T.final_exp(*zs)])
        assert np.array_equal(pr.FinalExponentiation(curve, *[enc[i] for i in range(len(zs))]).reshape(1, -1), want)
        assert np.array_equal(_host(pr.FinalExponentiation(curve, *[_dev(enc[i]) for i in range(len(zs))])), want)


def _distinct(curve, n, seed):
    """n distinct pairs ([a_i]G1, [b_i]G2) from the batch scalar multiplication, and c = sum a_i b_i mod r"""
    import gnark_crypto_b200 as pkg

    T = PR.tower(curve)
    rng = random.Random(seed)
    a = [rng.randrange(1, T.r) for _ in range(n)]
    b = [rng.randrange(1, T.r) for _ in range(n)]
    g1 = T.G1.encode_affine([T.G1.gen])[0]
    g2 = T.G2.encode_affine([T.G2.gen])[0]
    pa = pkg.BatchScalarMultiplication(T.G1.name, g1, T.G1.encode_scalars(a))
    qa = pkg.BatchScalarMultiplication(T.G2.name, g2, T.G2.encode_scalars(b))
    return a, b, pa, qa, sum(x * y for x, y in zip(a, b)) % T.r


def _check_distinct(curve, n, seed):
    """Pair over n distinct pairs equals Pair(G1, [sum a_i b_i]G2), whose value the restatement gives"""
    pr = _pkg()
    T = PR.tower(curve)
    _, _, pa, qa, c = _distinct(curve, n, seed)
    got = _host(pr.Pair(curve, _dev(pa), _dev(qa)))
    q1 = T.G2.scalar_mul(T.G2.gen, c)
    p1, q1a = PC.encode_pairs(curve, [T.G1.gen], [q1])
    assert np.array_equal(pr.Pair(curve, p1, q1a).reshape(1, -1), T.encode([T.pair([T.G1.gen], [q1])]))
    assert np.array_equal(got, T.encode([T.pair([T.G1.gen], [q1])]))


@pytest.mark.parametrize("curve", CURVES)
def test_pair_2_16_distinct(curve):
    _check_distinct(curve, 1 << 16, seed=26)


@pytest.mark.parametrize("curve", CURVES)
def test_pairing_check_2_16_distinct(curve):
    """(P_i, Q_i) and (-P_i, Q_i) for 2^15 distinct pairs cancel; one perturbed pair breaks the check"""
    import gnark_crypto_b200 as pkg

    pr = _pkg()
    T = PR.tower(curve)
    half = 1 << 15
    a, _, pa, qa, _ = _distinct(curve, half, seed=27)
    g1 = T.G1.encode_affine([T.G1.gen])[0]
    neg = pkg.BatchScalarMultiplication(T.G1.name, g1, T.G1.encode_scalars([T.r - x for x in a]))
    P = np.concatenate([pa, neg])
    Q = np.concatenate([qa, qa])
    assert pr.PairingCheck(curve, _dev(P), _dev(Q))
    P[12345] = pkg.BatchScalarMultiplication(T.G1.name, g1, T.G1.encode_scalars([a[12345] + 1]))[0]
    assert not pr.PairingCheck(curve, _dev(P), _dev(Q))


def test_bn254_2_20_distinct_chunked():
    """2^20 distinct pairs: sixteen chunks of the Miller loop, each reading its own pairs"""
    _check_distinct("bn254", 1 << 20, seed=28)


def test_wrong_lengths():
    pr = _pkg()
    P, Q = PC.random_pairs("bn254", 2, seed=29)
    pa, qa = PC.encode_pairs("bn254", P, Q)
    with pytest.raises(ValueError):
        pr.Pair("bn254", _dev(pa)[:-1], _dev(qa))
    with pytest.raises(ValueError):
        pr.MillerLoop("bn254", pa, qa.reshape(-1)[:-3])


def test_errors():
    import gnark_crypto_b200  # noqa: F401
    import importlib

    pr = _pkg()
    nat = importlib.import_module("gnark-crypto_b200._native")
    L = nat.lib()
    P, Q = PC.random_pairs("bn254", 2, seed=27)
    pa, qa = PC.encode_pairs("bn254", P, Q)
    with pytest.raises(ValueError):
        pr.MillerLoop("bn254", pa[:0], qa[:0])
    with pytest.raises(ValueError):
        pr.Pair("bn254", pa, qa[:1])
    for c in ("bls12377", "bw6761", "bls24315"):
        with pytest.raises(ValueError):
            pr.Pair(c, pa, qa)
    out = np.zeros(72, dtype=np.uint64)
    vp = lambda a: ctypes.c_void_p(a.ctypes.data)
    assert L.gmsm_pair(0, vp(pa), vp(qa), 0, vp(out)) == 1                  # n = 0
    for cid in (1, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12):                        # not bn254 / bls12-381 G1 ids
        assert L.gmsm_pair(cid, vp(pa), vp(qa), 2, vp(out)) == 1
        assert L.gmsm_pairing_miller_loop(cid, vp(pa), vp(qa), 2, vp(out)) == 1
        assert L.gmsm_pairing_final_exp(cid, vp(out), 1, vp(out)) == 1
    assert L.gmsm_pair(0, None, vp(qa), 2, vp(out)) == 1
    assert L.gmsm_pairing_final_exp(0, vp(out), 0, vp(out)) == 1
