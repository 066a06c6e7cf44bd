"""The big-int pairing restatement (tests/pairing_ref.py) pinned by checks that do not depend on it: the final exponentiation
equals a plain pow by its exponent, bilinearity, e(P, Q)^r = 1 with e(G1, G2) != 1, and e(-P, Q) e(P, Q) = 1.  CPU only."""
import random

import pytest

from tests import pairing_ref as PR

CURVES = ["bn254", "bls12381"]


def _exponent(T):
    # the hard part's multiple: bn254 2 x0 (6 x0^2 + 3 x0 + 1), bls12-381 3 (the chains' comments, pinned here)
    s = 2 * T.x0 * (6 * T.x0 ** 2 + 3 * T.x0 + 1) if T.curve == "bn254" else 3
    return s * (T.q ** 12 - 1) // T.r


def _random_e12(T, rng):
    return T.unflat([rng.randrange(T.q) for _ in range(12)])


@pytest.mark.parametrize("curve", CURVES)
def test_final_exp_is_plain_pow(curve):
    T = PR.tower(curve)
    rng = random.Random(1)
    e = _exponent(T)
    for _ in range(2):
        f = _random_e12(T, rng)
        assert T.final_exp(f) == T.gt_pow(f, e)


@pytest.mark.parametrize("curve", CURVES)
def test_bilinear_order_nondegenerate(curve):
    T = PR.tower(curve)
    rng = random.Random(2)
    g = T.pair([T.G1.gen], [T.G2.gen])
    assert g != T.one()
    assert T.gt_pow(g, T.r) == T.one()
    a, b = rng.randrange(1, T.r), rng.randrange(1, T.r)
    assert T.pair([T.G1.scalar_mul(T.G1.gen, a)], [T.G2.scalar_mul(T.G2.gen, b)]) == T.gt_pow(g, a * b % T.r)


@pytest.mark.parametrize("curve", CURVES)
def test_negation_cancels(curve):
    T = PR.tower(curve)
    P = T.G1.scalar_mul(T.G1.gen, 12345)
    Q = T.G2.scalar_mul(T.G2.gen, 678)
    assert T.pairing_check([P, T.G1.aff_neg(P)], [Q, Q])
    assert not T.pairing_check([P, P], [Q, Q])


@pytest.mark.parametrize("curve", CURVES)
def test_special_inputs(curve):
    T = PR.tower(curve)
    inf1, inf2 = T.G1.aff_inf(), T.G2.aff_inf()
    assert T.miller_loop([inf1, T.G1.gen], [T.G2.gen, inf2]) == T.one()
    assert T.final_exp(T.one()) == T.one()
    fp_elem = T.unflat([7] + [0] * 11)          # an Fp element: the easy part maps it to 1
    assert T.final_exp(fp_elem) == T.one()
    with pytest.raises(ValueError):
        T.miller_loop([], [])
    with pytest.raises(ValueError):
        T.miller_loop([T.G1.gen], [])
