"""Pins the oracle's Fr FFT restatement for the scalar fields of bls24-315, bls24-317, bw6-633 and bw6-761
(ecc/*/fr/generator.go:23-24, fr/fft/domain.go:59): each stored root of unity is GeneratorFullMultiplicativeGroup^((r - 1)
>> maxOrderRoot) and has order exactly 2^maxOrderRoot; then the properties test_oracle_fft.py checks for the first three
fields (O(n^2) definition, DIF / DIT / coset round trips, custom shift).  CPU only."""
import random

import pytest

from oracle import oracle as O
from tests import fft_more_fields as M

NEW_FIELDS = ["bls24315_fr", "bls24317_fr", "bw6633_fr", "bw6761_fr"]
# maxOrderRoot and GeneratorFullMultiplicativeGroup as the reference states them
EXPECTED = {"bls24315_fr": (22, 7), "bls24317_fr": (60, 7), "bw6633_fr": (20, 13), "bw6761_fr": (46, 15)}


@pytest.mark.parametrize("frname", NEW_FIELDS)
def test_root_is_the_generator_power_of_exact_order(frname):
    q = O.FIELDS[frname].q
    P = M.FFT_PARAMS[frname]
    assert (P["max_order"], P["mult_gen"]) == EXPECTED[frname]
    # the 2-adicity of r - 1 is maxOrderRoot
    assert (q - 1) % (1 << P["max_order"]) == 0 and ((q - 1) >> P["max_order"]) % 2 == 1
    assert P["root"] == pow(P["mult_gen"], (q - 1) >> P["max_order"], q)
    assert pow(P["root"], 1 << P["max_order"], q) == 1
    assert pow(P["root"], 1 << (P["max_order"] - 1), q) == q - 1
    # mult_gen generates the full group: in particular it is a non-residue
    assert pow(P["mult_gen"], (q - 1) // 2, q) == q - 1


@pytest.mark.parametrize("frname", NEW_FIELDS)
def test_domain_constants_and_size_limit(frname):
    q = O.FIELDS[frname].q
    mx = M.FFT_PARAMS[frname]["max_order"]
    for lg in (1, 4, 10, min(20, mx)):
        d = M.FFTDomain(frname, (1 << lg) - (1 if lg > 1 else 0))
        assert d.cardinality == 1 << lg
        assert pow(d.generator, 1 << lg, q) == 1 and pow(d.generator, 1 << (lg - 1), q) == q - 1
        assert d.generator * d.generator_inv % q == 1 and d.cardinality * d.cardinality_inv % q == 1
    M.FFTDomain(frname, 1 << mx)
    with pytest.raises(ValueError, match="too big"):
        M.FFTDomain(frname, (1 << mx) + 1)


@pytest.mark.parametrize("frname", NEW_FIELDS)
def test_fft_matches_definition_and_roundtrips(frname):
    q = O.FIELDS[frname].q
    rng = random.Random(5)
    n = 32
    d = M.FFTDomain(frname, n)
    a = [rng.randrange(q) for _ in range(n)]
    evals = [sum(a[i] * pow(d.generator, i * k, q) for i in range(n)) % q for k in range(n)]
    assert O.bit_reverse(list(d.fft(list(a), O.DIF))) == evals
    assert d.fft(O.bit_reverse(list(a)), O.DIT) == evals
    assert d.fft_inverse(d.fft(list(a), O.DIF), O.DIT) == a
    assert d.fft_inverse(d.fft(O.bit_reverse(list(a)), O.DIT), O.DIF) == O.bit_reverse(list(a))
    cos = [sum(a[i] * pow(d.shift * pow(d.generator, k, q) % q, i, q) for i in range(n)) % q for k in range(n)]
    assert O.bit_reverse(d.fft(list(a), O.DIF, coset=True)) == cos
    assert d.fft(O.bit_reverse(list(a)), O.DIT, coset=True) == cos
    assert d.fft_inverse(d.fft(list(a), O.DIF, coset=True), O.DIT, coset=True) == a
    assert d.fft_inverse(d.fft(O.bit_reverse(list(a)), O.DIT, coset=True), O.DIF, coset=True) == O.bit_reverse(list(a))
    d2 = M.FFTDomain(frname, n, shift=12345)
    cos2 = [sum(a[i] * pow(12345 * pow(d2.generator, k, q) % q, i, q) for i in range(n)) % q for k in range(n)]
    assert d2.fft(O.bit_reverse(list(a)), O.DIT, coset=True) == cos2
