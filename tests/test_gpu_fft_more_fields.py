"""The GPU Fr FFT for the scalar fields of bls24-315, bls24-317, bw6-633 and bw6-761 against the oracle (every size from 1 to
2^13, all decimation / coset / inverse variants, a custom shift that fills every limb), size-independent properties at
2^20 / 2^22 (round trips, the DIF+DIT compositions gnark uses, a sparse polynomial in closed form), and NewDomain's limit
at each field's maxOrderRoot."""
import importlib
import random

import numpy as np
import pytest

from oracle import oracle as O
from tests import fft_more_fields as M

pytestmark = pytest.mark.gpu
FR = {"bls24315": "bls24315_fr", "bls24317": "bls24317_fr", "bw6633": "bw6633_fr", "bw6761": "bw6761_fr"}
WORDS = {"bls24315": 4, "bls24317": 4, "bw6633": 5, "bw6761": 6}


def _fft():
    import gnark_crypto_b200  # noqa: F401

    return importlib.import_module("gnark-crypto_b200.fft")


def _enc(f, vals):
    return np.array([f.to_limbs(f.to_mont(v)) for v in vals], dtype=np.uint64)


def _dec(f, arr):
    return [f.from_mont(O.Field.from_limbs([int(x) for x in r])) for r in arr]


@pytest.mark.parametrize("curve", list(FR))
@pytest.mark.parametrize("logn", list(range(14)))
def test_fft_matches_oracle(curve, logn):
    fft = _fft()
    f = O.FIELDS[FR[curve]]
    n = 1 << logn
    rng = random.Random(1000 + logn)
    vals = [rng.randrange(f.q) for _ in range(n)]
    od = M.FFTDomain(FR[curve], n)
    d = fft.NewDomain(curve, n)
    assert d.Cardinality == n and d.words == WORDS[curve]
    consts = np.stack([d.Generator, d.GeneratorInv, d.CardinalityInv, d.FrMultiplicativeGen, d.FrMultiplicativeGenInv])
    assert consts.shape == (5, WORDS[curve])
    assert _dec(f, consts) == [od.generator, od.generator_inv, od.cardinality_inv, od.shift, od.shift_inv]
    for dec in (O.DIT, O.DIF):
        for coset in (False, True):
            a = _enc(f, vals)
            assert a.shape == (n, WORDS[curve])
            assert _dec(f, d.FFT(a, dec, OnCoset=coset)) == od.fft(vals, dec, coset), (dec, coset)
            a = _enc(f, vals)
            assert _dec(f, d.FFTInverse(a, dec, OnCoset=coset)) == od.fft_inverse(vals, dec, coset), (dec, coset)
    d.close()


@pytest.mark.parametrize("curve", list(FR))
def test_fft_custom_shift_and_errors(curve):
    fft = _fft()
    f = O.FIELDS[FR[curve]]
    n = 2048
    vals = [(i * i + 5) % f.q for i in range(n)]
    shift = (f.q - 1) // 3 + 987654321                 # uses the top limb of the element
    d = fft.NewDomain(curve, n - 5, shift=_enc(f, [shift])[0])
    od = M.FFTDomain(FR[curve], n, shift=shift)
    for dec in (O.DIT, O.DIF):
        assert _dec(f, d.FFT(_enc(f, vals), dec, OnCoset=True)) == od.fft(vals, dec, True)
        assert _dec(f, d.FFTInverse(_enc(f, vals), dec, OnCoset=True)) == od.fft_inverse(vals, dec, True)
    with pytest.raises(Exception, match="cardinality"):
        d.FFT(_enc(f, vals[:1024]), O.DIF)
    with pytest.raises(Exception, match="cardinality"):
        d.FFT(np.zeros((n, 4 if WORDS[curve] != 4 else 5), dtype=np.uint64), O.DIF)   # the wrong element width
    d.close()
    mx = M.FFT_PARAMS[FR[curve]]["max_order"]
    with pytest.raises(Exception, match="too big"):
        fft.NewDomain(curve, (1 << mx) + 1)


@pytest.mark.parametrize("curve,logn", [("bls24315", 20), ("bls24315", 22), ("bls24317", 20), ("bls24317", 22), ("bw6633", 20),
                                        ("bw6761", 20)])
def test_fft_large_properties(curve, logn):
    import torch

    fft = _fft()
    f = O.FIELDS[FR[curve]]
    w = WORDS[curve]
    n = 1 << logn
    d = fft.NewDomain(curve, n)
    rng = np.random.default_rng(logn)
    a = rng.integers(0, 2**62, size=(n, w), dtype=np.uint64)
    a[:, w - 1] = 0                                     # < q, arbitrary Montgomery residues
    da = torch.from_numpy(a.view(np.int64)).cuda()
    orig = da.clone()
    d.fft_device(da, False, O.DIF)
    assert not torch.equal(da, orig)
    d.fft_device(da, True, O.DIT)
    assert torch.equal(da, orig)
    d.fft_device(da, False, O.DIF, coset=True)
    d.fft_device(da, True, O.DIT, coset=True)
    assert torch.equal(da, orig)
    d.bit_reverse_device(da)
    d.fft_device(da, False, O.DIT)
    d.fft_device(da, True, O.DIF)
    d.bit_reverse_device(da)
    assert torch.equal(da, orig)
    # closed form: p(X) = c0 + c1 X^k  ->  evaluations c0 + c1 w^(k i)
    k, c0, c1 = 12345, 7, 11
    vals = np.zeros((n, w), dtype=np.uint64)
    vals[0] = _enc(f, [c0])[0]
    vals[k] = _enc(f, [c1])[0]
    dv = torch.from_numpy(vals.view(np.int64)).cuda()
    d.bit_reverse_device(dv)
    d.fft_device(dv, False, O.DIT)
    out = dv.cpu().numpy().view(np.uint64)
    od = M.FFTDomain(FR[curve], n)
    for i in (0, 1, 2, 1000, n // 2 + 3, n - 1):
        want = (c0 + c1 * pow(od.generator, k * i, f.q)) % f.q
        assert _dec(f, out[i : i + 1])[0] == want, i
    d.close()
