"""The sm_90a device arithmetic of all thirteen groups at the operands where carry chains break (tests/arith_stress.py):
Montgomery product, dedicated squaring, fused two- and four-product reductions (GMSM_OP_FDOT2), the Fp2 product, addition,
subtraction, negation, doubling, binary-GCD inversion, fromMont, the signed-digit recoding at every window width, the point
formulas on extreme z and the Fr FFT butterflies on extreme inputs -- limb-exact against big-int references.  The CPU twin
(tests/test_arith_stress_cpu.py) runs the same generators through the emulated carry-chain builds."""
import importlib

import numpy as np
import pytest

from oracle import cref
from oracle import oracle as O
from tests import arith_stress as S

pytestmark = pytest.mark.gpu
GROUPS = list(O.GROUPS)


def _mx():
    import gnark_crypto_b200  # noqa: F401

    return importlib.import_module("gnark-crypto_b200.multiexp")


def _runner(g):
    mx = _mx()

    def run(op, a, b, out_words):
        return mx.test_op(g, op, a, b, out_words)

    return run


@pytest.mark.parametrize("g", GROUPS)
def test_field_arith_extremes_device(g):
    """Fp: every ordered pair of extremes (FMUL, FADD, FSUB), 2^16 sampled quadruples (FDOT2); Fp2: 2^16 sampled pairs and
    quadruples plus the corners; unary ops on every extreme; FINV on every extreme plus 4096 random values"""
    G = O.GROUPS[g]
    S.check_field_stress(G, _runner(g), "device %s" % g)
    S.check_fr_from_mont_stress(G, _runner(g), "device %s" % g)


@pytest.mark.parametrize("g", GROUPS)
def test_point_ops_extreme_z_device(g):
    S.check_point_stress(O.GROUPS[g], _runner(g), "device %s" % g)


@pytest.mark.parametrize("g", GROUPS)
def test_digits_all_widths_device(g):
    """k_digits_dump (DigitStream over Fr::N limbs) against the C port of partitionScalars at every width 2..24"""
    mx = _mx()
    G = O.GROUPS[g]
    for c in range(2, 25):
        s = S.digit_scalars(G, c, 2000, 7000 + c)
        got = mx.test_digits(g, c, s)
        want = cref.partition_scalars(g, s, c)
        if not np.array_equal(got, want):
            j, i = (int(x[0]) for x in np.nonzero(got != want))
            raise AssertionError("device %s digits c=%d: first failure at scalar #%d (plain %d), window %d: got %d, want %d"
                                 % (g, c, i, G.decode_scalars(s[i : i + 1])[0], j, got[j, i], want[j, i]))


@pytest.mark.parametrize("frname", ["bn254_fr", "bls12381_fr", "bls12377_fr"])
@pytest.mark.parametrize("logn", [1, 5, 11])
def test_fft_extreme_inputs_device(frname, logn):
    """FFT / FFTInverse, DIT and DIF, with and without coset, of all q-1, all -1, 0 / q-1 alternations, a single q-1
    spike and all R mod q"""
    fft = importlib.import_module("gnark-crypto_b200.fft")
    f = O.FIELDS[frname]
    n = 1 << logn
    od = O.FFTDomain(frname, n)
    d = fft.NewDomain(frname.split("_")[0], n)
    try:
        for name, stored in S.fft_inputs(f, n).items():
            plain = [f.from_mont(v) for v in stored]
            for dec in (O.DIT, O.DIF):
                for coset in (False, True):
                    for inverse in (False, True):
                        a = np.array([f.to_limbs(v) for v in stored], dtype=np.uint64)
                        out = (d.FFTInverse if inverse else d.FFT)(a, dec, OnCoset=coset)
                        got = [O.Field.from_limbs([int(x) for x in r]) for r in out]
                        want = (od.fft_inverse if inverse else od.fft)(plain, dec, coset)
                        what = "device %s logn=%d %s %s%s%s" % (frname, logn, name, "FFTInverse" if inverse else "FFT",
                                                               " DIF" if dec == O.DIF else " DIT", " coset" if coset else "")
                        assert all(v < f.q for v in got), what + ": non-canonical output"
                        assert [f.from_mont(v) for v in got] == want, what
    finally:
        d.close()
