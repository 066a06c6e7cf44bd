"""CPU twin of tests/test_gpu_arith_stress.py: the same operand generators (tests/arith_stress.py), thinned, through the
hostcheck builds of the device's carry-chain formulation (tests/test_hostcheck.py: -DGMSM_EMULATE_PTX, dropped carries
trap) -- "emulated" (plain product), "emulated_fp2dot" (dedicated squaring, fused two-product reduction, Fp2 product as two
fused reductions) and "emulated_dot4" (plus the four-product reduction behind the Fp2 sum of products) -- and the digit
recoding kernel k_digits_hist run by the kernel emulator (tests/emu).  A device-only failure of the GPU twin then points at
the PTX / the compiler, a failure here at the formulation."""
import ctypes
import types

import numpy as np
import pytest

from oracle import cref
from oracle import oracle as O
from tests import arith_stress as S
from tests import test_emu_kernels as EMU
from tests import test_hostcheck as HC

GROUPS = list(O.GROUPS)
FP2_GROUPS = [g for g in GROUPS if O.GROUPS[g].K.ext == 2]
# the fused four-product reduction only changes the Fp2 groups; the other two builds change every group
CASES = [("emulated", g) for g in GROUPS] + [("emulated_fp2dot", g) for g in GROUPS] + [("emulated_dot4", g) for g in FP2_GROUPS]


@pytest.mark.parametrize("variant,g", CASES)
def test_field_arith_extremes_host(variant, g):
    G = O.GROUPS[g]
    run = HC._runner(HC._build(variant), g)
    S.check_field_stress(G, run, "%s %s" % (variant, g), n_sample=2000, all_pairs=False, n_inv_random=16)
    if variant == "emulated":
        S.check_fr_from_mont_stress(G, run, "%s %s" % (variant, g))


@pytest.mark.parametrize("variant", ["emulated", "emulated_fp2dot"])
def test_field_arith_extremes_host_secp256k1_fr(variant):
    """the second full-width modulus (no spare top bit) through the same multiplier, as a coordinate field"""
    G = types.SimpleNamespace(K=O.FpOps(O.FIELDS["secp256k1_fr"]))
    S.check_field_stress(G, HC._runner(HC._build(variant), "secp256k1_fr"), "%s secp256k1_fr" % variant, n_sample=2000,
                         all_pairs=False, n_inv_random=16)


@pytest.mark.parametrize("variant,g", [("emulated_fp2dot", g) for g in GROUPS] + [("emulated_dot4", "bn254_g2")])
def test_point_ops_extreme_z_host(variant, g):
    S.check_point_stress(O.GROUPS[g], HC._runner(HC._build(variant), g), "%s %s" % (variant, g), n=48)


def emu_digits(g, s, c, rank_mode):
    s = np.ascontiguousarray(s, dtype=np.uint64)
    n = s.shape[0]
    W = O.compute_nb_chunks(O.GROUPS[g].fr.bits, c)
    out = np.full((W, n), 0xFFFFFFFF, dtype=np.uint32)
    rc = getattr(EMU._lib(), "emu_digits_%d" % GROUPS.index(g))(s.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(n), c, rank_mode,
                                                                 out.ctypes.data_as(ctypes.c_void_p))
    assert rc == 0, rc
    return out


@pytest.mark.parametrize("g", GROUPS)
def test_digits_emulated_kernel(g):
    """k_digits_hist (plain mode at every width below, rank mode at two) against the C port of partitionScalars, on the
    scalar families and random scalars, at a spread of widths and every width at which the last window holds 1 bit or c
    bits (digit with carry c + 1 bits)"""
    G = O.GROUPS[g]
    widths = sorted({2, 3, 5, 8, 13, 16, 17, 20, 24} | set(S.last_window_widths(G.fr.bits)))
    for c in widths:
        s = S.digit_scalars(G, c, 200, 9000 + c)
        want = cref.partition_scalars(g, s, c)
        for rank_mode in ((0, 1) if c in (5, 16) else (0,)):
            got = emu_digits(g, s, c, rank_mode)
            if not np.array_equal(got, want):
                j, i = (int(x[0]) for x in np.nonzero(got != want))
                raise AssertionError("emulated %s digits c=%d rank_mode=%d: first failure at scalar #%d (plain %d), window %d: got %d, "
                                     "want %d" % (g, c, rank_mode, i, G.decode_scalars(s[i : i + 1])[0], j, got[j, i], want[j, i]))
