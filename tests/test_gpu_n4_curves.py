"""Next-row N4 remainder on the GPU (SURVEY.md section 8f; VERDICT r01 "what's missing" item 3): MultiExp of
  * secp256k1 G1 (ecc/secp256k1/multiexp.go:32) -- the base field AND the scalar field fill all 256 bits, so the field
    layer's carry-aware path runs (field.cuh Params::FULL) and a 16-bit window needs 17-bit digits in the last window
    (fr.Bits = 256 is a multiple of 16; the reference leaves c = 16 out of implementedCs for this curve, multiexp.go:77);
  * bw6-761 G1 and G2 (ecc/bw6-761/multiexp.go:32, :306) -- 12-word Fp (24 32-bit limbs per coordinate), BOTH groups
    over Fp, scalars of 6 words / 377 bits (48-byte fr.Element: every scalar stride of the C ABI is per curve);
  * bls24-315 / bls24-317 G1 (ecc/bls24-315/multiexp.go:32, ecc/bls24-317/multiexp.go:32) -- 5-word Fp: 40-byte coordinates,
    80-byte points, 120-byte Jacobian results, i.e. sizes that are not multiples of 16 bytes (8-byte load / store granules);
    G2 of these curves is over Fp4 and not provided;
  * bw6-633 G1 and G2 (ecc/bw6-633/multiexp.go:32, :304) -- 10-word Fp, both groups over Fp, 5-word scalars (40 bytes).
Same criteria as tests/test_gpu_msm.py: bit-exact affine limbs against the CPU oracle, through the C ABI."""
from importlib import import_module

import numpy as np
import pytest

from oracle import cref
from oracle import oracle as O
from tests.gpu_common import jac_to_affine_bytes, load_golden_msm, make_inputs

pytestmark = pytest.mark.gpu

N4 = ["secp256k1_g1", "bw6761_g1", "bw6761_g2", "bls24315_g1", "bls24317_g1", "bw6633_g1", "bw6633_g2"]


def _pkg():
    import gnark_crypto_b200 as pkg

    return pkg


@pytest.fixture(params=["affine", "xyzz"])
def accumulate_mode(request, monkeypatch):
    """both bucket-accumulation paths: the extended-Jacobian segmented reduction (the default) and the batch-affine tree
    (GMSM_AFFINE=1)"""
    monkeypatch.setenv("GMSM_AFFINE", "1" if request.param == "affine" else "0")
    return request.param


def _jac_cls(g):
    A1, J1, A2, J2 = _pkg().curve_package(g.split("_")[0])
    return (J1, A1) if g.endswith("g1") else (J2, A2)


def _engine_msm(g, pts, s, c):
    pkg = _pkg()
    n = pts.shape[0]
    eng = pkg.Engine(g, max(n, 1), c=c)
    try:
        return eng.msm_host_result(eng.to_device(pts), eng.to_device(s), n), eng.c
    finally:
        eng.close()


def test_sizes_of_the_new_curves():
    L = import_module("gnark-crypto_b200._native").lib()
    pkg = _pkg()
    for g, (ab, sb) in {"secp256k1_g1": (64, 32), "bw6761_g1": (192, 48), "bw6761_g2": (192, 48), "bls24315_g1": (80, 32),
                        "bls24317_g1": (80, 32), "bw6633_g1": (160, 40), "bw6633_g2": (160, 40)}.items():
        cid = pkg.CURVES[g]
        assert (L.gmsm_affine_bytes(cid), L.gmsm_scalar_bytes(cid), L.gmsm_jac_bytes(cid)) == (ab, sb, ab // 2 * 3)
        assert O.GROUPS[g].fr.limbs * 8 == sb
    for cv in ("secp256k1", "bls24315", "bls24317"):
        assert pkg.curve_package(cv)[2:] == (None, None)                # no G2 (bls24: over Fp4, not provided)


@pytest.mark.parametrize("g,n,cs", [("secp256k1_g1", 1500, [2, 4, 7, 8, 11, 13, 15, 16, 17, 19]),    # 16: last window 17 bits wide
                                     ("bw6761_g1", 500, [4, 5, 8, 10, 13, 16, 18]),                  # 13 * 29 = 377: last_c = 14
                                     ("bw6761_g2", 400, [5, 10, 16]),
                                     ("bls24315_g1", 1000, [2, 5, 8, 11, 13, 16, 19]),               # 253 = 11 * 23: last_c = 12
                                     ("bls24317_g1", 1000, [3, 8, 15, 16, 17]),                      # 255 = 15 * 17: last windows of c + 1 bits
                                     ("bw6633_g1", 600, [4, 5, 6, 7, 8, 9, 12, 15, 16, 18]),         # 315 = 5 * 63 = 7 * 45 = 9 * 35 = 15 * 21
                                     ("bw6633_g2", 400, [6, 12, 16])])
def test_window_sizes_agree_with_oracle(g, n, cs, accumulate_mode):
    """the widths the reference implements for the curve (multiexp.go:77) and the wider ones the GPU model may pick; inputs
    with the cross-test ingredients (infinities, duplicates, P / -P, zero scalars); both accumulation paths"""
    pts, s = make_inputs(g, n, 4321)
    want, _, used_c, _ = cref.msm(g, pts, s, c=0, nthreads=4)
    assert used_c in O.IMPLEMENTED_CS[g]
    G = O.GROUPS[g]
    w = pts.shape[1] // 2
    for c in cs:
        jac, used = _engine_msm(g, pts, s, c)
        assert used == c
        assert np.array_equal(jac[2 * w:], np.array(G.K.encode(G.K.one), dtype=np.uint64))
        assert np.array_equal(jac[: 2 * w], want), c
        assert np.array_equal(jac_to_affine_bytes(g, jac), want), c


@pytest.mark.parametrize("g", N4)
def test_committed_golden_vectors_and_one_shot_call(g):
    """tests/golden/msm_vectors.json (extreme scalars 0, 1, r - 1, 2^(Bits-1) + ...) through the engine and through the
    one-shot drop-in call of the curve's package"""
    pts, s, want = load_golden_msm(g)
    w = pts.shape[1] // 2
    for c in (6, 12):
        jac, _ = _engine_msm(g, pts, s, c)
        assert np.array_equal(jac[: 2 * w], want), c
    Jac, Aff = _jac_cls(g)
    pkg = _pkg()
    assert np.array_equal(Aff().MultiExp(pts, s, pkg.MultiExpConfig()).limbs, want)
    with pytest.raises(pkg.MultiExpError, match="len"):
        Jac().MultiExp(pts, s[:-1], pkg.MultiExpConfig())
    with pytest.raises(ValueError):
        Jac().MultiExp(pts, np.zeros((pts.shape[0], s.shape[1] + 1), dtype=np.uint64), pkg.MultiExpConfig())   # wrong fr.Limbs


@pytest.mark.parametrize("g", N4)
def test_infinity_zero_empty_and_extreme_scalars(g):
    pkg = _pkg()
    Jac, Aff = _jac_cls(g)
    G = O.GROUPS[g]
    pts, s = make_inputs(g, 300, 5, specials=False)
    j = Jac().MultiExp(np.zeros_like(pts), s, pkg.MultiExpConfig())
    assert j.IsInfinity() and not j.limbs.any()
    j = Jac().MultiExp(pts, np.zeros_like(s), pkg.MultiExpConfig())
    assert j.IsInfinity() and not j.limbs.any()
    assert Jac().MultiExp(pts[:0], s[:0], pkg.MultiExpConfig()).IsInfinity()
    j = Jac().MultiExp(pts[7:8], G.encode_scalars([1]), pkg.MultiExpConfig())
    assert np.array_equal(j.limbs[: pts.shape[1]], pts[7])
    # every scalar r - 1 (all windows at their extreme digits, carries rippling to the last window): sum of the negated points
    r = G.fr.q
    s_max = np.repeat(G.encode_scalars([r - 1]), 300, axis=0)
    want, _, _, _ = cref.msm(g, pts, s_max, c=0, nthreads=4)
    for c in (8, 16):
        jac, _ = _engine_msm(g, pts, s_max, c)
        assert np.array_equal(jac[: pts.shape[1]], want), c
    # scalars with the top bit of the scalar field's bit length set
    ks = [(1 << (G.fr.bits - 1)) + 17 * i for i in range(300)]
    ks = [k % r for k in ks]
    s_top = G.encode_scalars(ks)
    want, _, _, _ = cref.msm(g, pts, s_top, c=0, nthreads=4)
    for c in (13, 16):
        jac, _ = _engine_msm(g, pts, s_top, c)
        assert np.array_equal(jac[: pts.shape[1]], want), c


@pytest.mark.parametrize("g,n", [("secp256k1_g1", (1 << 19) + 11), ("bw6761_g1", (1 << 16) + 3), ("bw6761_g2", 1 << 15),
                                 ("bls24315_g1", (1 << 18) + 7), ("bls24317_g1", 1 << 18), ("bw6633_g1", (1 << 17) + 1), ("bw6633_g2", 1 << 15)])
def test_large_closed_form_and_host_paths(g, n):
    """bases [i+1]B generated on the device (pinned against the oracle on a sample), random scalars: the engine with its own
    window choice, the one-shot host call on pageable arrays (pinned staging ring; 48-byte scalars for bw6-761), resident
    bases and their window tables must all give [sum (i+1) s_i mod r] B"""
    pkg = _pkg()
    mx = import_module("gnark-crypto_b200.multiexp")
    G = O.GROUPS[g]
    base = G.encode_affine([G.scalar_mul(G.gen, 0xC0FFEE)])[0]
    w = base.size
    eng = pkg.Engine(g, n, c=0)
    try:
        d_pts = eng.generate_multiples(base, 1, n)
        host = d_pts.cpu().numpy().view(np.uint64).reshape(n, w)
        for i in (0, 1, 15, 16, 17, 4095, n // 2, n - 2, n - 1):
            assert np.array_equal(host[i], cref.scalar_mul(g, base, i + 1)), i
        s = cref.random_scalars(g, n, 4242)
        want = cref.scalar_mul(g, base, cref.dot_index(g, s, 1))
        assert np.array_equal(eng.msm_host_result(d_pts, eng.to_device(s), n)[:w], want)
    finally:
        eng.close()
    Jac, Aff = _jac_cls(g)
    assert np.array_equal(Aff().MultiExp(host, s, pkg.MultiExpConfig()).limbs, want)
    rb = mx.ResidentBases(g, host)
    try:
        assert np.array_equal(rb.MultiExp(s)[:w], want)
        m = n // 3
        want2 = cref.scalar_mul(g, base, cref.dot_index(g, s[:m], 1))
        assert np.array_equal(rb.MultiExp(s[:m])[:w], want2)
        rb.Precompute(0)
        assert np.array_equal(rb.MultiExp(s)[:w], want)
    finally:
        rb.close()


@pytest.mark.parametrize("g", ["secp256k1_g1", "bw6761_g1", "bls24317_g1", "bw6633_g1"])
@pytest.mark.parametrize("kind", ["smallvalues", "redundancy", "one_bucket"])
def test_skewed_scalar_distributions(g, kind):
    """multiexp_test.go:319-334's distributions: both modes of the counting sort and the carry levels with the new strides"""
    n = 20000 if g == "secp256k1_g1" else 6000
    pts, s = make_inputs(g, n, 77, specials=False)
    if kind == "smallvalues":
        s[::5] = 0
        s[::5, 0] = 1
    elif kind == "redundancy":
        for i in range(0, n, 100):
            s[i: i + 100] = s[i]
    else:
        s[:] = s[0]
    want, _, _, _ = cref.msm(g, pts, s, c=0, nthreads=8)
    for c in (8, 13):
        jac, _ = _engine_msm(g, pts, s, c)
        assert np.array_equal(jac[: pts.shape[1]], want), (kind, c)


def test_sharded_window_sums_compose_bw6761():
    """the multi-GPU decomposition with 6-word scalars: per-shard window partials, finalize over the 'ranks'"""
    import torch

    pkg = _pkg()
    g = "bw6761_g1"
    n = 6000
    pts, s = make_inputs(g, n, 31)
    want, _, _, _ = cref.msm(g, pts, s, c=0, nthreads=8)
    eng = pkg.Engine(g, n, c=10)
    try:
        parts = []
        for a, b in ((0, 1000), (1000, 4500), (4500, n)):
            out = torch.zeros(eng.partials_bytes // 8, dtype=torch.int64, device="cuda")
            eng.window_sums(eng.to_device(pts[a:b]), eng.to_device(s[a:b]), b - a, out=out)
            parts.append(out)
        jac = eng.finalize(torch.cat(parts), 3).cpu().numpy().view(np.uint64)
        assert np.array_equal(jac[: pts.shape[1]], want)
    finally:
        eng.close()


@pytest.mark.parametrize("g", ["secp256k1_g1", "bw6761_g2", "bls24315_g1", "bw6633_g1"])
def test_batch_scalar_multiplication_fixed_base(g):
    """BatchScalarMultiplicationG1 (ecc/secp256k1/g1.go, ecc/bw6-761/g2.go): same base, n scalars, affine out"""
    pkg = _pkg()
    G = O.GROUPS[g]
    base = G.encode_affine([G.scalar_mul(G.gen, 0xBEEF)])[0]
    n = 300
    s = cref.random_scalars(g, n, 9)
    specials = [0, 1, 2, G.fr.q - 1, G.fr.q - 2, (1 << 200) + 12345]
    s[: len(specials)] = G.encode_scalars(specials)
    got = pkg.BatchScalarMultiplication(g, base, s)
    ks = G.decode_scalars(s)
    for i in list(range(len(specials))) + [17, 100, 299]:
        assert np.array_equal(got[i], cref.scalar_mul(g, base, ks[i])), i
    assert not got[0].any() and np.array_equal(got[1], base)
