"""mpcsetup on the GPU (gmsm_scale_powers*, csrc/mpc_kernels.cuh; gnark-crypto_b200/mpcsetup.py) for the G1 and G2 groups of the
seven pairing curves, and secp256k1 through the C ABI:
  * the edge cases of the kernel (infinity inputs, c and r through 0, 1, r - 1 and random, tails of a thread) limb-exact against
    the big-int restatement (mpcsetup_ref);
  * closed forms at production size: UpdateMonomials on [tau^i]g is [(r tau)^i]g, ScaleG with (alpha, tau) on [g] * n is
    [alpha tau^i]g, the expected points from BatchScalarMultiplication (the independent fixed-base kernels);
  * the chunks of the host entry point, the device entry point (torch tensors, in place, a non-default stream, the input left
    unmodified out of place), the errors;
  * LinearCombinationsG1 / G2 on the tables of TestLinearCombinationsG1 / G2 (mpcsetup_test.go:67-218) against MultiExp with the
    expected coefficient vectors, against the restatement, on a geometric sequence (shifted = [tau] truncated);
  * a two-party contribution: r1 then r2 on [tau^i] gives [(tau r1 r2)^i]."""
import random
from importlib import import_module

import numpy as np
import pytest

from oracle import oracle as O
from tests import mpcsetup_ref as MR

pytestmark = pytest.mark.gpu

curves = import_module("gnark-crypto_b200.curves")
PAIRING = ("bn254", "bls12381", "bls12377", "bls24315", "bls24317", "bw6633", "bw6761")
G2_CURVES = ("bn254", "bls12381", "bls12377", "bw6633", "bw6761")
GROUPS = [c + "_g1" for c in PAIRING] + [c + "_g2" for c in G2_CURVES]


def _mpc():
    return import_module("gnark-crypto_b200.mpcsetup")


def _mx():
    return import_module("gnark-crypto_b200.multiexp")


def _native():
    return import_module("gnark-crypto_b200._native")


def _enc(name, ks):
    q = O.GROUPS[name].fr.q
    return curves._fr_encode([k % q for k in ks], q)


def _bsm(name, ks, base=None):
    G = O.GROUPS[name]
    base = G.encode_affine([G.gen])[0] if base is None else base
    return _mx().BatchScalarMultiplication(name, base, _enc(name, ks))


def _fns(name):
    curve, g = name.split("_")
    m = _mpc()
    suf = g.upper()
    return curve, getattr(m, "UpdateMonomials" + suf), getattr(m, "Scale" + suf), getattr(m, "LinearCombinations" + suf)


def _points(G, n, seed):
    """random multiples of the generator with infinity at 0, n - 1 and every 7th index from 2"""
    rng = random.Random(seed)
    pts = O.consecutive_multiples(G, n, 1, G.scalar_mul(G.gen, rng.randrange(1, G.fr.q)))
    for i in [0, n - 1] + list(range(2, n, 7)):
        pts[i] = G.aff_inf()
    return pts


def _first_diff(got, want):
    bad = [i for i in range(len(want)) if not np.array_equal(got[i], want[i])]
    return bad[0] if bad else None


@pytest.mark.parametrize("name", GROUPS + ["secp256k1_g1"])
def test_scale_powers_restatement(name):
    """out[i] = [c r^i] P[i] at n = 11 for c, r in {0, 1, r - 1, random}, and n = 1; UpdateMonomials on the same points (G1 / G2
    of the pairing curves through mpcsetup.py, secp256k1 through gmsm_scale_powers)"""
    G = O.GROUPS[name]
    q = G.fr.q
    rng = random.Random(G_ID(name))
    pts = _points(G, 11, 3)
    enc = G.encode_affine(pts)
    vals = [0, 1, q - 1, rng.randrange(2, q - 1)]
    L = _native().lib()
    for c in vals:
        for r in vals:
            got = enc.copy()
            cl, rl = _enc(name, [c, r])
            if name == "secp256k1_g1":
                assert L.gmsm_scale_powers(G_ID(name), got.ctypes.data, got.shape[0], cl.ctypes.data, rl.ctypes.data, 0, got.ctypes.data) == 0
            else:
                curve, _, scale, _ = _fns(name)
                scale(curve, got, cl, rl)
            want = G.encode_affine(MR.scale_powers(G, pts, c, r))
            assert _first_diff(got, want) is None, (name, c, r, _first_diff(got, want))
    if name != "secp256k1_g1":
        curve, upd, _, _ = _fns(name)
        r = rng.randrange(2, q)
        got = enc.copy()
        upd(curve, got, _enc(name, [r])[0])
        assert np.array_equal(got, G.encode_affine(MR.update_monomials(G, pts, r)))
        assert np.array_equal(got[0], enc[0])
        one = G.encode_affine(pts[1:2])
        _fns(name)[2](curve, one, _enc(name, [r])[0], _enc(name, [5])[0])
        assert np.array_equal(one, G.encode_affine([G.scalar_mul(pts[1], r)]))


def G_ID(name):
    return curves.GROUPS[name].id


@pytest.mark.parametrize("name", GROUPS)
def test_closed_forms_production_size(name):
    """2^20 points on G1, 2^18 on G2: UpdateMonomials(A = [tau^i]g, r) = [(r tau)^i]g (host array) and Scale(alpha, tau) on
    [g] * n = [alpha tau^i]g (device tensor, in place)"""
    import torch

    G = O.GROUPS[name]
    q = G.fr.q
    n = 1 << (20 if name.endswith("g1") else 18)
    rng = random.Random(7 + G_ID(name))
    tau, r, alpha = rng.randrange(2, q), rng.randrange(2, q), rng.randrange(2, q)
    curve, upd, scale, _ = _fns(name)

    def powers(x, c=1):
        out, v = [], c % q
        for _ in range(n):
            out.append(v)
            v = v * x % q
        return out

    A = _bsm(name, powers(tau))
    upd(curve, A, _enc(name, [r])[0])
    want = _bsm(name, powers(r * tau))
    assert _first_diff(A, want) is None, _first_diff(A, want)
    g = G.encode_affine([G.gen])
    d = torch.from_numpy(np.repeat(g, n, axis=0).view(np.int64)).cuda()
    scale(curve, d, _enc(name, [alpha])[0], _enc(name, [tau])[0])
    got = d.cpu().numpy().view(np.uint64)
    want = _bsm(name, powers(tau, alpha))
    assert _first_diff(got, want) is None, _first_diff(got, want)


@pytest.mark.parametrize("name,n", [("bn254_g1", (1 << 20) + 37), ("bn254_g2", (1 << 20) + 5)])
def test_host_chunks(name, n):
    """one host call across the 2^20-point chunk boundary: the second chunk continues the powers (c r^(2^20 + i))"""
    G = O.GROUPS[name]
    q = G.fr.q
    rng = random.Random(n)
    c, r = rng.randrange(2, q), rng.randrange(2, q)
    ks = [rng.randrange(1, q) for _ in range(64)] * (n // 64 + 1)
    ks = ks[:n]
    A = _bsm(name, ks)
    A[(1 << 20) - 1] = 0
    A[1 << 20] = 0
    out = np.zeros_like(A)
    cl, rl = _enc(name, [c, r])
    assert _native().lib().gmsm_scale_powers(G_ID(name), A.ctypes.data, n, cl.ctypes.data, rl.ctypes.data, 0, out.ctypes.data) == 0
    want_ks, s = [], c
    for i, k in enumerate(ks):
        want_ks.append(0 if i in ((1 << 20) - 1, 1 << 20) else k * s % q)
        s = s * r % q
    want = _bsm(name, want_ks)
    assert _first_diff(out, want) is None, _first_diff(out, want)


@pytest.mark.parametrize("name", ["bls12381_g1", "bw6761_g2"])
def test_device_entry(name):
    """gmsm_scale_powers_device on torch tensors on a non-default stream: out of place (input unmodified), then in place; equal
    to the host entry point"""
    import torch

    G = O.GROUPS[name]
    q = G.fr.q
    n = 3001
    rng = random.Random(11)
    c, r = rng.randrange(2, q), rng.randrange(2, q)
    A = _bsm(name, [rng.randrange(0, q) for _ in range(n)])
    cl, rl = _enc(name, [c, r])
    want = A.copy()
    L = _native().lib()
    assert L.gmsm_scale_powers(G_ID(name), want.ctypes.data, n, cl.ctypes.data, rl.ctypes.data, 0, want.ctypes.data) == 0
    d = torch.from_numpy(A.view(np.int64).copy()).cuda()
    d2 = d.clone()
    out = torch.empty_like(d)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        assert L.gmsm_scale_powers_device(G_ID(name), d.data_ptr(), n, cl.ctypes.data, rl.ctypes.data, out.data_ptr(), s.cuda_stream) == 0
    s.synchronize()
    assert np.array_equal(d.cpu().numpy().view(np.uint64), A)
    with torch.cuda.stream(s):
        assert L.gmsm_scale_powers_device(G_ID(name), d.data_ptr(), n, cl.ctypes.data, rl.ctypes.data, d.data_ptr(), s.cuda_stream) == 0
    s.synchronize()
    assert np.array_equal(out.cpu().numpy().view(np.uint64), want)
    assert np.array_equal(d.cpu().numpy().view(np.uint64), want)
    with torch.cuda.stream(s):
        _fns(name)[2](name.split("_")[0], d2, cl, rl)   # mpcsetup.py: the current stream, s
    s.synchronize()
    assert np.array_equal(d2.cpu().numpy().view(np.uint64), want)


def test_errors():
    import torch

    m = _mpc()
    L = _native().lib()
    name = "bn254_g1"
    G = O.GROUPS[name]
    q = G.fr.q
    A = _bsm(name, [3, 5, 7, 9])
    keep = A.copy()
    good = _enc(name, [2])[0]
    unreduced = np.array([(q >> (64 * i)) & (2**64 - 1) for i in range(4)], dtype=np.uint64)
    Err = _mx().MultiExpError
    with pytest.raises(Err, match="c is not a reduced fr.Element"):
        m.UpdateMonomialsG1("bn254", A, unreduced)
    with pytest.raises(Err, match="c is not a reduced fr.Element"):
        m.ScaleG1("bn254", A, unreduced)
    with pytest.raises(Err, match="r is not a reduced fr.Element"):
        m.ScaleG1("bn254", A, good, unreduced)
    assert np.array_equal(A, keep)
    with pytest.raises(IndexError):
        m.UpdateMonomialsG1("bn254", A[:1].copy(), good)
    with pytest.raises(IndexError):
        m.UpdateMonomialsG2("bn254", np.zeros((0, 16), dtype=np.uint64), good)
    for curve in ("bls24315", "bls24317"):
        with pytest.raises(ValueError, match="has no G2"):
            m.UpdateMonomialsG2(curve, np.zeros((4, 20), dtype=np.uint64), good)
        with pytest.raises(ValueError, match="has no G2"):
            m.LinearCombinationsG2(curve, np.zeros((4, 20), dtype=np.uint64), np.zeros((4, 4), dtype=np.uint64), [4])
    with pytest.raises(ValueError, match="writable"):
        m.ScaleG1("bn254", A.astype(np.int64), good)
    c = good.ctypes.data
    assert L.gmsm_scale_powers(13, A.ctypes.data, 4, c, c, 0, A.ctypes.data) == 1
    assert L.gmsm_scale_powers(0, None, 4, c, c, 0, A.ctypes.data) == 1
    assert L.gmsm_scale_powers(0, A.ctypes.data, 4, None, c, 0, A.ctypes.data) == 1
    assert L.gmsm_scale_powers(0, None, 0, None, None, 0, None) == 0     # n = 0: a no-op
    d = torch.from_numpy(A.view(np.int64).copy()).cuda()
    assert L.gmsm_scale_powers_device(0, d.data_ptr(), 3, c, c, d.data_ptr() + 64, None) == 1
    assert "overlap" in _native().last_error()
    assert L.gmsm_scale_powers_device(0, d.data_ptr(), 1 << 32, c, c, d.data_ptr(), None) == 1
    assert L.gmsm_scale_powers_device(0, d.data_ptr(), 4, unreduced.ctypes.data, c, d.data_ptr(), None) == 1
    assert np.array_equal(d.cpu().numpy().view(np.uint64), keep)


def _table_g1():
    """TestLinearCombinationsG1 (mpcsetup_test.go:67-168): (ends, powers, truncated powers, shifted powers, points or None); the
    points None are random multiples of the generator in place of the test's hash-to-curve points ("g" / "0": generator /
    infinity)"""
    return [
        ([3], [1, -1, 1], [1, -1, 0], [0, 1, -1], "0g0"),
        ([3], [1, 1, 1], [1, 1, 0], [0, 1, 1], "0g0"),
        ([3], [1, 1, 1], [1, 1, 0], [0, 1, 1], "00g"),
        ([3], [1, 1, 1], [1, 1, 0], [0, 1, 1], "g00"),
        ([3], [1, 2, 4], [1, 2, 0], [0, 1, 2], None),
        ([3, 6], [1] * 6, [1, 1, 0, 1, 1, 0], [0, 1, 1, 0, 1, 1], "g00000"),
        ([3, 6], [1, -1, 1, 1, -1, 1], [1, -1, 0, 1, -1, 0], [0, 1, -1, 0, 1, -1], "g00000"),
        ([4, 7], [1, 2, 4, 8, 3, 6, 12], [1, 2, 4, 0, 3, 6, 0], [0, 1, 2, 4, 0, 3, 6], None),
    ]


def _table_g2():
    """TestLinearCombinationsG2 (mpcsetup_test.go:170-218): one slice; truncated = powers[:-1], shifted = [0] + powers[:-1]"""
    rows = [([1, 1, 1], "g00"), ([1, 2, 4], "00g"), ([1, -1, 1], None), ([1, 3, 9, 27, 81], None)]
    return [([len(p)], p, p[:-1] + [0], [0] + p[:-1], pts) for p, pts in rows]


def _msm_affine(name, A, ks):
    words = 2 * curves.GROUPS[name].words
    j = _mx().curve_package(name.split("_")[0])[1 if name.endswith("g1") else 3]().MultiExp(A, _enc(name, ks))
    return j.limbs[:words] if j.limbs[words:].any() else np.zeros(words, dtype=np.uint64)


@pytest.mark.parametrize("name", GROUPS)
def test_linear_combinations_tables(name):
    """the reference's tables against MultiExp with the expected coefficients and against the restatement; host arrays and device
    tensors; A and powers unmodified"""
    import torch

    G = O.GROUPS[name]
    q = G.fr.q
    curve, _, _, lc = _fns(name)
    rng = random.Random(G_ID(name))
    table = _table_g1() if name.endswith("g1") else _table_g2()
    for ends, pw, tp, sp, spec in table:
        n = len(pw)
        if spec is None:
            A = _bsm(name, [rng.randrange(1, q) for _ in range(n)])
        else:
            A = G.encode_affine([G.gen if ch == "g" else G.aff_inf() for ch in spec])
        P = _enc(name, pw)
        A0, P0 = A.copy(), P.copy()
        t, s = lc(curve, A, P, ends)
        assert np.array_equal(t, _msm_affine(name, A, tp)), (ends, pw, spec, "truncated")
        assert np.array_equal(s, _msm_affine(name, A, sp)), (ends, pw, spec, "shifted")
        rt, rs = MR.linear_combinations(G, G.decode_affine(A), pw, ends)
        assert np.array_equal(t, G.encode_affine([rt])[0]) and np.array_equal(s, G.encode_affine([rs])[0])
        dA = torch.from_numpy(A.view(np.int64).copy()).cuda()
        dP = torch.from_numpy(P.view(np.int64).copy()).cuda()
        t2, s2 = lc(curve, dA, dP, ends)
        assert np.array_equal(t2, t) and np.array_equal(s2, s)
        t3, s3 = lc(curve, dA, P, ends)
        assert np.array_equal(t3, t) and np.array_equal(s3, s)
        assert np.array_equal(A, A0) and np.array_equal(P, P0)
        assert np.array_equal(dA.cpu().numpy().view(np.uint64), A0) and np.array_equal(dP.cpu().numpy().view(np.uint64), P0)
    # the reference's shortcut and its quirks: ends = [2]; a first slice of two points (powers[1] is zeroed, so its inverse is 0)
    A = _bsm(name, [rng.randrange(1, q) for _ in range(5)])
    t, s = lc(curve, A[:2].copy(), _enc(name, [1, 9]), [2])
    assert np.array_equal(t, A[0]) and np.array_equal(s, A[1])
    pw = [rng.randrange(q) for _ in range(5)]
    t, s = lc(curve, A, _enc(name, pw), [2, 5])
    rt, rs = MR.linear_combinations(G, G.decode_affine(A), pw, [2, 5])
    assert np.array_equal(t, G.encode_affine([rt])[0]) and np.array_equal(s, G.encode_affine([rs])[0])
    with pytest.raises(ValueError, match="lengths mismatch"):
        lc(curve, A, _enc(name, pw[:4]), [5])
    with pytest.raises(IndexError):
        lc(curve, A[:4].copy(), _enc(name, pw[:4]), [2, 4])


@pytest.mark.parametrize("name", ["bn254_g1", "bls12381_g2", "bw6761_g1"])
def test_linear_combinations_geometric(name):
    """UpdateMonomials turns [tau^i]g into a geometric sequence with ratio tau r; with random powers [1, x, x^2, ...] and several
    slices, shifted = [tau r] truncated"""
    G = O.GROUPS[name]
    q = G.fr.q
    curve, upd, _, lc = _fns(name)
    rng = random.Random(3)
    tau, r, x = rng.randrange(2, q), rng.randrange(2, q), rng.randrange(2, q)
    n = 4096
    A = _bsm(name, [pow(tau, i, q) for i in range(n)])
    upd(curve, A, _enc(name, [r])[0])
    # three slices, each geometric from its own start
    ends = [1000, 2500, n]
    pw, prev = [], 0
    for e in ends:
        pw += [pow(x, j, q) for j in range(e - prev)]
        prev = e
    P = _enc(name, pw)
    t, s = lc(curve, A, P, ends)
    want = _bsm(name, [tau * r % q], base=t)
    assert np.array_equal(s, want[0])
    assert t.any()


@pytest.mark.parametrize("curve", G2_CURVES)
def test_two_party_contribution(curve):
    """contributions r1 then r2 to [tau^i]G1 and [tau^i]G2 give [(tau r1 r2)^i]"""
    m = _mpc()
    rng = random.Random(len(curve))
    n = 1 << 12
    for g, upd in (("g1", m.UpdateMonomialsG1), ("g2", m.UpdateMonomialsG2)):
        name = curve + "_" + g
        q = O.GROUPS[name].fr.q
        tau, r1, r2 = rng.randrange(2, q), rng.randrange(2, q), rng.randrange(2, q)
        A = _bsm(name, [pow(tau, i, q) for i in range(n)])
        upd(curve, A, _enc(name, [r1])[0])
        upd(curve, A, _enc(name, [r2])[0])
        want = _bsm(name, [pow(tau * r1 * r2, i, q) for i in range(n)])
        assert _first_diff(A, want) is None, (name, _first_diff(A, want))
