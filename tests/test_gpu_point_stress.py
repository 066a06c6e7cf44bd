"""The sm_90a variable-base point kernels shared by kzg.ToLagrangeG1 and mpcsetup (lag_scalar_mul, k_lag_stage, k_lag_finish,
k_scale_powers) at adversarial scalars, colliding butterflies and production sizes (generators and references in
tests/point_stress.py; the CPU twin is tests/test_point_stress_cpu.py):

A. scalars that steer the ladder, all thirteen groups (ScaleG1 / ScaleG2 of mpcsetup.py, gmsm_scale_powers_device for
   secp256k1): geometric families that walk every bit, r - 2^i, repeated halving, r - 2 on every point (the ladder's last addition
   is then a doubling: xyzz_add's P == Q branch), and scalars built digit by digit for W = 3, 4 and 5 (extreme digits, one
   non-zero window, the top digit at its maximum, Horner loops of zero and one step); expected points from the oracle's C port;
B. every infinity mask of the per-thread shared inversion of k_scale_powers, against BatchScalarMultiplication;
C. equal, opposite and infinite butterfly partners planted at every stage of ToLagrangeG1, at j = 0, 1 and the last j of a block,
   seven curves (stages s >= 1 are where a + b cancels and a - b doubles inside the twiddle's block);
D. production sizes: ToLagrangeG1 on the largest domains of bls24-315 (2^22) and bw6-633 (2^20), and 2^20 on bls12-377,
   bls24-317 and bls12-381; UpdateMonomials on device tensors above 2^20 points, so that bits 20 to 23 of the thread index
   `first` of k_scale_powers build the first scalar of a thread.  Bits 24 to 31 would need 2^30 or more points and are not run.

The references of A and C run in a pool of worker processes while the device computes."""
import multiprocessing
import os
import random
from concurrent.futures import ProcessPoolExecutor
from importlib import import_module

import numpy as np
import pytest

from tests import lagrange_ref as LR
from tests import point_stress as S

pytestmark = pytest.mark.gpu


def _torch():
    return import_module("torch")


def _native():
    return import_module("gnark-crypto_b200._native")


def _mx():
    return import_module("gnark-crypto_b200.multiexp")


def _mpc():
    return import_module("gnark-crypto_b200.mpcsetup")


def _kzg():
    return import_module("gnark-crypto_b200.kzg")


def _dev(a):
    return _torch().from_numpy(np.ascontiguousarray(a, dtype=np.uint64).view(np.int64).reshape(-1).copy()).cuda()


def _host(t, w):
    return t.cpu().numpy().view(np.uint64).reshape(-1, w)


def _stream():
    return _torch().cuda.current_stream().cuda_stream


def _cid(name):
    return _mx().CURVES[name]


def _bsm(name, ks):
    """[k_i]G by BatchScalarMultiplication (k = 0: infinity)"""
    G = S.group(name)
    return _mx().BatchScalarMultiplication(name, S.gen_enc(name), G.encode_scalars([k % G.fr.q for k in ks]))


@pytest.fixture(scope="module")
def refs():
    """submit over a pool of spawned worker processes (no CUDA in them), shut down with the module"""
    ex = ProcessPoolExecutor(max_workers=max(1, min(16, (os.cpu_count() or 2) - 1)), mp_context=multiprocessing.get_context("spawn"))
    try:
        yield ex
    finally:
        ex.shutdown(cancel_futures=True)


def _scale(name, d, c, r):
    """d[i] <- [c r^i] d[i] in place on a device tensor: ScaleG1 / ScaleG2 for the pairing groups, the C ABI for secp256k1"""
    G = S.group(name)
    cl, rl = (np.ascontiguousarray(x) for x in G.encode_scalars([c, r]))
    if name == "secp256k1_g1":
        n = d.numel() // G.aff_words
        assert _native().lib().gmsm_scale_powers_device(_cid(name), d.data_ptr(), n, cl.ctypes.data, rl.ctypes.data, d.data_ptr(),
                                                         _stream()) == 0, _native().last_error()
        return
    curve, g = name.split("_")
    getattr(_mpc(), "Scale" + g.upper())(curve, d, cl, rl)


# ---- A ----
def _ladder_calls(name):
    """family A as calls (family, case, points, c, r): 19 random points per digit-built call (r = 1), fr.Bits + 40 points for a
    geometric family; one infinity per call, at a position that moves from call to call"""
    ks, pts = S.random_points(name, S.CALL_POINTS, 21)
    calls = []
    for fam in S.GEOMETRIC:
        c, r, n = S.geometric(name, fam)
        calls.append(("geometric", "(c, r) = (%s)" % fam, pts[np.arange(n) % S.CALL_POINTS], c, r))
    for W in S.WIDTHS:
        for case, s, _ in S.digit_cases(name, W):
            calls.append(("digits", "%s W=%d" % (case, W), pts, s, 1))
    out = []
    for k, (fam, case, p, c, r) in enumerate(calls):
        p = p.copy()
        p[(7 * k) % p.shape[0]] = 0
        out.append((fam, case, p, c, r))
    return out


@pytest.mark.parametrize("name", S.GROUPS)
def test_ladder_scalars_device(name, refs):
    """family A: every call is one launch of k_scale_powers on its own slice of one device tensor, compared limb for limb with
    [c r^i] P_i from the C port.  The r - 2 calls (geometric (r - 2, 1), (r - 2, r - 1) and the digit case r - 2) are the ones
    whose last ladder addition takes xyzz_add's doubling branch; the others steer the digits (see point_stress.digit_cases)."""
    q = S.group(name).fr.q
    w = S.group(name).aff_words
    calls = _ladder_calls(name)
    pts = np.concatenate([p for _, _, p, _, _ in calls])
    ss = [s for _, _, p, c, r in calls for s in S.geometric_scalars(q, c, r, p.shape[0])]
    cut = list(range(0, pts.shape[0], 256)) + [pts.shape[0]]
    want = [refs.submit(S.expected_scaled, (name, pts[a:b], ss[a:b])) for a, b in zip(cut, cut[1:])]
    d = _dev(pts)
    lo = 0
    for _, _, p, c, r in calls:
        m = p.shape[0]
        _scale(name, d[lo * w : (lo + m) * w], c, r)
        lo += m
    got = _host(d, w)
    want = np.concatenate([f.result() for f in want])
    lo = 0
    for fam, case, p, c, r in calls:
        m = p.shape[0]
        S.compare("%s A %s %s (c = %d, r = %d)" % (name, fam, case, c, r), got[lo : lo + m], want[lo : lo + m], ss[lo : lo + m])
        lo += m


# ---- B ----
@pytest.mark.parametrize("name", ["bn254_g1", "bls12381_g2", "bw6761_g1", "secp256k1_g1"])
def test_mask_normalisation_device(name):
    """family B: 256 threads of 8 points carrying every infinity mask over the distinct points [i + 1]G (the device generator),
    then a tail of 5; out[i] = [c r^i][i + 1]G with r != 1, so every finite output differs"""
    torch = _torch()
    G = S.group(name)
    q, w = G.fr.q, G.aff_words
    rng = random.Random(_cid(name))
    c, r = rng.randrange(2, q), rng.randrange(2, q)
    d = torch.empty(S.MASK_N * w, dtype=torch.int64, device="cuda")
    base = S.gen_enc(name)
    assert _native().lib().gmsm_generate_multiples_device(_cid(name), base.ctypes.data, 1, S.MASK_N, d.data_ptr(), _stream()) == 0
    inf = torch.tensor(S.mask_layout(), device="cuda")
    d.view(S.MASK_N, w)[inf] = 0
    _scale(name, d, c, r)
    _, ks_out = S.mask_logs(name, c, r)
    S.compare("%s B infinity masks (c = %d, r = %d)" % (name, c, r), _host(d, w), _bsm(name, ks_out), ks_out)


# ---- C ----
@pytest.mark.parametrize("curve", LR.CURVES)
def test_planted_stages_device(curve, refs):
    """family C: for every stage s, equal, opposite, one-sided and two-sided infinite partners planted at j = 0, 1 and h - 1 of the
    state at the start of stage s; n = 32 against the point-domain restatement (lagrange_ref.to_lagrange_g1), n = 1024 against
    BatchScalarMultiplication of the scalar-domain one"""
    kzg = _kzg()
    name = curve + "_g1"
    small = S.planted_transforms(curve, 32, 5)
    want_small = [refs.submit(S.lagrange_points_ref, (curve, logs)) for _, _, logs in small]
    for s, plan, logs in S.planted_transforms(curve, 1024, 9):
        got = kzg.ToLagrangeG1(_bsm(name, logs), curve)
        S.compare("%s C n=1024 stage %d: %s" % (curve, s, S.plan_text(plan)), got, _bsm(name, LR.to_lagrange_scalars(curve, logs)))
    gots = [kzg.ToLagrangeG1(_bsm(name, logs), curve) for _, _, logs in small]
    for (s, plan, _), got, want in zip(small, gots, want_small):
        S.compare("%s C n=32 stage %d: %s" % (curve, s, S.plan_text(plan)), got, want.result())


# ---- D ----
def _msm_all_ones(name, d_pts, n):
    """sum of the n points of a device tensor: one MultiExp with every scalar 1 (np.tile of the encoded 1), as an affine row"""
    G = S.group(name)
    ones = _dev(np.tile(G.encode_scalars([1])[0], n))
    eng = _mx().Engine(name, n)
    try:
        j = eng.msm_host_result(d_pts, ones, n)
    finally:
        eng.close()
    w = G.aff_words // 2
    return j[: 2 * w] if j[2 * w :].any() else np.zeros(2 * w, dtype=np.uint64)


@pytest.mark.parametrize("curve,logn", [("bls24315", 22), ("bw6633", 20), ("bls12377", 20), ("bls24317", 20), ("bls12381", 20)])
def test_to_lagrange_production_size(curve, logn):
    """family D, ToLagrangeG1 on the ramp [1]G ... [n]G (the device generator), device tensors in and out: >= 4096 sampled
    indices against the closed form (out_0 = [(n + 1)/2]G, out_j = [1 / (w^-j - 1)]G), and the whole output by its sum, which is
    in_0 = G.  bls24-315 at 2^22 and bw6-633 at 2^20 run the largest domain each admits (the full 2-adic root)."""
    torch = _torch()
    name = curve + "_g1"
    G = S.group(name)
    n, w = 1 << logn, G.aff_words
    pts = torch.empty(n * w, dtype=torch.int64, device="cuda")
    base = S.gen_enc(name)
    assert _native().lib().gmsm_generate_multiples_device(_cid(name), base.ctypes.data, 1, n, pts.data_ptr(), _stream()) == 0
    out = _kzg().ToLagrangeG1(pts, curve)
    del pts
    idx = S.sample_indices(n, logn)
    got = _host(out.view(n, w)[torch.tensor(idx, device="cuda")], w)
    ks = S.ramp_lagrange(curve, n, idx)
    S.compare("%s D ToLagrangeG1 ramp n=2^%d (scalar: the expected log)" % (curve, logn), got, _bsm(name, ks), ks, idx)
    assert np.array_equal(_msm_all_ones(name, out, n), base), (curve, logn, "sum of the outputs is not G")


@pytest.mark.parametrize("name,n", [("bn254_g1", (1 << 24) + 3), ("bls12381_g1", (1 << 22) + 1), ("bn254_g2", (1 << 21) + 5)])
def test_update_monomials_production_size(name, n):
    """family D, UpdateMonomials on a device tensor of n copies of G: out_0 = G, out_i = [r^i]G at 0, 7, 8, 9, every 2^k - 1, 2^k,
    2^k + 1, the last 64 and 4096 random indices; the whole output by its sum [(r^n - 1)/(r - 1)]G.  The threads past 2^20 points
    build their first scalar from r^(2^k) for k up to 23."""
    torch = _torch()
    G = S.group(name)
    q, w = G.fr.q, G.aff_words
    curve, g = name.split("_")
    r = random.Random(n).randrange(2, q)
    base = S.gen_enc(name)
    d = torch.from_numpy(base.view(np.int64).copy()).cuda().repeat(n)
    getattr(_mpc(), "UpdateMonomials" + g.upper())(curve, d, G.encode_scalars([r])[0])
    idx = S.monomial_indices(n, n)
    got = _host(d.view(n, w)[torch.tensor(idx, device="cuda")], w)
    ks = [pow(r, i, q) for i in idx]
    S.compare("%s D UpdateMonomials n=%d r=%d" % (name, n, r), got, _bsm(name, ks), ks, idx)
    total = (pow(r, n, q) - 1) * pow(r - 1, -1, q) % q
    assert np.array_equal(_msm_all_ones(name, d, n), _bsm(name, [total])[0]), (name, n, "sum of the outputs")
