"""kzg.ToLagrangeG1 on the GPU (gmsm_g1_to_lagrange*, csrc/lagrange_kernels.cuh) for the G1 groups of the seven pairing curves:
limb-exact against the big-int restatement of the reference (lagrange_ref) on small inputs with infinity, equal and opposite
butterfly partners; the closed form L_i(alpha) of an SRS with known alpha (TestToLagrangeG1, kzg_test.go:81-118), expected points
from BatchScalarMultiplication (the independent fixed-base kernels); structural closed forms; Commit with the Lagrange-form key
equals CommitLagrange (TestCommitLagrange, kzg_test.go:120-155); the reference's errors; torch tensors, in-place and stream use of
the device entry point; the C++ mirror (tests/cpp/lagrange_test.cpp)."""
import os
import random
import subprocess
from importlib import import_module

import numpy as np
import pytest

from tests import lagrange_ref as LR

curves = import_module("gnark-crypto_b200.curves")

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBDIR = os.path.join(ROOT, "gnark-crypto_b200")


def _kzg():
    return import_module("gnark-crypto_b200.kzg")


def _mx():
    return import_module("gnark-crypto_b200.multiexp")


def _gen(curve):
    G = LR.group(curve)
    return G.encode_affine([G.gen])[0]


def _bsm(curve, base, ks):
    """[k_i] base for every k_i (BatchScalarMultiplication on the GPU; k = 0 gives infinity)"""
    r = LR.fr_modulus(curve)
    return _mx().BatchScalarMultiplication(curve + "_g1", base, _kzg()._fr_encode([k % r for k in ks], r))


def _special_scalars(curve, n, seed):
    """discrete logs with infinity, equal and opposite partners of the first stage (i, i + n/2)"""
    r = LR.fr_modulus(curve)
    rng = random.Random(seed)
    ks = [rng.randrange(1, r) for _ in range(n)]
    h = n // 2
    if n == 2:
        ks[1] = ks[0]
    if n >= 4:
        ks[h], ks[h + 1] = 0, ks[1]
    if n >= 8:
        ks[h + 2], ks[h - 1] = r - ks[2], 0
    return ks


@pytest.mark.parametrize("curve", LR.CURVES)
def test_matches_reference(curve):
    """n = 1, 2, 4, 32 against the point-domain restatement; n = 1024 against the scalar-domain one"""
    kzg = _kzg()
    G = LR.group(curve)
    for n in (1, 2, 4, 32):
        ks = _special_scalars(curve, n, 31 + n)
        pts = [G.scalar_mul(G.gen, k) if k else G.aff_inf() for k in ks]
        enc = G.encode_affine(pts)
        keep = enc.copy()
        got = kzg.ToLagrangeG1(enc, curve)
        assert np.array_equal(enc, keep)
        assert np.array_equal(got, G.encode_affine(LR.to_lagrange_g1(curve, pts))), (curve, n)
    n = 1024
    ks = _special_scalars(curve, n, 77)
    gen = _gen(curve)
    got = kzg.ToLagrangeG1(_bsm(curve, gen, ks), curve)
    assert np.array_equal(got, _bsm(curve, gen, LR.to_lagrange_scalars(curve, ks)))


def _closed_form(curve, logn, alpha):
    """TestToLagrangeG1: the SRS [alpha^i]G in, [L_i(alpha)]G out, L_i(alpha) = w^i (alpha^n - 1) / (n (alpha - w^i))"""
    kzg = _kzg()
    r = LR.fr_modulus(curve)
    n = 1 << logn
    w_inv, _ = LR.domain_inverses(curve, n)
    w = pow(w_inv, -1, r)
    gen = _gen(curve)
    srs, a = [], 1
    for _ in range(n):
        srs.append(a)
        a = a * alpha % r
    num = (pow(alpha, n, r) - 1) % r
    dens, wi = [], 1
    for _ in range(n):
        dens.append(n * (alpha - wi) % r)
        wi = wi * w % r
    # batch inversion of the denominators
    pref, acc = [], 1
    for d in dens:
        pref.append(acc)
        acc = acc * d % r
    inv = pow(acc, -1, r)
    lag = [0] * n
    wi = pow(w, n - 1, r)
    for i in range(n - 1, -1, -1):
        lag[i] = wi * num % r * (inv * pref[i] % r) % r
        inv = inv * dens[i] % r
        wi = wi * w_inv % r
    got = kzg.ToLagrangeG1(_bsm(curve, gen, srs), curve)
    assert np.array_equal(got, _bsm(curve, gen, lag)), (curve, logn)


@pytest.mark.parametrize("curve", LR.CURVES)
def test_closed_form_srs(curve):
    _closed_form(curve, 12, 0x1234567890ABCDEF123 + len(curve))


@pytest.mark.parametrize("curve,logn", [("bn254", 20), ("bw6761", 16)])
def test_closed_form_srs_large(curve, logn):
    _closed_form(curve, logn, 0xFEDCBA987654321)


@pytest.mark.parametrize("curve", LR.CURVES)
def test_structural_closed_forms(curve):
    """at 2^16: a constant input P gives (P, inf, ..., inf) (every difference cancels); P at index 0, infinity elsewhere, gives
    [1/n]P everywhere"""
    kzg = _kzg()
    n = 1 << 16
    r = LR.fr_modulus(curve)
    P = _bsm(curve, _gen(curve), [0x5EED1234 + len(curve)])[0]
    got = kzg.ToLagrangeG1(np.tile(P, (n, 1)), curve)
    assert np.array_equal(got[0], P) and not got[1:].any()
    x = np.zeros((n, P.shape[0]), dtype=np.uint64)
    x[0] = P
    got = kzg.ToLagrangeG1(x, curve)
    want = _bsm(curve, P, [pow(n, -1, r)])[0]
    assert np.array_equal(got, np.tile(want, (n, 1)))


@pytest.mark.parametrize("curve", LR.CURVES)
def test_commit_with_lagrange_key(curve):
    """TestCommitLagrange at 2^16 with arbitrary (non-SRS) points: Commit(evals, ProvingKey(ToLagrangeG1(P))) ==
    CommitLagrange(evals, ProvingKey(P), domain)"""
    kzg = _kzg()
    fft = import_module("gnark-crypto_b200.fft")
    n = 1 << 16
    r = LR.fr_modulus(curve)
    rng = random.Random(99)
    P = _bsm(curve, _gen(curve), [rng.randrange(1, r) for _ in range(n)])
    evals = curves._fr_encode([rng.randrange(r) for _ in range(n)], r)
    pk_lag = kzg.ProvingKey(curve, kzg.ToLagrangeG1(P, curve))
    pk = kzg.ProvingKey(curve, P)
    dom = fft.NewDomain(curve, n)
    try:
        assert np.array_equal(kzg.Commit(evals, pk_lag), kzg.CommitLagrange(evals, pk, dom))
    finally:
        pk.close()
        pk_lag.close()
        dom.close()


def test_errors():
    kzg = _kzg()
    mx = _mx()
    words = {c: LR.group(c).aff_words for c in LR.CURVES}
    for curve in LR.CURVES:
        for n in (0, 3, 6):
            with pytest.raises(mx.MultiExpError, match=r"^len\(coeffs\) must be a power of 2$"):
                kzg.ToLagrangeG1(np.zeros((n, words[curve]), dtype=np.uint64), curve)
    with pytest.raises(mx.MultiExpError, match=r"^m \(2097152\) is too big: the required root of unity does not exist$"):
        kzg.ToLagrangeG1(np.zeros((1 << 21, words["bw6633"]), dtype=np.uint64), "bw6633")
    with pytest.raises(mx.MultiExpError, match=r"^m \(8388608\) is too big: the required root of unity does not exist$"):
        kzg.ToLagrangeG1(np.zeros((1 << 23, words["bls24315"]), dtype=np.uint64), "bls24315")
    L = import_module("gnark-crypto_b200._native").lib()
    for cname in ("bn254_g2", "bls12381_g2", "bls12377_g2", "bw6761_g2", "bw6633_g2", "secp256k1_g1"):
        cid = mx.CURVES[cname]
        assert L.gmsm_g1_to_lagrange_workspace_bytes(cid, 4) == 0
        pts = np.zeros((4, 2 * curves.GROUPS[cname].words), dtype=np.uint64)
        with pytest.raises(mx.MultiExpError, match="pairing curves only"):
            kzg.ToLagrangeG1(pts, cname)


def test_torch_inputs_in_place_and_streams():
    """a tensor input is left unmodified and the result stays on its device; d_out == d_points; the device entry point ordered on
    a non-default stream"""
    import torch

    kzg = _kzg()
    mx = _mx()
    L = import_module("gnark-crypto_b200._native").lib()
    for curve in ("bn254", "bw6761"):
        n = 256
        ks = _special_scalars(curve, n, 5)
        host = _bsm(curve, _gen(curve), ks)
        want = kzg.ToLagrangeG1(host, curve)
        dev = torch.device("cuda", 0)
        t = torch.from_numpy(host.view(np.int64).copy()).to(dev)
        keep = t.clone()
        got = kzg.ToLagrangeG1(t, curve)
        assert got.is_cuda and got.device == t.device and got.shape == t.shape
        assert torch.equal(t, keep)
        assert np.array_equal(got.cpu().numpy().view(np.uint64), want)
        cid = mx.CURVES[curve + "_g1"]
        work = torch.empty(int(L.gmsm_g1_to_lagrange_workspace_bytes(cid, n)) // 8, dtype=torch.int64, device=dev)
        s = torch.cuda.Stream(dev)
        x = keep.clone()
        torch.cuda.current_stream(dev).synchronize()
        with torch.cuda.stream(s):
            mx._check(L.gmsm_g1_to_lagrange_device(cid, x.data_ptr(), n, x.data_ptr(), work.data_ptr(), s.cuda_stream))
        s.synchronize()
        assert np.array_equal(x.cpu().numpy().view(np.uint64), want)
        one = keep[:1].clone()   # n = 1: the identity
        assert torch.equal(kzg.ToLagrangeG1(one, curve), one)


def test_cpp_mirror_to_lagrange():
    exe = os.path.join(LIBDIR, "build", "lagrange_test")
    os.makedirs(os.path.dirname(exe), exist_ok=True)
    cuda_lib = "/usr/local/cuda/lib64"
    subprocess.run(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "lagrange_test.cpp"),
                    "-o", exe, "-L", LIBDIR, "-lgmsm", "-L", cuda_lib, "-lcudart", "-Wl,-rpath," + LIBDIR, "-Wl,-rpath," + cuda_lib],
                   check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "LAGRANGE_OK" in r.stdout, r.stdout + r.stderr
