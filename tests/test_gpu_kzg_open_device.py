"""KZG opening on the device: gmsm_fr_poly_div_x_minus_a_device / gmsm_fr_poly_fold_device against the host reference of kzg.py
(`_eval`, `_divide_by_x_minus_a`) for all seven scalar fields, closed forms at 2^22 / 2^20 coefficients, and kzg.Open /
BatchOpenSinglePoint / FoldProof / Commit on all seven curves, checked in the exponent with a test SRS of known alpha and against
the host path they replace."""
import ctypes
import hashlib
import random
from importlib import import_module

import numpy as np
import pytest

from oracle import cref
from oracle import oracle as O

curves = import_module("gnark-crypto_b200.curves")

pytestmark = pytest.mark.gpu
CURVES = ["bn254", "bls12381", "bls12377", "bls24315", "bls24317", "bw6633", "bw6761"]
FIELD = {c: i for i, c in enumerate(CURVES)}      # GMSM_FR_*
TILE = {32: 1024, 40: 1024, 48: 512}              # coefficients per block in fft.cu, by fr.Bytes


def _kzg():
    return import_module("gnark-crypto_b200.kzg")


def _lib():
    return import_module("gnark-crypto_b200._native").lib()


def _torch():
    return import_module("torch")


def _dev(a: np.ndarray):
    torch = _torch()
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint64).view(np.int64).reshape(-1).copy()).cuda()


def _host(t, w):
    return t.cpu().numpy().view(np.uint64).reshape(-1, w)


def _div(c, d_f, n, a_limbs, quotient=True):
    """(f(a) limbs, quotient limbs or None) through the C ABI; workspace sized by gmsm_fr_poly_workspace_bytes"""
    torch = _torch()
    L = _lib()
    w = _kzg().CURVE_PARAMS[c].fr_words
    d_h = torch.empty(max(n - 1, 1) * w, dtype=torch.int64, device="cuda") if quotient else None
    d_fa = torch.empty(w, dtype=torch.int64, device="cuda")
    ws = int(L.gmsm_fr_poly_workspace_bytes(FIELD[c], n))
    d_work = torch.empty(max(ws // 8, 1), dtype=torch.int64, device="cuda")
    a_limbs = np.ascontiguousarray(a_limbs, dtype=np.uint64)
    rc = L.gmsm_fr_poly_div_x_minus_a_device(FIELD[c], d_f.data_ptr(), n, a_limbs.ctypes.data, d_h.data_ptr() if quotient else None,
                                             d_fa.data_ptr(), d_work.data_ptr(), torch.cuda.current_stream().cuda_stream)
    assert rc == 0, import_module("gnark-crypto_b200._native").last_error()
    return _host(d_fa, w)[0], (_host(d_h, w)[:n - 1] if quotient else None)


@pytest.mark.parametrize("c", CURVES)
def test_abi_divide_and_evaluate(c):
    """full outputs against the host reference: lengths 1, 2, 3, T - 1, T, T + 1, 3T + 5 and 2^16 (two carry levels), a in
    {0, 1, r - 1, random}, random and all-(r - 1) coefficients; the polynomial is unchanged and evaluation only gives the same f(a)"""
    kzg = _kzg()
    cp = kzg.CURVE_PARAMS[c]
    r, t = cp.r, TILE[cp.fr_bytes]
    rng = random.Random(3 + FIELD[c])
    cases = [[rng.randrange(r) for _ in range(n)] for n in (1, 2, 3, t - 1, t, t + 1, 3 * t + 5, 1 << 16)]
    cases.append([r - 1] * (t + 3))
    for coeffs in cases:
        n = len(coeffs)
        f = curves._fr_encode(coeffs, r)
        d_f = _dev(f)
        for a in (0, 1, r - 1, rng.randrange(r)):
            a_limbs = curves._fr_encode([a], r)[0]
            fa, h = _div(c, d_f, n, a_limbs)
            want = kzg._eval(coeffs, a, r)
            assert np.array_equal(fa, curves._fr_encode([want], r)[0]), (n, a)
            assert np.array_equal(h, curves._fr_encode(kzg._divide_by_x_minus_a(coeffs, want, a, r), r).reshape(-1, cp.fr_words)), (n, a)
            fa_only, _ = _div(c, d_f, n, a_limbs, quotient=False)
            assert np.array_equal(fa_only, fa), (n, a)
        assert np.array_equal(_host(d_f, cp.fr_words), f)


@pytest.mark.parametrize("c", CURVES)
def test_abi_fold(c):
    """out[j] = sum_i gamma^i f_i[j]: unequal lengths with a length-1 polynomial, k = 1, gamma = 0, k = 11 (more than one batch)"""
    kzg = _kzg()
    r = kzg.CURVE_PARAMS[c].r
    torch = _torch()
    rng = random.Random(5 + FIELD[c])
    for lens, gamma in (([3000, 17, 1, 1025], rng.randrange(r)), ([513], rng.randrange(r)), ([40, 900], 0),
                        ([33, 7, 1, 50, 2, 9, 64, 1, 12, 70, 5], r - 1)):
        polys = [[rng.randrange(r) for _ in range(m)] for m in lens]
        d_polys = [_dev(curves._fr_encode(p, r)) for p in polys]
        out_len = max(lens)
        w = kzg.CURVE_PARAMS[c].fr_words
        d_out = torch.full((out_len * w,), -1, dtype=torch.int64, device="cuda")
        ptrs = (ctypes.c_void_p * len(polys))(*[d.data_ptr() for d in d_polys])
        ln = np.array(lens, dtype=np.uint64)
        g = curves._fr_encode([gamma], r)[0]
        rc = _lib().gmsm_fr_poly_fold_device(FIELD[c], ptrs, ln.ctypes.data, len(polys), g.ctypes.data, d_out.data_ptr(), out_len,
                                             torch.cuda.current_stream().cuda_stream)
        assert rc == 0
        want = [0] * out_len
        for i, p in enumerate(polys):
            gi = pow(gamma, i, r)
            for j, v in enumerate(p):
                want[j] = (want[j] + gi * v) % r
        assert np.array_equal(_host(d_out, w), curves._fr_encode(want, r)), (lens, gamma)


def test_abi_rejects_bad_arguments():
    kzg = _kzg()
    torch = _torch()
    L = _lib()
    nat = import_module("gnark-crypto_b200._native")
    r = kzg.CURVE_PARAMS["bn254"].r
    d_f = _dev(curves._fr_encode(list(range(1, 100)), r))
    d_fa = torch.empty(4, dtype=torch.int64, device="cuda")
    a = curves._fr_encode([7], r)[0]
    assert L.gmsm_fr_poly_div_x_minus_a_device(0, d_f.data_ptr(), 0, a.ctypes.data, None, d_fa.data_ptr(), None, None) == nat.GMSM_EINVAL
    assert "n = 0" in nat.last_error()
    assert L.gmsm_fr_poly_div_x_minus_a_device(9, d_f.data_ptr(), 99, a.ctypes.data, None, d_fa.data_ptr(), None, None) == nat.GMSM_EINVAL
    assert "unknown scalar field" in nat.last_error()
    assert L.gmsm_fr_poly_div_x_minus_a_device(0, d_f.data_ptr(), 99, a.ctypes.data, d_f.data_ptr() + 32, d_fa.data_ptr(), None,
                                               None) == nat.GMSM_EINVAL
    assert "overlap" in nat.last_error()
    big = np.array([0xFFFFFFFFFFFFFFFF] * 4, dtype=np.uint64)
    assert L.gmsm_fr_poly_div_x_minus_a_device(0, d_f.data_ptr(), 99, big.ctypes.data, None, d_fa.data_ptr(), None, None) == nat.GMSM_EINVAL
    assert L.gmsm_fr_poly_workspace_bytes(9, 1000) == 0 and L.gmsm_fr_poly_workspace_bytes(0, 1024) == 0
    assert L.gmsm_fr_poly_workspace_bytes(0, 1025) == 2 * 32
    ptrs = (ctypes.c_void_p * 1)(d_f.data_ptr())
    ln = np.array([99], dtype=np.uint64)
    assert L.gmsm_fr_poly_fold_device(0, ptrs, ln.ctypes.data, 0, a.ctypes.data, d_fa.data_ptr(), 1, None) == nat.GMSM_EINVAL


@pytest.mark.parametrize("c,n", [("bn254", (1 << 22) + 3), ("bw6761", (1 << 20) + 5)])
def test_large_closed_form(c, n):
    """f = all ones: f(a) = (a^n - 1) / (a - 1), h[i] = (a^(n-1-i) - 1) / (a - 1) at 256 indices: 0, n - 2, the tile and carry-level
    boundaries and random ones"""
    kzg = _kzg()
    torch = _torch()
    cp = kzg.CURVE_PARAMS[c]
    r, w, t = cp.r, cp.fr_words, TILE[cp.fr_bytes]
    one = torch.from_numpy(curves._fr_encode([1], r)[0].view(np.int64).copy()).cuda()
    d_f = one.repeat(n)
    a = 0x1234567890ABCDEF1234567 % r
    fa, h = _div(c, d_f, n, curves._fr_encode([a], r)[0])
    inv = pow(a - 1, -1, r)
    assert np.array_equal(fa, curves._fr_encode([(pow(a, n, r) - 1) * inv % r], r)[0])
    rng = random.Random(n)
    idx = {0, n - 2, 1, t - 2, t - 1, t, t * t - 1, t * t, t * t - 2}
    for k in range(1, 40):
        idx |= {min(k * t * 97 + e, n - 2) for e in (-1, 0)}
    while len(idx) < 256:
        idx.add(rng.randrange(n - 1))
    idx = sorted(idx)
    want = curves._fr_encode([(pow(a, n - 1 - i, r) - 1) * inv % r for i in idx], r)
    assert np.array_equal(h[idx], want)
    fa_only, _ = _div(c, d_f, n, curves._fr_encode([a], r)[0], quotient=False)
    assert np.array_equal(fa_only, fa)
    assert bool((d_f.view(-1, w) == one).all())


def _srs_pk(c, size, alpha, window_tables=False):
    kzg = _kzg()
    G = O.GROUPS[c + "_g1"]
    gen = G.encode_affine([G.gen])[0]
    return kzg.ProvingKey(c, kzg.new_srs_g1(c, size, alpha, gen, kzg.CURVE_PARAMS[c].r, G.encode_scalars), window_tables=window_tables), gen


def _ev(p, x, r):
    acc = 0
    for v in reversed(p):
        acc = (acc * x + v) % r
    return acc


def _check_open(c, pk, gen, alpha, coeffs, a):
    kzg = _kzg()
    g = c + "_g1"
    G = O.GROUPS[g]
    r = kzg.CURVE_PARAMS[c].r
    enc = G.encode_scalars(coeffs)
    point = G.encode_scalars([a])[0]
    op = kzg.Open(enc, point, pk)
    fa = _ev(coeffs, a, r)
    assert np.array_equal(op.ClaimedValue, G.encode_scalars([fa])[0])
    assert np.array_equal(op.H, cref.scalar_mul(g, gen, (_ev(coeffs, alpha, r) - fa) * pow(alpha - a, -1, r) % r))
    # the host path this replaces, on the same inputs
    h = kzg._divide_by_x_minus_a(coeffs, fa, a, r)
    assert np.array_equal(op.H, kzg.Commit(curves._fr_encode(h, r), pk))
    return op


@pytest.mark.parametrize("c", CURVES)
def test_open_all_curves(c):
    kzg = _kzg()
    r = kzg.CURVE_PARAMS[c].r
    alpha = 0x7654321FEDCBA9876543 % r
    pk, gen = _srs_pk(c, 3000, alpha)
    rng = random.Random(FIELD[c])
    for n in (2, 3, 700, 1025, 3000):
        _check_open(c, pk, gen, alpha, [rng.randrange(r) for _ in range(n)], rng.randrange(r))
    _check_open(c, pk, gen, alpha, [r - 1] * 1500, r - 1)
    pk.close()


def test_open_bn254_2_20_and_window_tables():
    kzg = _kzg()
    r = kzg.CURVE_PARAMS["bn254"].r
    n = 1 << 20
    alpha = 0xC0FFEE12345 % r
    rng = random.Random(20)
    coeffs = [rng.randrange(r) for _ in range(n)]
    a = rng.randrange(r)
    pk, gen = _srs_pk("bn254", n, alpha)
    op = _check_open("bn254", pk, gen, alpha, coeffs, a)
    pk.close()
    pk, gen = _srs_pk("bn254", 4096, alpha, window_tables=True)
    _check_open("bn254", pk, gen, alpha, coeffs[:4096], a)
    pk.close()
    assert op.H.shape == (8,)


def _gamma(c, a, digests, claimed, extra):
    cp = _kzg().CURVE_PARAMS[c]
    G = O.GROUPS[c + "_g1"]
    h = hashlib.sha256()
    h.update(b"gamma")
    h.update(a.to_bytes(cp.fr_bytes, "big"))
    for d in digests:
        x, y = G.decode_affine(d.reshape(1, -1))[0]
        h.update(int(x).to_bytes(cp.fp_bytes, "big") + int(y).to_bytes(cp.fp_bytes, "big"))
    for v in claimed:
        h.update(v.to_bytes(cp.fr_bytes, "big"))
    h.update(extra)
    return int.from_bytes(h.digest(), "big") % cp.r


@pytest.mark.parametrize("c", CURVES)
def test_batch_open_and_fold_all_curves(c):
    """mixed lengths including a length-1 polynomial; gamma re-derived here; H and the folded digest checked in the exponent"""
    kzg = _kzg()
    g = c + "_g1"
    G = O.GROUPS[g]
    r = kzg.CURVE_PARAMS[c].r
    alpha = 0x1EADBEEF0123 % r
    pk, gen = _srs_pk(c, 2100, alpha)
    rng = random.Random(40 + FIELD[c])
    polys = [[rng.randrange(r) for _ in range(m)] for m in (2100, 513, 1, 1024, 64)]
    polys[0][7] = r - 1
    enc = [G.encode_scalars(p) for p in polys]
    digests = [kzg.Commit(e, pk) for e in enc]
    a = rng.randrange(r)
    point = G.encode_scalars([a])[0]
    extra = b"device-open"
    proof = kzg.BatchOpenSinglePoint(enc, digests, point, hashlib.sha256, pk, extra)
    claimed = [_ev(p, a, r) for p in polys]
    assert np.array_equal(proof.ClaimedValues, G.encode_scalars(claimed))
    gamma = _gamma(c, a, digests, claimed, extra)
    fold_alpha = sum(pow(gamma, i, r) * _ev(p, alpha, r) for i, p in enumerate(polys)) % r
    fold_a = sum(pow(gamma, i, r) * v for i, v in enumerate(claimed)) % r
    assert np.array_equal(proof.H, cref.scalar_mul(g, gen, (fold_alpha - fold_a) * pow(alpha - a, -1, r) % r))
    op, folded = kzg.FoldProof(digests, proof, point, hashlib.sha256, c, extra)
    assert np.array_equal(folded, cref.scalar_mul(g, gen, fold_alpha))
    assert np.array_equal(op.ClaimedValue, G.encode_scalars([fold_a])[0]) and np.array_equal(op.H, proof.H)
    # a batch of constant polynomials has an empty folded quotient: the reference's Commit error
    with pytest.raises(kzg.ErrInvalidPolynomialSize):
        kzg.BatchOpenSinglePoint([enc[2], enc[2]], digests[2:3] * 2, point, hashlib.sha256, pk)
    pk.close()


def test_device_path_is_taken(monkeypatch):
    """with the host reference disabled, Open and BatchOpenSinglePoint still succeed on a single-device proving key"""
    kzg = _kzg()
    G = O.GROUPS["bls12381_g1"]
    r = kzg.CURVE_PARAMS["bls12381"].r
    alpha = 0x5151 % r
    pk, gen = _srs_pk("bls12381", 600, alpha)
    rng = random.Random(9)
    polys = [[rng.randrange(r) for _ in range(m)] for m in (600, 100)]
    enc = [G.encode_scalars(p) for p in polys]
    digests = [kzg.Commit(e, pk) for e in enc]
    a = rng.randrange(r)
    point = G.encode_scalars([a])[0]
    want_open = kzg.Open(enc[0], point, pk)
    want_batch = kzg.BatchOpenSinglePoint(enc, digests, point, hashlib.sha256, pk)

    def boom(*args, **kw):
        raise AssertionError("host Fr loop called")

    monkeypatch.setattr(kzg, "_eval", boom)
    monkeypatch.setattr(kzg, "_divide_by_x_minus_a", boom)
    op = kzg.Open(enc[0], point, pk)
    assert np.array_equal(op.H, want_open.H) and np.array_equal(op.ClaimedValue, want_open.ClaimedValue)
    proof = kzg.BatchOpenSinglePoint(enc, digests, point, hashlib.sha256, pk)
    assert np.array_equal(proof.H, want_batch.H) and np.array_equal(proof.ClaimedValues, want_batch.ClaimedValues)
    fa = _ev(polys[0], a, r)
    assert np.array_equal(op.H, cref.scalar_mul("bls12381_g1", gen, (_ev(polys[0], alpha, r) - fa) * pow(alpha - a, -1, r) % r))
    pk.close()


@pytest.mark.parametrize("c", ["bn254", "bw6633", "bw6761"])
def test_torch_tensor_inputs(c):
    """device tensors in fr.Element layout give the same digests and proofs as numpy inputs and are left unmodified; the error
    paths raise the same exceptions"""
    kzg = _kzg()
    torch = _torch()
    G = O.GROUPS[c + "_g1"]
    cp = kzg.CURVE_PARAMS[c]
    r, w = cp.r, cp.fr_words
    pk, _ = _srs_pk(c, 800, 0xABCDEF % r)
    rng = random.Random(77)
    enc = [G.encode_scalars([rng.randrange(r) for _ in range(m)]) for m in (800, 300, 1)]
    dev = [_dev(e) for e in enc]
    keep = [d.clone() for d in dev]
    digests = [kzg.Commit(e, pk) for e in enc]
    assert all(np.array_equal(kzg.Commit(d, pk), want) for d, want in zip(dev, digests))
    point = G.encode_scalars([rng.randrange(r)])[0]
    op_np, op_t = kzg.Open(enc[0], point, pk), kzg.Open(dev[0], point, pk)
    assert np.array_equal(op_np.H, op_t.H) and np.array_equal(op_np.ClaimedValue, op_t.ClaimedValue)
    pr_np = kzg.BatchOpenSinglePoint(enc, digests, point, hashlib.sha256, pk)
    pr_t = kzg.BatchOpenSinglePoint(dev, digests, point, hashlib.sha256, pk)
    pr_mix = kzg.BatchOpenSinglePoint([dev[0], enc[1], dev[2]], digests, point, hashlib.sha256, pk)
    for pr in (pr_t, pr_mix):
        assert np.array_equal(pr.H, pr_np.H) and np.array_equal(pr.ClaimedValues, pr_np.ClaimedValues)
    assert all(torch.equal(d, k) for d, k in zip(dev, keep))
    empty = torch.empty(0, dtype=torch.int64, device="cuda")
    too_big = _dev(G.encode_scalars([1] * 801))
    for bad in (empty, too_big):
        with pytest.raises(kzg.ErrInvalidPolynomialSize):
            kzg.Commit(bad, pk)
        with pytest.raises(kzg.ErrInvalidPolynomialSize):
            kzg.Open(bad, point, pk)
        with pytest.raises(kzg.ErrInvalidPolynomialSize):
            kzg.BatchOpenSinglePoint([dev[1], bad], digests[:2], point, hashlib.sha256, pk)
    with pytest.raises(kzg.ErrInvalidPolynomialSize):
        kzg.Open(dev[2], point, pk)                       # constant polynomial: empty quotient
    with pytest.raises(kzg.ErrInvalidNbDigests):
        kzg.BatchOpenSinglePoint(dev, digests[:2], point, hashlib.sha256, pk)
    assert dev[0].numel() == 800 * w
    pk.close()
