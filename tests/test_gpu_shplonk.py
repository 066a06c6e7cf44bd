"""SHPLONK / FFLONK on the device: gmsm_fr_poly_lincomb_device against a big-integer restatement for all seven scalar fields and its
rejected arguments; shplonk.BatchOpen, fflonk.BatchOpen and fflonk.FoldAndCommit bit-identical to the line-by-line restatement of
the reference (shplonk.batch_open_host) at small sizes, and checked by BatchVerify in the exponent with a known-alpha SRS at 2^16
(all curves) and 2^20 (bn254, bw6-761)."""
import ctypes
import hashlib
import random
from importlib import import_module

import numpy as np
import pytest

from oracle import oracle as O
from tests import shplonk_ref as ref
from tests.test_emu_lincomb_cpu import cases as lincomb_cases
from tests.test_emu_lincomb_cpu import lincomb_ref

curves = import_module("gnark-crypto_b200.curves")

pytestmark = pytest.mark.gpu
CURVES = ["bn254", "bls12381", "bls12377", "bls24315", "bls24317", "bw6633", "bw6761"]
FIELD = {c: i for i, c in enumerate(CURVES)}


def _mods():
    return import_module("gnark-crypto_b200.kzg"), import_module("gnark-crypto_b200.shplonk"), import_module("gnark-crypto_b200.fflonk")


def _torch():
    return import_module("torch")


def _dev(a):
    return _torch().from_numpy(np.ascontiguousarray(a, dtype=np.uint64).view(np.int64).reshape(-1).copy()).cuda()


def _host(t, w):
    return t.cpu().numpy().view(np.uint64).reshape(-1, w)


def _lincomb(c, d_polys, lens, scalars, strides, offsets, d_out, out_len, accumulate):
    kzg = _mods()[0]
    nat = import_module("gnark-crypto_b200._native")
    r = kzg.CURVE_PARAMS[c].r
    ptrs = (ctypes.c_void_p * len(d_polys))(*[d.data_ptr() if d is not None else None for d in d_polys])
    ln, st, off = (np.array(v, dtype=np.uint64) for v in (lens, strides, offsets))
    sc = scalars if isinstance(scalars, np.ndarray) else curves._fr_encode(scalars, r)
    return nat.lib().gmsm_fr_poly_lincomb_device(FIELD[c], ptrs, ln.ctypes.data, sc.ctypes.data, st.ctypes.data, off.ctypes.data,
                                                  len(d_polys), d_out.data_ptr() if d_out is not None else None, out_len,
                                                  accumulate, _torch().cuda.current_stream().cuda_stream)


@pytest.mark.parametrize("c", CURVES)
def test_abi_lincomb(c):
    """strides 1, 2, 3, 9 with offsets, lengths 1 and (8 x 256) +- 1, eleven inputs, scalars 0, 1, r - 1, accumulate, an output
    shorter than the inputs reach; the inputs are left unchanged"""
    kzg = _mods()[0]
    torch = _torch()
    cp = kzg.CURVE_PARAMS[c]
    r, w = cp.r, cp.fr_words
    rng = random.Random(61 + FIELD[c])
    for lens, scalars, strides, offsets, out_len in lincomb_cases(r, rng) + [([70000, 3], [rng.randrange(r), 1], [3, 1], [2, 0], 210003)]:
        polys = [[rng.randrange(r) for _ in range(m)] for m in lens]
        enc = [curves._fr_encode(p, r) for p in polys]
        d_polys = [_dev(e) for e in enc]
        for init in (None, [rng.randrange(r) for _ in range(out_len)]):
            d_out = _dev(curves._fr_encode(init, r)) if init else torch.full((out_len * w,), -1, dtype=torch.int64, device="cuda")
            assert _lincomb(c, d_polys, lens, scalars, strides, offsets, d_out, out_len, 1 if init else 0) == 0
            want = lincomb_ref(polys, scalars, strides, offsets, out_len, r, init)
            assert np.array_equal(_host(d_out, w), curves._fr_encode(want, r)), (lens, strides, offsets)
        assert all(np.array_equal(_host(d, w), e) for d, e in zip(d_polys, enc))


def test_abi_lincomb_rejects_bad_arguments():
    kzg = _mods()[0]
    torch = _torch()
    nat = import_module("gnark-crypto_b200._native")
    r = kzg.CURVE_PARAMS["bn254"].r
    d_f = _dev(curves._fr_encode(list(range(1, 100)), r))
    d_out = torch.zeros(400, dtype=torch.int64, device="cuda")
    ok = dict(lens=[99], scalars=[3], strides=[1], offsets=[0])

    def call(c="bn254", polys=(d_f,), out=d_out, out_len=100, **kw):
        a = dict(ok)
        a.update(kw)
        return _lincomb(c, list(polys), a["lens"], a["scalars"], a["strides"], a["offsets"], out, out_len, 0)

    assert call() == 0
    assert _lincomb("bn254", [d_f], [99], [3], [1], [0], d_out, 100, 0) == 0
    nat_fail = [
        (lambda: _lincomb_field(9), "unknown scalar field"),
        (lambda: _lincomb("bn254", [], [], np.zeros((0, 4), dtype=np.uint64), [], [], d_out, 100, 0), "nothing to combine"),
        (lambda: call(out_len=0), "nothing to combine"),
        (lambda: call(strides=[0]), "stride of polynomial 0 is 0"),
        (lambda: call(scalars=np.array([[0xFFFFFFFFFFFFFFFF] * 4], dtype=np.uint64)), "not a reduced fr.Element"),
        (lambda: call(out=d_f, out_len=10), "overlaps the output"),
        (lambda: _lincomb("bn254", [d_f], [99], [3], [1], [0], _Ptr(d_f.data_ptr() + 98 * 32), 5, 0), "overlaps the output"),
        (lambda: call(polys=(None,)), "polynomial 0 is null"),
        (lambda: call(out=None), "null argument"),
    ]

    def _lincomb_field(f):
        ptrs = (ctypes.c_void_p * 1)(d_f.data_ptr())
        ln = np.array([99], dtype=np.uint64)
        one = np.array([1], dtype=np.uint64)
        sc = curves._fr_encode([3], r)
        return nat.lib().gmsm_fr_poly_lincomb_device(f, ptrs, ln.ctypes.data, sc.ctypes.data, one.ctypes.data, one.ctypes.data, 1,
                                                      d_out.data_ptr(), 100, 0, None)

    for fn, text in nat_fail:
        assert fn() == nat.GMSM_EINVAL, text
        assert text in nat.last_error(), (text, nat.last_error())
    torch.cuda.synchronize()


class _Ptr:
    def __init__(self, p):
        self.p = p

    def data_ptr(self):
        return self.p


def _pk(c, size, alpha, window_tables=False):
    kzg = _mods()[0]
    G = O.GROUPS[c + "_g1"]
    gen = G.encode_affine([G.gen])[0]
    srs = kzg.new_srs_g1(c, size, alpha, gen, kzg.CURVE_PARAMS[c].r, G.encode_scalars)
    return kzg.ProvingKey(c, srs, window_tables=window_tables)


def _rand_limbs(n, c, seed):
    """n reduced fr.Elements as limbs: uniform below 2^(bits(r) - 1) < r"""
    cp = _mods()[0].CURVE_PARAMS[c]
    rng = np.random.default_rng(seed)
    a = rng.integers(0, 2**63, size=(n, cp.fr_words), dtype=np.uint64) * 2 + rng.integers(0, 2, size=(n, cp.fr_words), dtype=np.uint64)
    top = (cp.r.bit_length() - 1) - 64 * (cp.fr_words - 1)
    a[:, -1] &= np.uint64((1 << top) - 1)
    return a


def _points_enc(c, sets):
    kzg = _mods()[0]
    r = kzg.CURVE_PARAMS[c].r
    return [curves._fr_encode(S, r).reshape(-1, kzg.CURVE_PARAMS[c].fr_words) for S in sets]


def _host_shplonk(c, pk, polys_limbs, sets, digests, hf, *data):
    kzg, shplonk, _ = _mods()
    r = kzg.CURVE_PARAMS[c].r
    polys = [curves._fr_decode(p, r) for p in polys_limbs]
    return shplonk.batch_open_host(polys, sets, digests, hf, c, shplonk._host_commit(pk), *data)


def _assert_proof(proof, want, c):
    kzg = _mods()[0]
    r = kzg.CURVE_PARAMS[c].r
    assert np.array_equal(proof.W, want[0]) and np.array_equal(proof.WPrime, want[1])
    assert [curves._fr_decode(v, r) if len(v) else [] for v in proof.ClaimedValues] == want[2]


@pytest.mark.parametrize("c", CURVES)
def test_shplonk_fflonk_small_equal_host(c):
    """device == host restatement: SHPLONK (ζ, ζω-style sets, a repeated point across sets, an empty set, a short polynomial, a
    point repeated inside one set) and FFLONK (packs of 1, 2, 3 and 5), sha256 and blake2b, with and without data transcript"""
    kzg, shplonk, fflonk = _mods()
    r = kzg.CURVE_PARAMS[c].r
    rng = random.Random(7 + FIELD[c])
    pk = _pk(c, 300, rng.randrange(r))
    z1, z2, z3 = (rng.randrange(r) for _ in range(3))
    polys = [_rand_limbs(n, c, 10 * FIELD[c] + k) for k, n in enumerate((257, 100, 3, 1, 200))]
    digests = [kzg.Commit(p, pk) for p in polys]
    for sets, hf, data in (([[z1], [z1, z2], [], [z3, z1], [z2]], hashlib.sha256, (b"transcript", b"more")),
                           ([[z1, z2, z3], [z2], [z1], [z1, z2], [z1, z1]], hashlib.blake2b, ())):
        proof = shplonk.BatchOpen(polys, digests, _points_enc(c, sets), hf, pk, *data)
        _assert_proof(proof, _host_shplonk(c, pk, polys, sets, digests, hf, *data), c)
    packs = [[_rand_limbs(n, c, 1000 + 10 * FIELD[c] + k) for k, n in enumerate(ns)] for ns in ([60], [50, 41], [9, 30, 1], [7, 8, 9, 10, 11])]
    sets = [[z1], [z2, z3], [z1, z2], [z3]]
    dig = [fflonk.FoldAndCommit(pk_, pk) for pk_ in packs]
    for pk_, d in zip(packs, dig):
        assert np.array_equal(d, kzg.Commit(fflonk.Fold(pk_, c), pk))
    for hf, data in ((hashlib.sha256, (b"fflonk",)), (hashlib.blake2b, ())):
        proof = fflonk.BatchOpen(packs, dig, _points_enc(c, sets), hf, pk, *data)
        ts = [fflonk._next_divisor_r_minus_one(len(p), r) for p in packs]
        ext = [fflonk._extend_set(S, t, c) for S, t in zip(sets, ts)]
        folded = [fflonk.Fold(p, c) for p in packs]
        _assert_proof(proof.SOpeningProof, _host_shplonk(c, pk, folded, ext, dig, hf, *data), c)
        outer = [[curves._fr_decode(v, r) for v in vals] for vals in proof.ClaimedValues]
        assert ref.fflonk_fold_consistent(outer, [curves._fr_decode(v, r) for v in proof.SOpeningProof.ClaimedValues], sets, c)
        for vals, pack, S, t in zip(outer, packs, sets, ts):
            assert len(vals) == t
            for i, p in enumerate(pack):
                assert vals[i] == [shplonk._eval(curves._fr_decode(p, r), pow(s, t, r), r) for s in S]
    pk.close()


def _verify(c, pk_alpha, polys, sets, proof, digests, hf, *data):
    kzg = _mods()[0]
    r = kzg.CURVE_PARAMS[c].r
    claimed = [curves._fr_decode(v, r) if len(v) else [] for v in proof.ClaimedValues]
    return ref.verify_in_exponent(polys, sets, proof.W, proof.WPrime, claimed, digests, hf, c, pk_alpha, *data)


@pytest.mark.parametrize("c,logn", [(c, 16) for c in CURVES] + [("bn254", 20), ("bw6761", 20)])
def test_verify_in_exponent(c, logn):
    """PLONK-style openings at {ζ} and {ζ, ζω}, and FFLONK packs of 3 at {ζ} and 2 at {ζ, ζ'}, pass BatchVerify in the exponent;
    a tampered claimed value fails it.  Device tensors are left unmodified."""
    kzg, shplonk, fflonk = _mods()
    torch = _torch()
    r = kzg.CURVE_PARAMS[c].r
    n = 1 << logn
    rng = random.Random(logn * 31 + FIELD[c])
    alpha = rng.randrange(r)
    pk = _pk(c, n + 8, alpha)
    zeta, omega = rng.randrange(r), fflonk._ith_root_one(2, c)
    polys = [_dev(_rand_limbs(n, c, 7 * logn + k)) for k in range(3)]
    keep = [p.clone() for p in polys]
    digests = [kzg.Commit(p, pk) for p in polys]
    sets = [[zeta], [zeta], [zeta, zeta * omega % r]]
    proof = shplonk.BatchOpen(polys, digests, _points_enc(c, sets), hashlib.sha256, pk, b"plonk")
    assert _verify(c, alpha, None, sets, proof, digests, hashlib.sha256, b"plonk")
    proof.ClaimedValues[2] = proof.ClaimedValues[2].copy()
    proof.ClaimedValues[2][1] = curves._fr_encode([(curves._fr_decode(proof.ClaimedValues[2][1:2], r)[0] + 1) % r], r)[0]
    assert not _verify(c, alpha, None, sets, proof, digests, hashlib.sha256, b"plonk")
    m = n // 4
    w = kzg.CURVE_PARAMS[c].fr_words
    packs = [[p[:m * w] for p in polys], [polys[0][:m * w], polys[1][:16 * w]]]
    dig = [fflonk.FoldAndCommit(p, pk) for p in packs]
    fsets = [[zeta], [zeta, rng.randrange(r)]]
    fp = fflonk.BatchOpen(packs, dig, _points_enc(c, fsets), hashlib.blake2b, pk)
    ts = [fflonk._next_divisor_r_minus_one(len(p), r) for p in packs]
    ext = [fflonk._extend_set(S, t, c) for S, t in zip(fsets, ts)]
    assert _verify(c, alpha, None, ext, fp.SOpeningProof, dig, hashlib.blake2b)
    outer = [[curves._fr_decode(v, r) for v in vals] for vals in fp.ClaimedValues]
    assert ref.fflonk_fold_consistent(outer, [curves._fr_decode(v, r) for v in fp.SOpeningProof.ClaimedValues], fsets, c)
    assert all(torch.equal(a, b) for a, b in zip(polys, keep))
    pk.close()


def test_device_path_taken_window_tables_and_errors(monkeypatch):
    kzg, shplonk, fflonk = _mods()
    c = "bls12377"
    r = kzg.CURVE_PARAMS[c].r
    rng = random.Random(5)
    alpha = rng.randrange(r)
    pk = _pk(c, 4096, alpha)
    pkw = _pk(c, 4096, alpha, window_tables=True)
    polys = [_rand_limbs(n, c, 90 + n) for n in (4096, 1000, 17)]
    digests = [kzg.Commit(p, pk) for p in polys]
    sets = [[rng.randrange(r)], [rng.randrange(r), rng.randrange(r)], []]
    pts = _points_enc(c, sets)
    small = [polys[0][:4094], polys[1], polys[2]]
    sdig = [kzg.Commit(p, pk) for p in small]
    want = _host_shplonk(c, pk, small, sets, sdig, hashlib.sha256)
    fwant = fflonk.BatchOpen([polys[1:]], [fflonk.FoldAndCommit(polys[1:], pk)], pts[1:2], hashlib.sha256, pk)

    def boom(*a, **k):
        raise AssertionError("host restatement called")

    monkeypatch.setattr(shplonk, "batch_open_host", boom)
    monkeypatch.setattr(shplonk, "_div", boom)
    monkeypatch.setattr(shplonk, "_mul", boom)
    with pytest.raises(kzg.ErrInvalidPolynomialSize):       # W fits (4096), W' does not (4096 + 3 - 1)
        shplonk.BatchOpen(polys, digests, pts, hashlib.sha256, pk)
    for key in (pk, pkw):
        proof = shplonk.BatchOpen(small, sdig, pts, hashlib.sha256, key)
        _assert_proof(proof, want, c)
        assert _verify(c, alpha, None, sets, proof, sdig, hashlib.sha256)
    proof_t = shplonk.BatchOpen([_dev(p) for p in small], sdig, pts, hashlib.sha256, pkw)
    assert np.array_equal(proof_t.W, proof.W) and np.array_equal(proof_t.WPrime, proof.WPrime)
    fp = fflonk.BatchOpen([polys[1:]], [fflonk.FoldAndCommit(polys[1:], pkw)], pts[1:2], hashlib.sha256, pkw)
    assert np.array_equal(fp.SOpeningProof.W, fwant.SOpeningProof.W) and np.array_equal(fp.SOpeningProof.WPrime, fwant.SOpeningProof.WPrime)
    monkeypatch.undo()
    with pytest.raises(shplonk.ErrInvalidNumberOfPoints, match="number of digests should be equal to the number of points"):
        shplonk.BatchOpen(polys, digests, pts[:2], hashlib.sha256, pk)
    with pytest.raises(shplonk.ErrInvalidNumberOfDigests, match="number of digests should be equal to the number of polynomials"):
        shplonk.BatchOpen(polys, digests[:2], pts, hashlib.sha256, pk)
    with pytest.raises(ValueError):
        shplonk.BatchOpen([], [], [], hashlib.sha256, pk)
    with pytest.raises(kzg.ErrInvalidPolynomialSize, match="larger than SRS"):
        shplonk.BatchOpen([_rand_limbs(4097, c, 1)], digests[:1], pts[:1], hashlib.sha256, pk)
    with pytest.raises(fflonk.ErrNbPolynomialsNbPoints):
        fflonk.BatchOpen([polys[1:]], [digests[0]], pts[:2], hashlib.sha256, pk)
    with pytest.raises(kzg.ErrInvalidPolynomialSize):
        fflonk.FoldAndCommit([polys[0], polys[1]], pk)            # t * 4096 > 4096
    pk.close()
    pkw.close()
