"""permutation.Prove on the device for the seven pairing curves: the new entry points (gmsm_fr_batch_invert_device,
gmsm_fr_permutation_accumulate_device, gmsm_fft_permutation_numerator_device) against the big-int restatements of
tests/permutation_ref.py with their rejected arguments; Prove bit-identical to the line-by-line restatement of permutation.go with
closed-form digests; Verify restated without the pairings on a known-alpha SRS at 2^16 (all curves) and 2^20 (bn254, bw6-761); the
reference's errors; the device path taken on single-device keys; the sharded-key path."""
import random
from importlib import import_module

import numpy as np
import pytest

from oracle import oracle as O
from tests import permutation_ref as ref

curves = import_module("gnark-crypto_b200.curves")

pytestmark = pytest.mark.gpu
CURVES = ["bn254", "bls12381", "bls12377", "bls24315", "bls24317", "bw6633", "bw6761"]
FIELD = {c: i for i, c in enumerate(CURVES)}


def _mods():
    return import_module("gnark-crypto_b200.kzg"), import_module("gnark-crypto_b200.permutation"), import_module("gnark-crypto_b200.fft")


def _nat():
    return import_module("gnark-crypto_b200._native")


def _torch():
    return import_module("torch")


def _dev(a):
    return _torch().from_numpy(np.ascontiguousarray(a, dtype=np.uint64).view(np.int64).reshape(-1).copy()).cuda()


def _host(t, w):
    return t.cpu().numpy().view(np.uint64).reshape(-1, w)


def _enc(vals, c):
    kzg = _mods()[0]
    return curves._fr_encode(vals, kzg.CURVE_PARAMS[c].r)


def _stream():
    return _torch().cuda.current_stream().cuda_stream


def _assert_limbs(got, want_vals, c, what):
    want = _enc(want_vals, c)
    bad = np.nonzero((got != want).any(axis=1))[0]
    assert bad.size == 0, "%s %s: first mismatch at %d of %d" % (c, what, bad[0], len(want_vals))


def _accumulate(c, d_t1, d_t2, n, eps):
    torch = _torch()
    L = _nat().lib()
    w = _mods()[0].CURVE_PARAMS[c].fr_words
    ws = int(L.gmsm_fr_permutation_workspace_bytes(FIELD[c], n))
    work = torch.empty(max(ws // 8, 1), dtype=torch.int64, device="cuda")
    d_z = torch.full((n * w,), -1, dtype=torch.int64, device="cuda")
    e = _enc([eps], c)[0]                  # held for the call: a temporary's buffer could be freed before the library reads it
    rc = L.gmsm_fr_permutation_accumulate_device(FIELD[c], d_t1.data_ptr(), d_t2.data_ptr(), n, e.ctypes.data, d_z.data_ptr(),
                                                 work.data_ptr(), _stream())
    assert rc == 0, _nat().last_error()
    return _host(d_z, w)


@pytest.mark.parametrize("c", CURVES)
def test_abi_batch_invert_and_accumulate(c):
    """BatchInvert with zeros at the start, the end, in a run and everywhere, across tile boundaries and in place; the accumulation
    polynomial at n = 1, 2, 2^10, 2^16 (one and two scan levels; three in test_gpu_perm_stress.py) with random eps and eps forced to a t2[k] and a t1[k]; inputs unchanged"""
    kzg = _mods()[0]
    torch = _torch()
    L = _nat().lib()
    cp = kzg.CURVE_PARAMS[c]
    r, w = cp.r, cp.fr_words
    rng = random.Random(13 + FIELD[c])
    for n in (1, 511, 512, 513, 100003):
        vals = [rng.randrange(1, r) for _ in range(n)]
        for pos in ([], [0], [n - 1], range(n // 3, n // 2 + 1), range(n)):
            v = list(vals)
            for p in pos:
                v[p] = 0
            a = _enc(v, c)
            d_a = _dev(a)
            d_out = torch.full_like(d_a, -1)
            assert L.gmsm_fr_batch_invert_device(FIELD[c], d_a.data_ptr(), n, d_out.data_ptr(), _stream()) == 0
            want = ref.batch_invert(v, r)
            _assert_limbs(_host(d_out, w), want, c, "BatchInvert n=%d" % n)
            assert np.array_equal(_host(d_a, w), a)
            assert L.gmsm_fr_batch_invert_device(FIELD[c], d_a.data_ptr(), n, d_a.data_ptr(), _stream()) == 0     # in place
            _assert_limbs(_host(d_a, w), want, c, "BatchInvert in place n=%d" % n)
    for n in (1, 2, 1 << 10, 1 << 16):
        t1 = [rng.randrange(r) for _ in range(n)]
        t2 = list(t1)
        rng.shuffle(t2)
        a, b = _enc(t1, c), _enc(t2, c)
        d_t1, d_t2 = _dev(a), _dev(b)
        epss = [rng.randrange(r)] + ([t2[n // 3], t1[n - 1]] if n > 1 else [])
        for eps in epss:
            _assert_limbs(_accumulate(c, d_t1, d_t2, n, eps), ref.accumulate(t1, t2, eps, r), c, "accumulate n=%d" % n)
        assert np.array_equal(_host(d_t1, w), a) and np.array_equal(_host(d_t2, w), b)
    torch.cuda.synchronize()


@pytest.mark.parametrize("c", CURVES)
def test_abi_numerator(c):
    """the quotient numerator at n = 1 ... 2^10 and 2^14 against evaluateFirstPartNumReverse / evaluateSecondPartNumReverse and the
    omega-fold; the inputs are left unchanged"""
    kzg, _, fft = _mods()
    torch = _torch()
    L = _nat().lib()
    cp = kzg.CURVE_PARAMS[c]
    r, w = cp.r, cp.fr_words
    rng = random.Random(71 + FIELD[c])
    for logn in list(range(0, 11)) + [14]:
        n = 1 << logn
        dom = fft.NewDomain(c, n)
        od = ref.domain(c, n)
        vals = [[rng.randrange(r) for _ in range(n)] for _ in range(3)]
        enc = [_enc(v, c) for v in vals]
        d_in = [_dev(e) for e in enc]
        eps, omega = rng.randrange(r), rng.randrange(r)
        d_out = torch.full_like(d_in[0], -1)
        e, o = _enc([eps], c)[0], _enc([omega], c)[0]
        rc = L.gmsm_fft_permutation_numerator_device(dom._h, *(d.data_ptr() for d in d_in), n, e.ctypes.data, o.ctypes.data,
                                                     d_out.data_ptr(), _stream())
        assert rc == 0, _nat().last_error()
        want = ref.numerator(*vals, eps, omega, n, od.shift, od.generator, r)
        _assert_limbs(_host(d_out, w), want, c, "numerator n=%d" % n)
        assert all(np.array_equal(_host(d, w), e) for d, e in zip(d_in, enc))
        dom.close()
    torch.cuda.synchronize()


def test_abi_rejects_bad_arguments():
    kzg, _, fft = _mods()
    torch = _torch()
    nat = _nat()
    L = nat.lib()
    c = "bn254"
    d_a = _dev(_enc(list(range(1, 65)), c))
    d_b = _dev(_enc(list(range(1, 65)), c))
    d_z = torch.zeros_like(d_a)
    work = torch.zeros(64, dtype=torch.int64, device="cuda")
    eps = _enc([5], c)[0]
    bad = np.array([0xFFFFFFFFFFFFFFFF] * 4, dtype=np.uint64)
    dom = fft.NewDomain(c, 64)

    def acc(field=0, t1=d_a, t2=d_b, n=64, e=eps, z=d_z, wk=work):
        return L.gmsm_fr_permutation_accumulate_device(field, t1.data_ptr() if t1 is not None else None, t2.data_ptr(), n, e.ctypes.data,
                                                       z.data_ptr() if z is not None else None, wk.data_ptr() if wk is not None else None,
                                                       None)

    def num(n=64, e=eps, o=eps, out=d_z, lz=d_b):
        return L.gmsm_fft_permutation_numerator_device(dom._h, d_a.data_ptr(), d_b.data_ptr(), lz.data_ptr(), n, e.ctypes.data, o.ctypes.data,
                                                       out.data_ptr(), None)

    assert acc() == 0 and num() == 0
    cases = [
        (lambda: L.gmsm_fr_batch_invert_device(9, d_a.data_ptr(), 64, d_z.data_ptr(), None), "unknown scalar field"),
        (lambda: L.gmsm_fr_batch_invert_device(0, d_a.data_ptr(), 0, d_z.data_ptr(), None), "n = 0"),
        (lambda: L.gmsm_fr_batch_invert_device(0, d_a.data_ptr(), 64, None, None), "null vector"),
        (lambda: L.gmsm_fr_batch_invert_device(0, d_a.data_ptr(), 64, d_a.data_ptr() + 32, None), "must equal the input or not overlap"),
        (lambda: acc(field=7), "unknown scalar field"),
        (lambda: acc(n=0), "must be a power of 2"),
        (lambda: acc(n=48), "must be a power of 2"),
        (lambda: acc(e=bad), "epsilon is not a reduced fr.Element"),
        (lambda: acc(z=d_a), "must not overlap t1 or t2"),
        (lambda: acc(t1=None), "null vector"),
        (lambda: num(n=32), "must equal the domain cardinality"),
        (lambda: num(e=bad), "epsilon is not a reduced"),
        (lambda: num(o=bad), "omega is not a reduced"),
        (lambda: num(out=d_b), "must not overlap"),
    ]
    for fn, text in cases:
        assert fn() == nat.GMSM_EINVAL, text
        assert text in nat.last_error(), (text, nat.last_error())
    if int(L.gmsm_fr_permutation_workspace_bytes(0, 1 << 12)):
        big = _dev(np.zeros((1 << 12, 4), dtype=np.uint64))
        big2, bz = torch.zeros_like(big), torch.zeros_like(big)
        assert acc(t1=big, t2=big2, n=1 << 12, z=bz, wk=None) == nat.GMSM_EINVAL and "null workspace" in nat.last_error()
    assert L.gmsm_fr_permutation_workspace_bytes(9, 64) == 0
    dom.close()
    torch.cuda.synchronize()


def _pk(c, size, alpha, window_tables=False, device=0):
    kzg = _mods()[0]
    G = O.GROUPS[c + "_g1"]
    gen = G.encode_affine([G.gen])[0]
    srs = kzg.new_srs_g1(c, size, alpha, gen, kzg.CURVE_PARAMS[c].r, G.encode_scalars)
    return kzg.ProvingKey(c, srs, device=device, window_tables=window_tables)


def _rand_perm(c, n, seed):
    """t1 random reduced elements (limbs), t2 a random permutation of its rows"""
    cp = _mods()[0].CURVE_PARAMS[c]
    rng = np.random.default_rng(seed)
    a = rng.integers(0, 2**63, size=(n, cp.fr_words), dtype=np.uint64) * 2 + rng.integers(0, 2, size=(n, cp.fr_words), dtype=np.uint64)
    top = (cp.r.bit_length() - 1) - 64 * (cp.fr_words - 1)
    a[:, -1] &= np.uint64((1 << top) - 1)
    return a, np.ascontiguousarray(a[rng.permutation(n)])


def _reference_vectors(c):
    """permutation_test.go: a[i] = 4i + 1, b[i] = a[5i mod 8]"""
    a = [4 * i + 1 for i in range(8)]
    return _enc(a, c), _enc([a[(5 * i) % 8] for i in range(8)], c)


def _assert_equal_ref(proof, want, c):
    kzg = _mods()[0]
    r = kzg.CURVE_PARAMS[c].r
    assert proof.size == want["size"]
    assert curves._fr_decode(proof.g, r)[0] == want["g"]
    for name in ("t1", "t2", "z", "q"):
        assert np.array_equal(proof.__dict__[name], want[name]), name
    assert np.array_equal(proof.batchedProof.H, want["H"])
    assert np.array_equal(proof.batchedProof.ClaimedValues, _enc(want["claimed"], c))
    assert np.array_equal(proof.shiftedProof.H, want["Hs"])
    assert np.array_equal(proof.shiftedProof.ClaimedValue, _enc([want["zs"]], c)[0])


@pytest.mark.parametrize("c", CURVES)
def test_prove_equals_restatement(c):
    """Prove == the line-by-line restatement with closed-form digests: the reference's own vectors, random permutations at n = 2, 4
    and 2^10, host and device inputs (left unchanged), a window-table key"""
    kzg, perm, _ = _mods()
    torch = _torch()
    r = kzg.CURVE_PARAMS[c].r
    rng = random.Random(23 + FIELD[c])
    alpha = rng.randrange(r)
    size = 1 << 10
    pk = _pk(c, size, alpha)
    pkw = _pk(c, size, alpha, window_tables=True)
    srs = ref.ClosedFormSRS(c, size, alpha)
    cases = [_reference_vectors(c)] + [_rand_perm(c, n, 100 * FIELD[c] + n) for n in (2, 4, 1 << 10)]
    for k, (a, b) in enumerate(cases):
        want = ref.prove(c, curves._fr_decode(a, r), curves._fr_decode(b, r), srs)
        keep = (a.copy(), b.copy())
        _assert_equal_ref(perm.Prove(pk, a, b), want, c)
        assert np.array_equal(a, keep[0]) and np.array_equal(b, keep[1])
        d_a, d_b = _dev(a), _dev(b)
        _assert_equal_ref(perm.Prove(pkw if k % 2 else pk, d_a, d_b), want, c)
        assert np.array_equal(_host(d_a, a.shape[1]), a) and np.array_equal(_host(d_b, b.shape[1]), b)
    torch.cuda.synchronize()
    pk.close()
    pkw.close()


@pytest.mark.parametrize("c,logn", [(c, 16) for c in CURVES] + [("bn254", 20), ("bw6761", 20)])
def test_verify_known_alpha(c, logn):
    """a proof of a random permutation passes Verify (restated without the pairings on the known-alpha SRS); with t1[0] replaced by
    a random value, as in the reference's "wrong proof" case, it fails"""
    kzg, perm, _ = _mods()
    r = kzg.CURVE_PARAMS[c].r
    n = 1 << logn
    rng = random.Random(logn * 7 + FIELD[c])
    alpha = rng.randrange(r)
    pk = _pk(c, n, alpha)
    a, b = _rand_perm(c, n, 31 * logn + FIELD[c])
    proof = perm.Prove(pk, _dev(a), _dev(b))
    assert ref.verify(c, proof, alpha)
    a[0] = _enc([rng.randrange(r)], c)[0]
    assert not ref.verify(c, perm.Prove(pk, a, b), alpha)
    pk.close()


def test_errors():
    """mismatched lengths, lengths 0, 3 and 6, n = 1 (the empty quotient of BatchOpenSinglePoint), an SRS shorter than n, a size past
    bw6-633's 2^20 domain"""
    kzg, perm, _ = _mods()
    c = "bn254"
    pk = _pk(c, 16, 12345)
    a, b = _rand_perm(c, 32, 1)
    with pytest.raises(perm.ErrIncompatibleSize, match="^t1 and t2 should be of the same size$"):
        perm.Prove(pk, a[:8], b[:4])
    for n in (0, 3, 6):
        with pytest.raises(perm.ErrSize, match="^t1 and t2 should be of size a power of 2$"):
            perm.Prove(pk, a[:n], b[:n])
    with pytest.raises(kzg.ErrInvalidPolynomialSize, match="larger than SRS or == 0"):
        perm.Prove(pk, a[:1], a[:1])
    with pytest.raises(kzg.ErrInvalidPolynomialSize, match="larger than SRS or == 0"):
        perm.Prove(pk, a, b)                                   # n = 32 > 16 points
    pk.close()
    pk6 = _pk("bw6633", 4, 3)
    big = np.zeros((1 << 21, 5), dtype=np.uint64)
    with pytest.raises(kzg.MultiExpError, match=r"^m \(2097152\) is too big: the required root of unity does not exist$"):
        perm.Prove(pk6, big, big)
    pk6.close()


def test_device_path_taken(monkeypatch):
    """on single-device keys (plain and window tables) no host FFT, host Fr loop or host MultiExp runs"""
    kzg, perm, fft = _mods()
    c = "bls12377"
    r = kzg.CURVE_PARAMS[c].r
    alpha = 987654321
    pk, pkw = _pk(c, 256, alpha), _pk(c, 256, alpha, window_tables=True)
    a, b = _rand_perm(c, 256, 5)
    want = ref.prove(c, curves._fr_decode(a, r), curves._fr_decode(b, r), ref.ClosedFormSRS(c, 256, alpha))

    def boom(*args, **kw):
        raise AssertionError("host path called")

    for name in ("_eval", "_divide_by_x_minus_a"):
        monkeypatch.setattr(kzg, name, boom)
    host_poly = kzg._host_poly

    def host_arrays_only(p, words):     # a device polynomial brought back to the host is the sharded-key path
        if kzg._is_device(p):
            boom()
        return host_poly(p, words)

    monkeypatch.setattr(kzg, "_host_poly", host_arrays_only)
    monkeypatch.setattr(fft.Domain, "FFT", boom)
    monkeypatch.setattr(fft.Domain, "FFTInverse", boom)
    for key in (pk, pkw):
        monkeypatch.setattr(key._bases, "MultiExp", boom)
        _assert_equal_ref(perm.Prove(key, a, b), want, c)
        _assert_equal_ref(perm.Prove(key, _dev(a), _dev(b)), want, c)
    monkeypatch.undo()
    pk.close()
    pkw.close()


def test_sharded_key(monkeypatch):
    """a proving key sharded over GMSM_DEVICES (device = -1; two shards on device 0 when there is one GPU) commits and opens through
    kzg's host entry points and gives the same proof as the restatement"""
    kzg, perm, _ = _mods()
    torch = _torch()
    ndev = torch.cuda.device_count()
    monkeypatch.setenv("GMSM_DEVICES", ",".join(str(d) for d in range(min(ndev, 4))) if ndev > 1 else "0,0")
    c = "bn254"
    r = kzg.CURVE_PARAMS[c].r
    alpha = 424242
    pk = _pk(c, 1 << 10, alpha, device=-1)
    for n in (8, 1 << 10):
        a, b = _rand_perm(c, n, 77 + n)
        want = ref.prove(c, curves._fr_decode(a, r), curves._fr_decode(b, r), ref.ClosedFormSRS(c, 1 << 10, alpha))
        _assert_equal_ref(perm.Prove(pk, a, b), want, c)
    pk.close()
