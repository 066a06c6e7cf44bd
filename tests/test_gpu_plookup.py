"""plookup.ProveLookupVector and ProveLookupTables on the device for the seven pairing curves: the new entry points
(gmsm_fr_sort_device, gmsm_fr_plookup_accumulate_device, gmsm_fft_plookup_numerator_device) against the big-int restatements of
tests/plookup_ref.py with their rejected arguments; the sort at 2^23 - 1 keys (bn254) and 2^21 - 1 keys (bw6-761) against
np.lexsort; both provers bit-identical to the line-by-line restatements of vector.go and table.go with closed-form digests; the
verifiers restated without the pairings on a known-alpha SRS; the errors; the device path taken on single-device keys; the
sharded-key path."""
import random
from importlib import import_module

import numpy as np
import pytest

from oracle import oracle as O
from tests import plookup_ref as ref

curves = import_module("gnark-crypto_b200.curves")

pytestmark = pytest.mark.gpu
CURVES = ["bn254", "bls12381", "bls12377", "bls24315", "bls24317", "bw6633", "bw6761"]
FIELD = {c: i for i, c in enumerate(CURVES)}


def _mods():
    return import_module("gnark-crypto_b200.kzg"), import_module("gnark-crypto_b200.plookup"), import_module("gnark-crypto_b200.fft")


def _nat():
    return import_module("gnark-crypto_b200._native")


def _torch():
    return import_module("torch")


def _dev(a):
    return _torch().from_numpy(np.ascontiguousarray(a, dtype=np.uint64).view(np.int64).reshape(-1).copy()).cuda()


def _host(t, w):
    return t.cpu().numpy().view(np.uint64).reshape(-1, w)


def _r(c):
    return _mods()[0].CURVE_PARAMS[c].r


def _enc(vals, c):
    return curves._fr_encode(vals, _r(c))


def _stream():
    return _torch().cuda.current_stream().cuda_stream


def _assert_limbs(got, want_vals, c, what):
    want = _enc(want_vals, c)
    bad = np.nonzero((got != want).any(axis=1))[0]
    assert bad.size == 0, "%s %s: first mismatch at %d of %d" % (c, what, bad[0], len(want_vals))


def _sort(c, d_in, n, d_out):
    torch = _torch()
    L = _nat().lib()
    work = torch.empty(int(L.gmsm_fr_sort_workspace_bytes(FIELD[c], n)) // 8 + 1, dtype=torch.int64, device="cuda")
    rc = L.gmsm_fr_sort_device(FIELD[c], d_in.data_ptr(), n, d_out.data_ptr(), work.data_ptr(), _stream())
    assert rc == 0, _nat().last_error()


@pytest.mark.parametrize("c", CURVES)
def test_abi_sort_accumulate_numerator(c):
    """the sort (random keys, equal keys, small values, 0 and r - 1, in place), the accumulation polynomial (with a forced zero
    denominator) and the numerator at big-domain sizes 2 ... 2^10 and 2^14 against the big-int restatements; inputs unchanged"""
    kzg, _, fft = _mods()
    torch = _torch()
    L = _nat().lib()
    r, w = _r(c), kzg.CURVE_PARAMS[c].fr_words
    rng = random.Random(11 + FIELD[c])
    for vals in ([rng.randrange(r) for _ in range(5000)], [rng.randrange(r)] * 300, [rng.randrange(1 << 12) for _ in range(70001)],
                 [0, r - 1] + [rng.randrange(r) for _ in range(1000)] + [r - 1, 0], [7]):
        a = _enc(vals, c)
        d_a = _dev(a)
        d_out = torch.full_like(d_a, -1)
        _sort(c, d_a, len(vals), d_out)
        _assert_limbs(_host(d_out, w), ref.sort(vals), c, "sort n=%d" % len(vals))
        assert np.array_equal(_host(d_a, w), a)
        _sort(c, d_a, len(vals), d_a)
        _assert_limbs(_host(d_a, w), ref.sort(vals), c, "sort in place n=%d" % len(vals))
    ws = int(L.gmsm_fr_permutation_workspace_bytes(FIELD[c], 1 << 16))
    work = torch.empty(max(ws // 8, 1), dtype=torch.int64, device="cuda")
    for n in (1, 2, 1 << 10, 1 << 16):
        lt = sorted(rng.randrange(r) for _ in range(n))
        lf = [lt[rng.randrange(n)] for _ in range(n)]
        h = sorted(lt + lf[:n - 1])
        vs = [lf, lt, h[:n], h[n - 1:]]
        enc = [_enc(v, c) for v in vs]
        d_in = [_dev(e) for e in enc]
        cases = [(rng.randrange(r), rng.randrange(r))]
        if n > 2:
            i, beta = n // 3, rng.randrange(r)
            cases.append((beta, -(h[i] + beta * h[i + 1]) * pow(1 + beta, r - 2, r) % r))
        for beta, gamma in cases:
            d_z = torch.full_like(d_in[0], -1)
            b, g = _enc([beta], c)[0], _enc([gamma], c)[0]
            rc = L.gmsm_fr_plookup_accumulate_device(FIELD[c], *(d.data_ptr() for d in d_in), n, b.ctypes.data, g.ctypes.data, d_z.data_ptr(),
                                                     work.data_ptr(), _stream())
            assert rc == 0, _nat().last_error()
            _assert_limbs(_host(d_z, w), ref.accumulate(*vs, beta, gamma, r), c, "accumulate n=%d" % n)
        assert all(np.array_equal(_host(d, w), e) for d, e in zip(d_in, enc))
    for logn in list(range(1, 11)) + [14]:
        n = 1 << logn
        dom = fft.NewDomain(c, n)
        od = ref.domain(c, n)
        vals = [[rng.randrange(r) for _ in range(n)] for _ in range(5)]
        enc = [_enc(v, c) for v in vals]
        d_in = [_dev(e) for e in enc]
        ch = [rng.randrange(r) for _ in range(3)]
        chl = [_enc([v], c)[0] for v in ch]
        d_out = torch.full_like(d_in[0], -1)
        rc = L.gmsm_fft_plookup_numerator_device(dom._h, *(d.data_ptr() for d in d_in), n, *(v.ctypes.data for v in chl), d_out.data_ptr(),
                                                 _stream())
        assert rc == 0, _nat().last_error()
        _assert_limbs(_host(d_out, w), ref.numerator(*vals, *ch, n, od.shift, od.generator, r), c, "numerator n=%d" % n)
        assert all(np.array_equal(_host(d, w), e) for d, e in zip(d_in, enc))
        dom.close()
    torch.cuda.synchronize()


@pytest.mark.parametrize("c,logn", [("bn254", 23), ("bw6761", 21)])
def test_sort_large(c, logn):
    """2^logn - 1 random keys against np.lexsort on the canonical limbs"""
    kzg = _mods()[0]
    torch = _torch()
    cp = kzg.CURVE_PARAMS[c]
    w = cp.fr_words
    n = (1 << logn) - 1
    rng = np.random.default_rng(logn)
    canon = rng.integers(0, 2**63, size=(n, w), dtype=np.uint64) * 2 + rng.integers(0, 2, size=(n, w), dtype=np.uint64)
    canon[:, -1] &= np.uint64((1 << ((cp.r.bit_length() - 1) - 64 * (w - 1))) - 1)
    want = canon[np.lexsort(canon.T)]           # the last column (the top limb) is the primary key
    d_in = _dev(_to_mont(canon, cp))
    d_out = torch.empty_like(d_in)
    _sort(c, d_in, n, d_out)
    assert np.array_equal(_from_mont(_host(d_out, w), cp), want)
    torch.cuda.synchronize()


def _to_mont(canon, cp):
    """x -> x R mod r on numpy limbs (object arrays of Python ints)"""
    return _mont_map(canon, cp, pow(2, 64 * cp.fr_words, cp.r))


def _from_mont(mont, cp):
    return _mont_map(mont, cp, pow(2, -64 * cp.fr_words, cp.r))


def _mont_map(a, cp, k):
    w = cp.fr_words
    objs = np.zeros(a.shape[0], dtype=object)
    for j in range(w):
        objs = objs + (a[:, j].astype(object) << (64 * j))
    objs = objs * k % cp.r
    out = np.empty_like(a)
    mask = (1 << 64) - 1
    for j in range(w):
        out[:, j] = ((objs >> (64 * j)) & mask).astype(np.uint64)
    return out


def test_abi_rejects_bad_arguments():
    kzg, _, fft = _mods()
    torch = _torch()
    nat = _nat()
    L = nat.lib()
    c = "bn254"
    d_a = _dev(_enc(list(range(1, 65)), c))
    d_b = _dev(_enc(list(range(1, 65)), c))
    d_z = torch.zeros_like(d_a)
    work = torch.zeros(int(L.gmsm_fr_sort_workspace_bytes(0, 64)) // 8 + 1, dtype=torch.int64, device="cuda")
    one = _enc([5], c)[0]
    bad = np.array([0xFFFFFFFFFFFFFFFF] * 4, dtype=np.uint64)
    dom = fft.NewDomain(c, 64)

    def srt(field=0, a=d_a, n=64, out=d_z, wk=work):
        return L.gmsm_fr_sort_device(field, a.data_ptr(), n, out.data_ptr() if out is not None else None,
                                     wk.data_ptr() if wk is not None else None, None)

    def acc(field=0, n=64, b=one, g=one, z=d_z, f=d_a):
        return L.gmsm_fr_plookup_accumulate_device(field, f.data_ptr() if f is not None else None, d_a.data_ptr(), d_b.data_ptr(),
                                                   d_b.data_ptr(), n, b.ctypes.data, g.ctypes.data, z.data_ptr(), work.data_ptr(), None)

    def num(n=64, b=one, a=one, out=d_z):
        return L.gmsm_fft_plookup_numerator_device(dom._h, d_a.data_ptr(), d_b.data_ptr(), d_b.data_ptr(), d_a.data_ptr(), d_a.data_ptr(), n,
                                                   b.ctypes.data, one.ctypes.data, a.ctypes.data, out.data_ptr(), None)

    assert srt() == 0 and acc() == 0 and num() == 0
    cases = [
        (lambda: srt(field=9), "unknown scalar field"),
        (lambda: srt(n=0), "n = 0"),
        (lambda: srt(out=None), "null vector"),
        (lambda: srt(wk=None), "null workspace"),
        (lambda: srt(out=d_a[4:]), "must equal the input or not overlap"),
        (lambda: srt(wk=d_a), "workspace must not overlap"),
        (lambda: acc(field=7), "unknown scalar field"),
        (lambda: acc(n=0), "n = 0"),
        (lambda: acc(f=None), "null vector"),
        (lambda: acc(b=bad), "beta is not a reduced fr.Element"),
        (lambda: acc(g=bad), "gamma is not a reduced fr.Element"),
        (lambda: acc(z=d_b), "must not overlap"),
        (lambda: num(n=32), "must equal the domain cardinality"),
        (lambda: num(b=bad), "beta is not a reduced"),
        (lambda: num(a=bad), "alpha is not a reduced"),
        (lambda: num(out=d_a), "must not overlap"),
    ]
    for fn, text in cases:
        assert fn() == nat.GMSM_EINVAL, text
        assert text in nat.last_error(), (text, nat.last_error())
    assert L.gmsm_fr_sort_workspace_bytes(9, 64) == 0 and L.gmsm_fr_sort_workspace_bytes(0, 0) == 0
    dom.close()
    torch.cuda.synchronize()


def _pk(c, size, alpha, window_tables=False, device=0):
    kzg = _mods()[0]
    G = O.GROUPS[c + "_g1"]
    gen = G.encode_affine([G.gen])[0]
    srs = kzg.new_srs_g1(c, size, alpha, gen, kzg.CURVE_PARAMS[c].r, G.encode_scalars)
    return kzg.ProvingKey(c, srs, device=device, window_tables=window_tables)


def _assert_vector(proof, want, c):
    assert proof.size == want["size"]
    assert curves._fr_decode(proof.g, _r(c))[0] == want["g"]
    for name in ("h1", "h2", "t", "z", "f", "h"):
        assert np.array_equal(proof.__dict__[name], want[name]), name
    assert np.array_equal(proof.BatchedProof.H, want["H"])
    assert np.array_equal(proof.BatchedProof.ClaimedValues, _enc(want["claimed"], c))
    assert np.array_equal(proof.BatchedProofShifted.H, want["Hs"])
    assert np.array_equal(proof.BatchedProofShifted.ClaimedValues, _enc(want["claimed_s"], c))


def _assert_tables(proof, want, c):
    assert len(proof.fs) == len(want["fs"]) and len(proof.ts) == len(want["ts"])
    for a, b in zip(proof.fs + proof.ts, want["fs"] + want["ts"]):
        assert np.array_equal(a, b)
    _assert_vector(proof.foldedProof, want["folded"], c)
    p, q = proof.permutationProof, want["permutation"]
    for name in ("t1", "t2", "z", "q"):
        assert np.array_equal(p.__dict__[name], q[name]), name
    assert np.array_equal(p.batchedProof.H, q["H"]) and np.array_equal(p.shiftedProof.H, q["Hs"])
    assert np.array_equal(p.batchedProof.ClaimedValues, _enc(q["claimed"], c))


def _reference_vector(c):
    """plookup_test.go TestLookupVector: t[i] = 2i for i < 8, f[i] = t[(4i + 1) mod 8] for i < 7"""
    t = [2 * i for i in range(8)]
    return [t[(4 * i + 1) % 8] for i in range(7)], t


def _reference_tables():
    """plookup_test.go TestLookupTable: 3 rows, t[i][j] = 2i + j (j < 8), f[i][j] = t[i][(4j + 1) mod 8] (j < 7)"""
    t = [[2 * i + j for j in range(8)] for i in range(3)]
    return [[row[(4 * j + 1) % 8] for j in range(7)] for row in t], t


def _random_vector(rng, r, nf, nt, dup=False):
    t = [rng.randrange(r) for _ in range(nt)]
    if dup:
        t = [t[rng.randrange(max(nt // 4, 1))] for _ in range(nt)]   # unsorted, with repeats
    return [t[rng.randrange(nt)] for _ in range(nf)], t


@pytest.mark.parametrize("c", CURVES)
def test_prove_equals_restatement(c):
    """ProveLookupVector and ProveLookupTables == the line-by-line restatements with closed-form digests: the reference's own vectors
    (SRS of 64, alpha = 13), its "wrong proof" cases (f[0] random: they prove and fail the restated verify), random cases with
    len(f) > len(t), len(f) a power of two (the domain doubles), unsorted t with duplicates; host and device inputs (unchanged), a
    window-table key"""
    kzg, pl, _ = _mods()
    r = _r(c)
    rng = random.Random(29 + FIELD[c])
    pk = _pk(c, 64, 13)
    srs = ref.ClosedFormSRS(c, 64, 13)
    f, t = _reference_vector(c)
    want = ref.prove_vector(c, f, t, srs)
    proof = pl.ProveLookupVector(pk, _enc(f, c), _enc(t, c))
    _assert_vector(proof, want, c)
    assert ref.verify_vector(c, proof, 13)
    f[0] = rng.randrange(r)
    proof = pl.ProveLookupVector(pk, _enc(f, c), _enc(t, c))
    _assert_vector(proof, ref.prove_vector(c, f, t, srs), c)
    assert not ref.verify_vector(c, proof, 13)
    ft, tt = _reference_tables()
    proof = pl.ProveLookupTables(pk, [_enc(v, c) for v in ft], [_enc(v, c) for v in tt])
    _assert_tables(proof, ref.prove_tables(c, ft, tt, srs), c)
    assert ref.verify_tables(c, proof, 13)
    ft[0][0] = rng.randrange(r)
    proof = pl.ProveLookupTables(pk, [_enc(v, c) for v in ft], [_enc(v, c) for v in tt])
    _assert_tables(proof, ref.prove_tables(c, ft, tt, srs), c)
    assert not ref.verify_tables(c, proof, 13)
    pk.close()

    alpha = rng.randrange(r)
    size = 1 << 10
    pk, pkw = _pk(c, size, alpha), _pk(c, size, alpha, window_tables=True)
    srs = ref.ClosedFormSRS(c, size, alpha)
    cases = [_random_vector(rng, r, 100, 20), _random_vector(rng, r, 64, 64), _random_vector(rng, r, 30, 200, dup=True),
             _random_vector(rng, r, 1, 1), _random_vector(rng, r, 255, 256, dup=True)]
    for k, (f, t) in enumerate(cases):
        want = ref.prove_vector(c, f, t, srs)
        a, b = _enc(f, c), _enc(t, c)
        keep = (a.copy(), b.copy())
        _assert_vector(pl.ProveLookupVector(pk, a, b), want, c)
        assert np.array_equal(a, keep[0]) and np.array_equal(b, keep[1])
        d_a, d_b = _dev(a), _dev(b)
        _assert_vector(pl.ProveLookupVector(pkw if k % 2 else pk, d_a, d_b), want, c)
        assert np.array_equal(_host(d_a, a.shape[1]), a) and np.array_equal(_host(d_b, b.shape[1]), b)
    ft = [[rng.randrange(r) for _ in range(37)] for _ in range(2)]
    tt = [[rng.randrange(r) for _ in range(50)] for _ in range(2)]
    rows = ([_enc(v, c) for v in ft], [_enc(v, c) for v in tt])
    keep = [x.copy() for x in rows[0] + rows[1]]
    want = ref.prove_tables(c, ft, tt, srs)
    _assert_tables(pl.ProveLookupTables(pkw, *rows), want, c)
    assert all(np.array_equal(x, y) for x, y in zip(rows[0] + rows[1], keep))
    _assert_tables(pl.ProveLookupTables(pk, [_dev(x) for x in rows[0]], [_dev(x) for x in rows[1]]), want, c)
    _torch().cuda.synchronize()
    pk.close()
    pkw.close()


@pytest.mark.parametrize("c,logn", [(c, 16) for c in CURVES] + [("bn254", 20), ("bw6761", 20)])
def test_verify_known_alpha(c, logn):
    """a proof of a random vector in a random table of 2^logn - 1 entries (s = 2^logn) passes VerifyLookupVector restated without
    the pairings on the known-alpha SRS of 2s points; with f[0] replaced by a value outside the table it proves and fails"""
    kzg, pl, _ = _mods()
    cp = kzg.CURVE_PARAMS[c]
    r, w = cp.r, cp.fr_words
    n = 1 << logn
    rng = random.Random(logn * 5 + FIELD[c])
    alpha = rng.randrange(r)
    pk = _pk(c, 2 * n, alpha)
    g = np.random.default_rng(logn + FIELD[c])
    t = g.integers(0, 2**63, size=(n - 1, w), dtype=np.uint64)
    t[:, -1] &= np.uint64((1 << 56) - 1)
    f = np.ascontiguousarray(t[g.integers(0, n - 1, size=n - 1)])
    proof = pl.ProveLookupVector(pk, _dev(f), _dev(t))
    assert proof.size == n
    assert ref.verify_vector(c, proof, alpha)
    f[0] = _enc([rng.randrange(r)], c)[0]
    assert not ref.verify_vector(c, pl.ProveLookupVector(pk, f, t), alpha)
    pk.close()


def test_errors():
    """unequal row counts and ragged rows (ErrIncompatibleSize), empty inputs (ValueError), an SRS too small for the 2s-coefficient
    quotient (ErrInvalidPolynomialSize at Commit(h), after the earlier commits), an SRS too small for the s-coefficient commits"""
    kzg, pl, _ = _mods()
    c = "bn254"
    pk = _pk(c, 16, 12345)
    t = _enc(list(range(16)), c)
    with pytest.raises(pl.ErrIncompatibleSize, match="^the tables in f and t are not of the same size$"):
        pl.ProveLookupTables(pk, [t[:7]] * 2, [t[:8]] * 3)
    with pytest.raises(pl.ErrIncompatibleSize):
        pl.ProveLookupTables(pk, [t[:7], t[:6]], [t[:8]] * 2)
    with pytest.raises(ValueError, match="must not be empty"):
        pl.ProveLookupVector(pk, t[:0], t)
    with pytest.raises(ValueError, match="must not be empty"):
        pl.ProveLookupTables(pk, [], [])
    commits = []
    real_commit = kzg.Commit

    def counting(p, key, *a):
        commits.append(kzg._poly_len(p, 4))
        return real_commit(p, key, *a)

    mp = pytest.MonkeyPatch()
    mp.setattr(kzg, "Commit", counting)
    with pytest.raises(kzg.ErrInvalidPolynomialSize, match="larger than SRS or == 0"):
        pl.ProveLookupVector(pk, t[:15], t[:16])       # s = 16: the five s-point commits fit, the quotient's 32 do not
    mp.undo()
    assert commits == [16] * 5 + [32]
    with pytest.raises(kzg.ErrInvalidPolynomialSize, match="larger than SRS or == 0"):
        pl.ProveLookupVector(pk, t[:16], t[:16])       # s = 32 > 16 points
    pk.close()


def test_device_path_taken(monkeypatch):
    """on single-device keys (plain and window tables) no host FFT, host Fr loop or host MultiExp runs, and no device polynomial is
    brought back to the host"""
    kzg, pl, fft = _mods()
    c = "bls12377"
    r = _r(c)
    alpha = 987654321
    pk, pkw = _pk(c, 512, alpha), _pk(c, 512, alpha, window_tables=True)
    rng = random.Random(3)
    f, t = _random_vector(rng, r, 150, 100, dup=True)
    srs = ref.ClosedFormSRS(c, 512, alpha)
    want = ref.prove_vector(c, f, t, srs)
    ft, tt = [[rng.randrange(r) for _ in range(20)] for _ in range(3)], [[rng.randrange(r) for _ in range(30)] for _ in range(3)]
    want_t = ref.prove_tables(c, ft, tt, srs)

    def boom(*args, **kw):
        raise AssertionError("host path called")

    for name in ("_eval", "_divide_by_x_minus_a"):
        monkeypatch.setattr(kzg, name, boom)
    host_poly = kzg._host_poly

    def host_arrays_only(p, words):
        if kzg._is_device(p):
            boom()
        return host_poly(p, words)

    monkeypatch.setattr(kzg, "_host_poly", host_arrays_only)
    monkeypatch.setattr(fft.Domain, "FFT", boom)
    monkeypatch.setattr(fft.Domain, "FFTInverse", boom)
    for key in (pk, pkw):
        monkeypatch.setattr(key._bases, "MultiExp", boom)
        _assert_vector(pl.ProveLookupVector(key, _enc(f, c), _enc(t, c)), want, c)
        _assert_vector(pl.ProveLookupVector(key, _dev(_enc(f, c)), _dev(_enc(t, c))), want, c)
        _assert_tables(pl.ProveLookupTables(key, [_enc(v, c) for v in ft], [_enc(v, c) for v in tt]), want_t, c)
    monkeypatch.undo()
    pk.close()
    pkw.close()


def test_sharded_key(monkeypatch):
    """a proving key sharded over GMSM_DEVICES (device = -1; two shards on device 0 when there is one GPU) commits and opens through
    kzg's host entry points and gives the same proofs as the restatements"""
    kzg, pl, _ = _mods()
    torch = _torch()
    ndev = torch.cuda.device_count()
    monkeypatch.setenv("GMSM_DEVICES", ",".join(str(d) for d in range(min(ndev, 4))) if ndev > 1 else "0,0")
    c = "bn254"
    r = _r(c)
    alpha = 424242
    pk = _pk(c, 1 << 10, alpha, device=-1)
    srs = ref.ClosedFormSRS(c, 1 << 10, alpha)
    rng = random.Random(8)
    for nf, nt in ((7, 8), (300, 200)):
        f, t = _random_vector(rng, r, nf, nt)
        _assert_vector(pl.ProveLookupVector(pk, _enc(f, c), _enc(t, c)), ref.prove_vector(c, f, t, srs), c)
    ft, tt = _reference_tables()
    _assert_tables(pl.ProveLookupTables(pk, [_enc(v, c) for v in ft], [_enc(v, c) for v in tt]), ref.prove_tables(c, ft, tt, srs), c)
    pk.close()
