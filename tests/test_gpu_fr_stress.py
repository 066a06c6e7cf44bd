"""The sm_90a Fr layer of the seven pairing curves at extreme operands and production sizes (generators and references in
tests/fr_stress.py; the CPU twin is tests/test_fr_stress_cpu.py):

A. every ordered pair of Fr extremes through the linear combination, both k_poly_fold instantiations, with and without
   accumulation: the inlined fp_mul / fp_add of fft.cu on the Fr moduli;
B. every ordered pair through the n = 2 butterflies, forward and inverse, both decimations: fp_add / fp_sub;
C. every FFT variant on extreme vectors from 2 to 2^13 (tile only, one and three strided stages), against the oracle;
D. every FFT variant in closed form on sparse vectors at 2^20 and 2^22, at 2048+ positions including every 2^b, 2^b - 1 and
   n - 1 - 2^b, and the bit reversal of a whole vector -- the twiddle tables, strided-stage indices, coset and inverse scalings
   and DIF's bit-reversed output order against independent values, where round trips would cancel a shared error;
E. the opening scan at three carry levels on random coefficients, with points whose level multipliers are 1 or -1."""
import ctypes
import random
from importlib import import_module

import numpy as np
import pytest

from tests import fr_stress as R

pytestmark = pytest.mark.gpu


def _torch():
    return import_module("torch")


def _lib():
    return import_module("gnark-crypto_b200._native").lib()


def _err():
    return import_module("gnark-crypto_b200._native").last_error()


def _fft():
    import gnark_crypto_b200  # noqa: F401

    return import_module("gnark-crypto_b200.fft")


def _dev(a):
    return _torch().from_numpy(np.ascontiguousarray(a, dtype=np.uint64).view(np.int64).reshape(-1).copy()).cuda()


def _host(t, w):
    return t.cpu().numpy().view(np.uint64).reshape(-1, w)


def _stream():
    return _torch().cuda.current_stream().cuda_stream


# ---- A ----
def _lincomb(c):
    torch = _torch()
    w = R.fr(c).limbs

    def run(polys, scalars, strides, offsets, out_len, init):
        up = {}
        d = [up.setdefault(id(p), (p, _dev(p)))[1] for p in polys]      # one upload per distinct input array
        d_out = _dev(init) if init is not None else torch.full((out_len * w,), -1, dtype=torch.int64, device="cuda")
        ptrs = (ctypes.c_void_p * len(d))(*[x.data_ptr() for x in d])
        ln = np.array([len(p) for p in polys], dtype=np.uint64)
        st = np.array(strides, dtype=np.uint64)
        off = np.array(offsets, dtype=np.uint64)
        sc = np.ascontiguousarray(scalars, dtype=np.uint64)
        rc = _lib().gmsm_fr_poly_lincomb_device(R.FIELD[c], ptrs, ln.ctypes.data, sc.ctypes.data, st.ctypes.data, off.ctypes.data,
                                                len(d), d_out.data_ptr(), out_len, 1 if init is not None else 0, _stream())
        assert rc == 0, _err()
        return _host(d_out, w)

    return run


@pytest.mark.parametrize("c", R.CURVES)
def test_lincomb_extremes_device(c):
    R.check_lincomb_extremes(c, _lincomb(c), "device")


# ---- B ----
@pytest.mark.parametrize("c", R.CURVES)
def test_butterfly_extremes_device(c):
    """one n = 2 transform per ordered pair, each called on its 2-element slice of one device buffer, one synchronise per
    variant"""
    torch = _torch()
    fft = _fft()
    L = _lib()
    w = R.fr(c).limbs
    d = fft.NewDomain(c, 2)

    def run(buf, inverse, dec):
        t = _dev(buf)
        base, step, st = t.data_ptr(), 2 * 8 * w, _stream()
        for s in range(len(buf) // 2):
            rc = L.gmsm_fft_device(d._h, base + s * step, 2, int(inverse), int(dec), 0, st)
            assert rc == 0, _err()
        torch.cuda.synchronize()
        return _host(t, w)

    try:
        R.check_butterflies(c, run, "device")
    finally:
        d.close()


# ---- C ----
@pytest.mark.parametrize("c", R.CURVES)
@pytest.mark.parametrize("logn", [1, 2, 5, 10, 11, 13])
def test_fft_extreme_vectors_device(c, logn):
    d = _fft().NewDomain(c, 1 << logn)

    def run(a, inverse, dec, coset):
        return (d.FFTInverse if inverse else d.FFT)(a, dec, OnCoset=coset)

    try:
        R.check_fft_extremes(c, logn, run, "device")
    finally:
        d.close()


# ---- D ----
LARGE = [(c, 20) for c in R.CURVES] + [(c, 22) for c in ("bn254", "bls12381", "bls24315", "bls24317", "bw6761")]


@pytest.mark.parametrize("c,logn", LARGE)
def test_fft_closed_forms_large(c, logn):
    """sparse vectors of 8 extremes at logical indices 0, 1, n/2, n - 1 and random ones (DIT input placed at bitrev(k)); every
    variant; outputs read at >= 2048 logical indices (DIF output at bitrev(i)); then gmsm_fft_bit_reverse_device on i -> i"""
    torch = _torch()
    f = R.fr(c)
    r, w = f.q, f.limbs
    n = 1 << logn
    rng = random.Random(1000 * logn + R.FIELD[c])
    od = R.domain(c, n)
    d = _fft().NewDomain(c, n)
    try:
        positions = R.check_positions(n, rng)
        for dec, coset, inverse in R.VARIANTS:
            terms = R.sparse_terms(c, n, rng)
            place = (lambda k: R.bitrev(k, logn)) if dec == R.DIT else (lambda k: k)
            read = (lambda i: R.bitrev(i, logn)) if dec == R.DIF else (lambda i: i)
            dv = torch.zeros((n, w), dtype=torch.int64, device="cuda")
            rows = torch.tensor([place(k) for k, _ in terms], dtype=torch.int64, device="cuda")
            dv[rows] = _dev(R.pack([v for _, v in terms], w)).view(len(terms), w)
            d.fft_device(dv, inverse, dec, coset=coset)
            idx = torch.tensor([read(i) for i in positions], dtype=torch.int64, device="cuda")
            got = dv[idx].cpu().numpy().view(np.uint64)
            want = R.closed_form(od, terms, positions, inverse, coset)
            R.compare("device %s logn=%d gmsm_fft_device %s" % (c, logn, R.variant_name(dec, coset, inverse)), got, want, r,
                      lambda t: tuple(v for _, v in terms), kind="logical output index; terms %s, stored values" % [k for k, _ in terms],
                      index=lambda t: positions[t])
            del dv
        # bit reversal of the whole vector: entry i holds i (+ the limb number in the high half, to catch a limb mix-up)
        i = torch.arange(n, dtype=torch.int64, device="cuda")
        dv = torch.stack([i + (k << 32) for k in range(w)], dim=1).contiguous()
        d.bit_reverse_device(dv)
        got = dv.cpu().numpy()
        want = R.bitrev(np.arange(n, dtype=np.int64), logn)
        for k in range(w):
            bad = np.nonzero(got[:, k] != want + (k << 32))[0]
            assert len(bad) == 0, "device %s logn=%d gmsm_fft_bit_reverse_device: position %d limb %d holds %d, want %d" % (
                c, logn, bad[0], k, got[bad[0], k], want[bad[0]] + (k << 32))
    finally:
        d.close()


# ---- E ----
def _div(c):
    torch = _torch()
    L = _lib()
    w = R.fr(c).limbs

    def run(F, A, quotient):
        n = len(F)
        d_f = _dev(F)
        d_h = torch.empty(max(n - 1, 1) * w, dtype=torch.int64, device="cuda") if quotient else None
        d_fa = torch.empty(w, dtype=torch.int64, device="cuda")
        ws = int(L.gmsm_fr_poly_workspace_bytes(R.FIELD[c], n))
        d_work = torch.empty(max(ws // 8, 1), dtype=torch.int64, device="cuda")
        a = np.ascontiguousarray(A[0], dtype=np.uint64)
        rc = L.gmsm_fr_poly_div_x_minus_a_device(R.FIELD[c], d_f.data_ptr(), n, a.ctypes.data, d_h.data_ptr() if quotient else None,
                                                 d_fa.data_ptr(), d_work.data_ptr(), _stream())
        assert rc == 0, _err()
        assert torch.equal(d_f, _dev(F)), "the polynomial was modified"
        return _host(d_fa, w), (_host(d_h, w)[: n - 1] if quotient else None)

    return run


def _scan_cases():
    out = []
    for c in R.CURVES:
        t = R.TILE[8 * R.fr(c).limbs]
        out += [(c, t * t + 1), (c, t * t + 5 * t + 3)]
    return out + [("bn254", (1 << 22) + 3)]


@pytest.mark.parametrize("c,n", _scan_cases())
def test_scan_three_levels_device(c, n):
    """n = T^2 + 1 (levels of T^2 + 1, T + 1 and 2 elements) and T^2 + 5 T + 3 (partial last tiles on two levels), T the tile of
    fft.cu; bn254 also at 2^22 + 3 with a random point.  Random coefficients; a in {random, 0, 1, r - 1, a primitive T-th root,
    a primitive 2T-th root}"""
    t = R.TILE[8 * R.fr(c).limbs]
    rng = random.Random(n + R.FIELD[c])
    points = R.scan_points(c, t, rng)
    if n > (1 << 22):
        points = points[:1]
    R.check_scan(c, R.random_stored(c, n, n + 31 * R.FIELD[c]), points, _div(c), "device")
