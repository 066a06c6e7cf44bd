"""Extreme operands, references and checks for the device Fr layer of the seven pairing curves: the linear combination
(k_poly_fold, both instantiations), the FFT (butterflies, strided stages, tile kernel, coset and inverse scaling, bit
reversal) and the opening scan (k_poly_heads / k_poly_write).

Shared by tests/test_gpu_fr_stress.py (the sm_90a kernels of fft.cu through the C ABI) and tests/test_fr_stress_cpu.py (the
same kernels built for the CPU with -DGMSM_EMULATE_PTX, through tests/emu).  Not a conftest.

Values are STORED values, as in tests/arith_stress.py: the Montgomery integer m < r a kernel reads, standing for m R^-1.  The
FFT and the scan are linear maps with plain constants (twiddles, coset powers, n^-1, the point a), and so is the Montgomery
map v -> v R mod r; their references therefore run directly on stored integers, with no conversion of the 10^6-element
vectors.  Only the linear combination's scalar is itself a stored value, which brings in R^-1.  Outputs are compared limb for
limb with the reference, so they must also be canonical (< r).  A failure names the field, the entry point, the variant, the
index and the operands as stored decimal integers, so that it can be replayed through the CPU twin."""
import random

import numpy as np

from oracle import oracle as O
from tests import arith_stress as S
from tests import fft_more_fields as M

CURVES = ["bn254", "bls12381", "bls12377", "bls24315", "bls24317", "bw6633", "bw6761"]
FIELD = {c: i for i, c in enumerate(CURVES)}      # GMSM_FR_*
TILE = {32: 1024, 40: 1024, 48: 512}              # coefficients per block of the opening scan in fft.cu, by fr.Bytes
DIT, DIF = O.DIT, O.DIF


def fr(c):
    return O.FIELDS[c + "_fr"]


def domain(c, n, shift=None):
    """the oracle's fft.Domain of n over the scalar field of c"""
    name = c + "_fr"
    return (O.FFTDomain if name in O.FFT_PARAMS else M.FFTDomain)(name, n, shift)


def extremes(c):
    return S.field_extremes(fr(c))


# ------------------------------------------------------------------------------------------
# stored integers <-> (m, fr.Limbs) u64 arrays
# ------------------------------------------------------------------------------------------


def pack(vals, w):
    nb = 8 * w
    buf = b"".join(v.to_bytes(nb, "little") for v in vals)
    return np.frombuffer(buf, dtype="<u8").astype(np.uint64).reshape(len(vals), w)


def unpack(arr):
    a = np.ascontiguousarray(arr, dtype=np.uint64)
    nb = 8 * a.shape[1]
    b = a.tobytes()
    return [int.from_bytes(b[nb * i : nb * (i + 1)], "little") for i in range(a.shape[0])]


def bitrev(i, logn):
    """bit reversal of logn-bit indices (an int or a numpy integer array)"""
    if isinstance(i, np.ndarray):
        out = np.zeros_like(i)
        for b in range(logn):
            out |= ((i >> b) & 1) << (logn - 1 - b)
        return out
    return int(format(i, "0%db" % logn)[::-1], 2) if logn else 0


def compare(what, got, want, r, operands, kind="stored operands (decimal Montgomery limbs)", index=None):
    """got: (m, w) limbs; want: m stored integers.  On a mismatch names the first bad entry i (index(i) when the entries are
    not in output order) with operands(i)"""
    got = np.ascontiguousarray(got, dtype=np.uint64).reshape(len(want), -1)
    exp = pack(want, got.shape[1])
    if np.array_equal(got, exp):
        return
    i = int(np.nonzero((got != exp).any(axis=1))[0][0])
    g = unpack(got[i : i + 1])[0]
    S._fail(what + ("" if g < r else " (non-canonical output)"), i if index is None else index(i), operands(i), g, want[i], kind)


# ------------------------------------------------------------------------------------------
# A. product and sum: the linear combination on the extremes
# ------------------------------------------------------------------------------------------


def check_lincomb_extremes(c, lincomb, label):
    """lincomb(polys, scalars, strides, offsets, out_len, init) runs gmsm_fr_poly_lincomb_device's contract on host arrays
    (polys: list of (len, w) limb arrays; scalars: (k, w); init: (out_len, w) to accumulate onto, or None) and returns the
    (out_len, w) output.  For every extreme x: E x R^-1 (the stride-1 kernel), then the same added onto E reversed; then one
    strided call whose output is the transposed product table E[j] E[i] R^-1 at j |E| + i"""
    f = fr(c)
    r, w, ri = f.q, f.limbs, f.Rinv
    E = extremes(c)
    m = len(E)
    P = pack(E, w)
    rev = E[::-1]
    Rev = pack(rev, w)
    ep = "%s %s gmsm_fr_poly_lincomb_device" % (label, c)
    for k, x in enumerate(E):
        X = P[k : k + 1]
        got = lincomb([P], X, [1], [0], m, None)
        compare("%s k=1 stride 1 (out = p x)" % ep, got, [e * x * ri % r for e in E], r, lambda j: (E[j], x))
        got = lincomb([P], X, [1], [0], m, Rev)
        compare("%s k=1 stride 1 accumulate (out = init + p x)" % ep, got, [(v + e * x * ri) % r for v, e in zip(rev, E)], r,
                lambda j: (rev[j], E[j], x))
    got = lincomb([P] * m, P, [m] * m, list(range(m)), m * m, None)
    compare("%s k=%d stride %d offsets 0..%d (out[j m + i] = p[j] s_i)" % (ep, m, m, m - 1), got,
            [E[j] * E[i] * ri % r for j in range(m) for i in range(m)], r, lambda t: (E[t // m], E[t % m]))


# ------------------------------------------------------------------------------------------
# B. sum and difference: n = 2 transforms on every ordered pair
# ------------------------------------------------------------------------------------------


def butterfly_pairs(c):
    E = extremes(c)
    return [(x, y) for x in E for y in E]


def check_butterflies(c, fft_pairs, label):
    """fft_pairs(buf, inverse, decimation) returns buf ((2 p, w) limbs) transformed as p independent FFTs of n = 2.  Forward
    DIF and DIT give [x + y, x - y]; FFTInverse gives the same times 1/2"""
    f = fr(c)
    r, w = f.q, f.limbs
    pairs = butterfly_pairs(c)
    buf = pack([v for p in pairs for v in p], w)
    half = (r + 1) // 2
    for inverse in (False, True):
        s = half if inverse else 1
        want = [v for x, y in pairs for v in ((x + y) * s % r, (x - y) * s % r)]
        for dec in (DIF, DIT):
            got = fft_pairs(buf.copy(), inverse, dec)
            compare("%s %s gmsm_fft_device n=2 %s %s (slot 2 i: x + y, 2 i + 1: x - y%s)" % (
                label, c, "FFTInverse" if inverse else "FFT", "DIF" if dec == DIF else "DIT", ", times 1/2" if inverse else ""),
                got, want, r, lambda t: pairs[t // 2])


# ------------------------------------------------------------------------------------------
# C. every FFT variant on extreme vectors, against the oracle
# ------------------------------------------------------------------------------------------


def fft_vectors(c, n):
    """arith_stress's butterfly inputs plus the extremes cycled over the vector"""
    f = fr(c)
    E = extremes(c)
    out = S.fft_inputs(f, n)
    out["extremes_cycled"] = [E[i % len(E)] for i in range(n)]
    return out


VARIANTS = [(dec, coset, inverse) for dec in (DIT, DIF) for coset in (False, True) for inverse in (False, True)]


def variant_name(dec, coset, inverse):
    return "%s %s%s" % ("FFTInverse" if inverse else "FFT", "DIF" if dec == DIF else "DIT", " coset" if coset else "")


def check_fft_extremes(c, logn, fft, label):
    """fft(a, inverse, decimation, coset) returns the transform of the (n, w) limbs a; every variant on every fft_vectors input"""
    f = fr(c)
    n = 1 << logn
    od = domain(c, n)
    for name, vals in fft_vectors(c, n).items():
        for dec, coset, inverse in VARIANTS:
            got = fft(pack(vals, f.limbs), inverse, dec, coset)
            want = (od.fft_inverse if inverse else od.fft)(vals, dec, coset)
            compare("%s %s logn=%d %s, input %s" % (label, c, logn, variant_name(dec, coset, inverse), name), got, want, f.q,
                    lambda i: (), kind="the input vector named above")


# ------------------------------------------------------------------------------------------
# D. closed forms of sparse vectors at production sizes
# ------------------------------------------------------------------------------------------


def sparse_terms(c, n, rng):
    """8 (logical index, stored value) terms: indices 0, 1, n/2, n - 1 and four random ones, values non-zero extremes"""
    E = [e for e in extremes(c) if e]
    idx = [0, 1, n // 2, n - 1]
    while len(idx) < 8:
        k = rng.randrange(2, n - 1)
        if k not in idx:
            idx.append(k)
    return [(k, rng.choice(E)) for k in idx]


def check_positions(n, rng, count=2048):
    """logical output indices: every 2^b, 2^b - 1 and n - 1 - 2^b, 0, n - 1, then random ones up to count"""
    logn = n.bit_length() - 1
    pos = {0, n - 1}
    for b in range(logn):
        pos |= {1 << b, (1 << b) - 1, n - 1 - (1 << b)}
    while len(pos) < count:
        pos.add(rng.randrange(n))
    return sorted(pos)


def closed_form(od, terms, positions, inverse, coset):
    """stored outputs at the logical indices `positions` of the transform of the sparse vector `terms` (logical index, stored
    value): FFT gives sum_k c_k u^k w^(i k) (u^k on a coset only); FFTInverse gives n^-1 u^-i sum_k e_k w^-(i k)"""
    r, n = od.q, od.cardinality
    g = od.generator_inv if inverse else od.generator
    if coset and not inverse:
        terms = [(k, v * pow(od.shift, k, r) % r) for k, v in terms]
    out = []
    for i in positions:
        acc = sum(v * pow(g, i * k % n, r) for k, v in terms) % r
        if inverse:
            acc = acc * od.cardinality_inv % r
            if coset:
                acc = acc * pow(od.shift_inv, i, r) % r
        out.append(acc)
    return out


# ------------------------------------------------------------------------------------------
# E. the opening scan
# ------------------------------------------------------------------------------------------


def scan_points(c, t, rng):
    """(name, plain a): random, 0, 1, r - 1, a primitive t-th root of unity (every carry level's multiplier a^(t^l) is 1) and a
    primitive 2t-th root (the first level's is -1)"""
    r = fr(c).q
    return [("random", rng.randrange(r)), ("0", 0), ("1", 1), ("r-1", r - 1), ("t-th root", domain(c, t).generator),
            ("2t-th root", domain(c, 2 * t).generator)]


def scan_ref(f, a, r):
    """b[n-1] = f[n-1], b[i] = f[i] + a b[i+1] on stored f with a plain: b[0] = f(a), b[1:] = (f - f(a)) / (X - a), stored"""
    b = list(f)
    acc = 0
    for i in range(len(f) - 1, -1, -1):
        acc = (f[i] + a * acc) % r
        b[i] = acc
    return b


def random_stored(c, n, seed):
    r = fr(c).q
    rng = random.Random(seed)
    return [rng.randrange(r) for _ in range(n)]


def check_scan(c, coeffs, points, div, label):
    """div(f, a, quotient) returns (f(a) as (1, w) limbs, h as (n - 1, w) limbs or None) for the (n, w) limbs f and the stored
    point a ((1, w) limbs).  Compares f(a) and the whole quotient, and f(a) from the evaluation-only path"""
    fld = fr(c)
    r, w = fld.q, fld.limbs
    n = len(coeffs)
    F = pack(coeffs, w)
    for name, a in points:
        A = pack([fld.to_mont(a)], w)
        b = scan_ref(coeffs, a, r)
        what = "%s %s gmsm_fr_poly_div_x_minus_a_device n=%d a=%s" % (label, c, n, name)
        ops = lambda i: (a, coeffs[i])                     # noqa: E731
        kind = "point a (plain), f[i] (stored)"
        fa, h = div(F, A, True)
        compare(what + " f(a)", fa, b[:1], r, ops, kind)
        compare(what + " quotient h[i] = b[i + 1]", h, b[1:], r, lambda i: (a, coeffs[i + 1]), kind)
        fa, _ = div(F, A, False)
        compare(what + " f(a), evaluation only", fa, b[:1], r, ops, kind)
