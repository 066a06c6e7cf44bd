"""The sort-by-bucket pipeline on the device -- K1 k_skew_probe / k_digits_hist in plain and rank mode, the K1b scan, the K1c
scatter (part of it on the auxiliary stream), the K2 accumulate (one launch, or two parts around the scatter), the K2b carry
levels, the K2' bucket merge of pipelined batches, the K3 segments and tree and the K4 finalize -- at shapes the heuristics
never pick, for all thirteen groups.

The GMSM_* experiment knobs force the shapes: GMSM_K1_MODE (counting-sort mode without the sampling pass), GMSM_SPLIT_W
(windows scattered before the accumulate), GMSM_ACC_K (chunk length), GMSM_K2_FIRST / GMSM_K2 (carry run lengths),
GMSM_SEG_L (segment length), GMSM_TABLE_PASSES (bucket-range passes of the window-table scatter), GMSM_CHUNKS (batches of
a host call), GMSM_AFFINE (batch-affine accumulation).  A context reads them when it is created; every case asserts through
the launch count that the shape it asked for is the one that ran.

Two oracles, both bit-exact on the affine limbs:
  * closed forms at large n: the bases are [w_i]B with known w_i (generated on the device), so the partial of window j is
    [sum_i d_ij w_i]B, d_ij the signed digits of cref.partition_scalars -- every partial is checked, then the finalize;
  * cref.msm at small n for the inputs with infinities, duplicates and P / -P pairs (gpu_common.make_inputs)."""
import ctypes
import os
import random
from importlib import import_module

import numpy as np
import pytest

from oracle import cref
from oracle import oracle as O
from tests.gpu_common import make_inputs

pytestmark = pytest.mark.gpu

GROUPS = list(O.GROUPS)
# the groups whose scatter can run under the accumulate (coordinate field of at most 48 bytes)
SPLIT = ["bn254_g1", "bls12381_g1", "bls12377_g1", "secp256k1_g1", "bls24315_g1", "bls24317_g1"]
NO_SPLIT = [g for g in GROUPS if g not in SPLIT]
BW6 = ["bw6761_g1", "bw6761_g2", "bw6633_g1", "bw6633_g2"]   # lane-parallel tail kernels by default
KNOBS = ["GMSM_AFFINE", "GMSM_QUAD", "GMSM_QUAD_MAX", "GMSM_SPLIT_W", "GMSM_TABLE_PASSES", "GMSM_K2_FIRST", "GMSM_K2",
         "GMSM_SEG_L", "GMSM_TABLE_SEG_L", "GMSM_ACC_K", "GMSM_K1_MODE", "GMSM_CHUNKS", "GMSM_SCHEDULE", "GMSM_C", "GMSM_TABLE_C"]
NCPU = os.cpu_count() or 1
NUM_SMS = 132   # GMSM_NUM_SMS (hd.cuh): pick_K's grid size


def _pkg():
    import gnark_crypto_b200 as pkg

    return pkg


def _native():
    return import_module("gnark-crypto_b200._native")


@pytest.fixture(autouse=True)
def _default_knobs(monkeypatch):
    """every case starts from the engine's defaults, whatever the caller's environment holds"""
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)


def _set(monkeypatch, **kv):
    for k, v in kv.items():
        if v is None:
            monkeypatch.delenv("GMSM_" + k, raising=False)
        else:
            monkeypatch.setenv("GMSM_" + k, str(v))


# ---------------------------------------------------------------------------------------------------------------------
# the launch sequence of run_accumulate / run_bucket_reduce (engine_impl.cuh), restated
# ---------------------------------------------------------------------------------------------------------------------
def _plan(g, c):
    bits = O.GROUPS[g].fr.bits
    nwin = -(-bits // c)
    last_c = c + 1 - (nwin * c - bits)
    return nwin, 1 << (c - 1), 1 << (last_c - 1)


def _pick_K(total):
    K = 4
    while K < 256 and K < total / (NUM_SMS * 512.0 * 8.0):
        K <<= 1
    return K


def _launches(g, n, c, *, tables=False, passes=0, K=0, K2_first=4, K2=16, L=0, split=0, k1_forced=False, msm=True, quad=None):
    """kernel launches of one device-level call (window sums, or + 1 for the finalize of a whole MSM) in the
    extended-Jacobian mode; knob values as the context holds them (0 = the default)"""
    nwin, nb, nb_last = _plan(g, c)
    nb_total = max(nb, nb_last) if tables else (nwin - 1) * nb + nb_last
    out = (1 if k1_forced else 2) + 3                       # probe + digits, scan
    if tables:
        npass = passes or int(min(16.0, max(4.0, n * nwin * 4.0 / 200e6 + 0.5)))
        rsz = -(-nb_total // npass)
        out += sum(1 for r in range(npass) if r * rsz < nb_total)
        sw = split or 1
    else:
        npass = nwin
        out += nwin
        sw = split or 2
    fbytes = 8 * O.GROUPS[g].K.words
    two_part = fbytes <= 48 and nwin >= 6 and n >= (1 << 16) and min(sw, npass) < npass
    out += 2 if two_part else 1
    K = K or _pick_K(n * nwin)
    n_in, first = -(-n * nwin // K), True
    while n_in > 1:
        n_in = -(-n_in // (K2_first if first else K2))
        first = False
        out += 1
    if quad is None:
        quad = (1, 20000) if g in BW6 else (0, 0)
    L = L or (64 if tables else 32)
    per, red = -(-max(nb, nb_last) // L), 1 if tables else nwin
    out += 1                                                # segments
    while per > 1:
        R = 16 if (quad[0] > 0 and red * per <= quad[1]) else 128
        per = -(-per // R)
        out += 1
    return out + (1 if msm else 0)


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
_BASES = {}


def _base(g):
    G = O.GROUPS[g]
    return G.encode_affine([G.scalar_mul(G.gen, 0xC0FFEE)])[0]


def _multiples(g, n):
    """host copy of [i + 1]B, i < n, generated on the device (cached)"""
    if (g, n) not in _BASES:
        eng = _pkg().Engine(g, 1, c=8)
        try:
            _BASES[(g, n)] = eng.generate_multiples(_base(g), 1, n).cpu().numpy().view(np.uint64).reshape(n, -1).copy()
        finally:
            eng.close()
    return _BASES[(g, n)]


def _neg(g, pts):
    """-P for every affine point (y -> q - y on the stored Montgomery limbs, each Fp component; infinity stays 0)"""
    G = O.GROUPS[g]
    w = G.K.words
    comps = 2 if isinstance(G.K, O.Fp2Ops) else 1
    lw = w // comps
    out = pts.copy()
    for k in range(comps):
        y = pts[:, w + k * lw: w + (k + 1) * lw]
        borrow = np.zeros(y.shape[0], dtype=np.uint64)
        neg = np.empty_like(y)
        for li in range(lw):
            ql = np.uint64((G.K.q >> (64 * li)) & 0xFFFFFFFFFFFFFFFF)
            neg[:, li] = ql - y[:, li] - borrow
            borrow = ((y[:, li] > ql) | ((y[:, li] == ql) & (borrow == 1))).astype(np.uint64)
        neg[~y.any(axis=1)] = 0
        out[:, w + k * lw: w + (k + 1) * lw] = neg
    return out


def _enc(g, ks):
    return O.GROUPS[g].encode_scalars(ks)


def _tiled(g, n, ks):
    e = _enc(g, ks)
    return np.ascontiguousarray(np.resize(e, (n, e.shape[1])))


FAMILIES = ["random", "smallvalues", "redundancy", "one_bucket", "equal_points", "r_minus_1", "zero", "low_empty",
            "high_empty", "pm_pairs"]
SKEWED = ["smallvalues", "redundancy", "one_bucket", "equal_points", "r_minus_1", "pm_pairs"]


def _family(g, kind, n, c=0, split=0, seed=1):
    """(Montgomery scalars, weights w_i, points kind): the MSM is sum_i s_i [w_i]B.  points kind: "mult" = [i + 1]B,
    "equal" = B everywhere, "pm" = [k + 1]B next to -[k + 1]B"""
    G = O.GROUPS[g]
    r = G.fr.q
    s = cref.random_scalars(g, n, seed)
    w = np.arange(1, n + 1, dtype=np.int64)
    pk = "mult"
    rng = random.Random(seed)
    if kind == "smallvalues":
        s[::5] = _enc(g, [1])[0]
    elif kind == "redundancy":
        s = np.ascontiguousarray(s[(np.arange(n) // 100) * 100])
    elif kind == "one_bucket":
        s[:] = s[0]
    elif kind == "equal_points":
        w[:] = 1
        pk = "equal"
    elif kind == "r_minus_1":
        s[:] = _enc(g, [r - 1])[0]
    elif kind == "zero":
        s[:] = 0
    elif kind == "low_empty":     # multiples of 2^(c*split): windows below `split` hold no entry
        s = _tiled(g, n, [rng.randrange(1, max(2, r >> (c * split))) << (c * split) for _ in range(2048)])
    elif kind == "high_empty":    # below 2^(c*split - 2): no digit reaches window `split`, not even by a borrow
        s = _tiled(g, n, [rng.randrange(1, 1 << (c * split - 2)) for _ in range(2048)])
    elif kind == "pm_pairs":      # P, -P with one scalar, side by side in one bucket per window; an unpaired tail
        m = (n - 37) // 2 * 2
        s[:m] = s[0]
        w[1:m:2] = -w[0:m:2]
        pk = "pm"
    else:
        assert kind == "random"
    return s, w, pk


def _points(g, n, pk):
    pts = _multiples(g, n)
    if pk == "equal":
        return np.ascontiguousarray(np.repeat(pts[:1], n, axis=0))
    if pk == "pm":
        m = (n - 37) // 2 * 2
        out = pts.copy()
        out[1:m:2] = _neg(g, pts[0:m:2])
        return out
    return pts


def _signed_digits(g, s, c):
    d = cref.partition_scalars(g, s, c).astype(np.int64)
    return np.where(d & 1 == 0, d >> 1, -((d >> 1) + 1))


def _xyzz_to_affine(g, limbs):
    G = O.GROUPS[g]
    w = G.K.words
    v = [G.K.decode([int(x) for x in limbs[k * w: (k + 1) * w]]) for k in range(4)]
    return G.encode_affine([G.xyzz_to_affine(v)])[0]


def _check_window_sums(g, eng, d_pts, s, wts, what):
    """every window partial against [sum_i d_ij w_i]B, then the finalize against the whole MSM"""
    G = O.GROUPS[g]
    r = G.fr.q
    n = s.shape[0]
    base = _base(g)
    part = eng.window_sums(d_pts, eng.to_device(s), n)
    host = part.cpu().numpy().view(np.uint64).reshape(eng.nwin, -1)
    ks = _signed_digits(g, s, eng.c) @ wts            # |d| <= 2^24, |w| <= n < 2^18, < 2^18 terms: exact in int64
    assert ks.shape == (eng.nwin,)
    for j in range(eng.nwin):
        want = cref.scalar_mul(g, base, int(ks[j]) % r)
        assert np.array_equal(_xyzz_to_affine(g, host[j]), want), (what, "window", j)
    total = sum(int(k) << (eng.c * j) for j, k in enumerate(ks)) % r
    jac = eng.finalize(part, 1).cpu().numpy().view(np.uint64)
    a = base.size
    assert np.array_equal(jac[:a], cref.scalar_mul(g, base, total)), (what, "finalize")


# ---------------------------------------------------------------------------------------------------------------------
# 1. the host entry points rebuild their context when a knob changes
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("knob,first", [("AFFINE", "1"), ("K1_MODE", "rank"), ("ACC_K", "256")])
def test_oneshot_context_follows_the_environment(knob, first, monkeypatch):
    """a one-shot call under a knob, then one at the same n without it: the session keeps its context between calls, so
    the second call must build a new one -- the launch counts differ -- and both results are exact"""
    pkg = _pkg()
    L = _native().lib()
    g = "bn254_g1"
    pts, s = make_inputs(g, 3000, 91)
    want, _, _, _ = cref.msm(g, pts, s, c=0, nthreads=NCPU)
    launches = []
    for v in (first, None, first):
        _set(monkeypatch, **{knob: v})
        assert np.array_equal(pkg.G1Affine().MultiExp(pts, s, pkg.MultiExpConfig()).limbs, want), (knob, v)
        launches.append(L.gmsm_last_oneshot_launches())
    assert launches[0] != launches[1] and launches[2] == launches[0], (knob, launches)


# ---------------------------------------------------------------------------------------------------------------------
# 2. per-window closed forms at large n
# ---------------------------------------------------------------------------------------------------------------------
def _window_c(g, n):
    return _native().lib().gmsm_choose_window_bits(_pkg().CURVES[g], ctypes.c_size_t(n))


@pytest.mark.parametrize("g", SPLIT)
@pytest.mark.parametrize("mode", ["plain", "rank"])
def test_window_sums_closed_form_split_scatter(g, mode, monkeypatch):
    """the six groups whose scatter overlaps the accumulate, at n = 2^17 + 13: both counting-sort modes, 1, 2 and W - 1
    windows scattered ahead (two accumulate parts), every scalar family -- including scalars whose low windows are empty
    (part 1 has no chunk) and whose high windows are empty (part 2 holds only empty chunks)"""
    n = (1 << 17) + 13
    c = _window_c(g, n)
    nwin = _plan(g, c)[0]
    for split in sorted({1, 2, nwin - 1}):
        _set(monkeypatch, K1_MODE=mode, SPLIT_W=split)
        eng = _pkg().Engine(g, n, c=c)
        try:
            assert eng.nwin == nwin
            dev = {}
            for kind in FAMILIES:
                s, wts, pk = _family(g, kind, n, c, split, seed=split)
                if kind == "low_empty":
                    assert not _signed_digits(g, s[:64], c)[:split].any()
                if kind == "high_empty":
                    assert not _signed_digits(g, s[:4096], c)[split:].any()
                if pk not in dev:
                    dev[pk] = eng.to_device(_points(g, n, pk))
                _check_window_sums(g, eng, dev[pk], s, wts, (g, mode, split, kind))
                assert eng.last_launches == _launches(g, n, c, split=split, k1_forced=True, msm=False)
        finally:
            eng.close()


@pytest.mark.parametrize("g", NO_SPLIT)
@pytest.mark.parametrize("mode", ["plain", "rank"])
def test_window_sums_closed_form_other_groups(g, mode, monkeypatch):
    """the seven groups whose scatter runs ahead of the accumulate (G2 groups at 255 registers, bw6), the skewed families,
    both counting-sort modes"""
    n = (1 << 16) + 3
    c = _window_c(g, n)
    _set(monkeypatch, K1_MODE=mode)
    eng = _pkg().Engine(g, n, c=c)
    try:
        dev = {}
        for kind in SKEWED:
            s, wts, pk = _family(g, kind, n, seed=5)
            if pk not in dev:
                dev[pk] = eng.to_device(_points(g, n, pk))
            _check_window_sums(g, eng, dev[pk], s, wts, (g, mode, kind))
            assert eng.last_launches == _launches(g, n, c, k1_forced=True, msm=False)
    finally:
        eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. forced shapes against cref.msm
# ---------------------------------------------------------------------------------------------------------------------
# (c, GMSM_ACC_K, GMSM_K2_FIRST, GMSM_K2, GMSM_SEG_L, GMSM_K1_MODE): every value of every knob, chunk lengths 1..3 where
# each bucket spans chunks and the carry levels go deepest, a segment length that is not a power of two, one segment
# longer than a window
SHAPES = [(5, 1, 2, 2, 2, "plain"), (10, 2, 64, 2, 3, "rank"), (13, 3, 2, 64, 31, "plain"), (16, 256, 64, 64, 1024, "rank"),
          (8, 1, 64, 64, 31, "rank"), (11, 3, 2, 2, 1024, "plain")]


@pytest.mark.parametrize("g", GROUPS)
def test_forced_shapes_agree_with_oracle(g, monkeypatch):
    """the cross-test inputs (infinities, duplicates, P / -P, zero scalars) and every scalar equal (one bucket per window
    over all the chunks), under chunk lengths, carry run lengths, segment lengths and counting-sort modes the heuristics
    never pick"""
    n = 2500
    pts, s = make_inputs(g, n, 606)
    s_eq = np.ascontiguousarray(np.repeat(s[3:4], n, axis=0))
    want = cref.msm(g, pts, s, c=0, nthreads=NCPU)[0]
    want_eq = cref.msm(g, pts, s_eq, c=0, nthreads=NCPU)[0]
    a = pts.shape[1]
    for c, K, K2f, K2, L, mode in SHAPES:
        _set(monkeypatch, ACC_K=K, K2_FIRST=K2f, K2=K2, SEG_L=L, K1_MODE=mode)
        eng = _pkg().Engine(g, n, c=c)
        try:
            dp = eng.to_device(pts)
            for sc, wn in ((s, want), (s_eq, want_eq)):
                got = eng.msm_host_result(dp, eng.to_device(sc), n)
                assert np.array_equal(got[:a], wn), (g, c, K, K2f, K2, L, mode)
                assert eng.last_launches == _launches(g, n, c, K=K, K2_first=K2f, K2=K2, L=L, k1_forced=True), (c, K)
        finally:
            eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4. batch-affine accumulation
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("g", GROUPS)
def test_batch_affine_agrees_with_oracle(g, monkeypatch):
    """GMSM_AFFINE=1 for every group: random scalars with the cross-test ingredients, one bucket per window (the deepest
    tree), all points equal (the doubling branch at every level), P / -P with one scalar (cancellation inside the tree)"""
    n = 2000
    pts, s = make_inputs(g, n, 707)
    cases = [("random", pts, s)]
    s1 = np.ascontiguousarray(np.repeat(s[3:4], n, axis=0))
    cases.append(("one_bucket", pts, s1))
    cases.append(("equal_points", np.ascontiguousarray(np.repeat(pts[3:4], n, axis=0)), s))
    p2, s2 = make_inputs(g, n, 708, specials=False)
    m = (n - 37) // 2 * 2
    p2[1:m:2] = _neg(g, p2[0:m:2])
    s2[:m] = s2[0]
    cases.append(("pm_pairs", p2, s2))
    G = O.GROUPS[g]
    assert np.array_equal(_neg(g, p2[:4:2]), G.encode_affine([G.aff_neg(q) for q in G.decode_affine(p2[:4:2])]))
    _set(monkeypatch, AFFINE=1)
    for kind, P, S in cases:
        want = cref.msm(g, P, S, c=0, nthreads=NCPU)[0]
        for c in (7, 13):
            eng = _pkg().Engine(g, n, c=c)
            try:
                got = eng.msm_host_result(eng.to_device(P), eng.to_device(S), n)
                assert np.array_equal(got[: P.shape[1]], want), (g, kind, c)
            finally:
                eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5. window tables
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("g", GROUPS)
def test_window_tables_passes_and_modes(g, monkeypatch):
    """one shared bucket set at two widths: 1 and 3 bucket-range passes and more passes than buckets (empty ranges),
    the scatter split ahead of the accumulate for the six groups that can, both counting-sort modes, skewed families;
    closed form [sum (i + 1) s_i]B at n = 2^16 + 5"""
    n = (1 << 16) + 5
    pts = _multiples(g, n)
    base = _base(g)
    a = base.size
    r = O.GROUPS[g].fr.q
    fams = []
    for kind in ("random", "smallvalues", "redundancy", "one_bucket"):
        s, _, _ = _family(g, kind, n, seed=9)
        fams.append((kind, s, cref.scalar_mul(g, base, cref.dot_index(g, s, 1) % r)))
    for c in (6, 13):
        nb_total = max(_plan(g, c)[1:])
        eng0 = _pkg().Engine(g, n, c=c, tables=True)
        try:
            tab = eng0.build_tables(eng0.to_device(pts), n)
        finally:
            eng0.close()
        for passes in (1, 3, 200):
            assert c != 6 or passes < 200 or passes > nb_total
            for mode in ("plain", "rank"):
                _set(monkeypatch, TABLE_PASSES=passes, K1_MODE=mode)
                eng = _pkg().Engine(g, n, c=c, tables=True)
                try:
                    for kind, s, want in fams:
                        got = eng.msm_tables(tab, n, eng.to_device(s), n).cpu().numpy().view(np.uint64)
                        assert np.array_equal(got[:a], want), (g, c, passes, mode, kind)
                        assert eng.last_launches == _launches(g, n, c, tables=True, passes=passes, k1_forced=True)
                finally:
                    eng.close()
        del tab


# ---------------------------------------------------------------------------------------------------------------------
# 6. pipelined host calls
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("g", GROUPS)
def test_pipelined_batches_mix_plain_and_rank(g, monkeypatch):
    """a host call cut into 2, 7 or 16 batches over one bucket array (scratch buckets + merge); exactly one batch has all
    its scalars equal, so the sampling pass puts it in rank mode and the others in plain mode; one-shot and resident
    bases, ragged n"""
    pkg = _pkg()
    mx = import_module("gnark-crypto_b200.multiexp")
    n = 40013
    pts = _multiples(g, n)
    base = _base(g)
    a = base.size
    r = O.GROUPS[g].fr.q
    A1, _, A2, _ = pkg.curve_package(g.split("_")[0])
    Aff = A1 if g.endswith("g1") else A2
    rb = mx.ResidentBases(g, pts)
    try:
        for nch in (2, 7, 16):
            s = cref.random_scalars(g, n, 100 + nch)
            lo, hi = n // nch, 2 * (n // nch)            # batch 1 of pipeline_run's equal cut
            s[lo:hi] = s[lo]
            want = cref.scalar_mul(g, base, cref.dot_index(g, s, 1) % r)
            _set(monkeypatch, CHUNKS=nch)
            assert np.array_equal(Aff().MultiExp(pts, s, pkg.MultiExpConfig()).limbs, want), (g, nch, "one-shot")
            assert np.array_equal(rb.MultiExp(s)[:a], want), (g, nch, "resident")
    finally:
        rb.close()
