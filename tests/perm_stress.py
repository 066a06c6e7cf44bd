"""Extreme operands, adversarial keys, references and checks for the Fr kernels of permutation.Prove and plookup.ProveLookupVector of
the seven pairing curves (perm_kernels.cuh, plookup_kernels.cuh): the tile batch inversion and its fp_inv, the ratio kernels, the
multi-level prefix-product scan, both quotient numerators and the radix sort.

Shared by tests/test_gpu_perm_stress.py (the sm_90a kernels of fft.cu through the C ABI) and tests/test_perm_stress_cpu.py (the
same kernels on the CPU through tests/emu at forced small tiles).  Not a conftest.

Values are STORED values, as in tests/fr_stress.py: the Montgomery integer m < r a kernel reads, standing for m R^-1.  The
references are plain big-int restatements on those integers -- pow(x, -1, r), sequential products, per-position formulas -- and
never the emulated kernels.  Ratios of two stored values are plain values (R cancels), so the prefix products run on stored
integers with one multiplication per element: z_stored[k] = R prod_{j<k} ratio_j.  Long vectors are drawn from small pools of
values with random indices, so that a reference costs one table look-up and one product per element while tile products still
differ from tile to tile.  Outputs are compared limb for limb, so they must also be canonical.  A failure names the field, the
entry point, the case, the index and the operands as stored decimal integers, so that it can be replayed through the CPU twin."""
import random

import numpy as np

from tests import fr_stress as R

CURVES = R.CURVES
FIELD = R.FIELD
SCAN_TILE = R.TILE            # elements per tile of the prefix-product scan in fft.cu, by fr.Bytes (poly_log_l + poly_log_b)
INV_TILE, INV_THREADS = 512, 256   # PERM_INV_LOG_T, PERM_INV_THREADS of perm_kernels.cuh
fr, pack, unpack, bitrev, domain, extremes = R.fr, R.pack, R.unpack, R.bitrev, R.domain, R.extremes


def two_adicity(c):
    q = fr(c).q
    return ((q - 1) & -(q - 1)).bit_length() - 1


def scan_tile(c):
    return SCAN_TILE[8 * fr(c).limbs]


def inv_stored(f, m):
    """stored inverse of the stored m (zero -> zero): (m R^-1)^-1 R = R^2 m^-1"""
    return f.R2 * pow(m, -1, f.q) % f.q if m else 0


def compare_packed(what, got, exp, r, operands, kind="stored operands (decimal Montgomery limbs)", index=None):
    """R.compare on an expected (m, w) limb array (long vectors: no per-element packing)"""
    got = np.ascontiguousarray(got, dtype=np.uint64).reshape(exp.shape)
    if np.array_equal(got, exp):
        return
    i = int(np.nonzero((got != exp).any(axis=1))[0][0])
    g, want = unpack(got[i : i + 1])[0], unpack(exp[i : i + 1])[0]
    R.S._fail(what + ("" if g < r else " (non-canonical output)"), i if index is None else index(i), operands(i), g, want, kind)


def random_canonical(c, n, seed):
    """(n, w) limbs of uniform values below 2^(bits - 1) < r (numpy, no big ints)"""
    f = fr(c)
    g = np.random.default_rng(seed)
    a = g.integers(0, 2**63, size=(n, f.limbs), dtype=np.uint64) * np.uint64(2) + g.integers(0, 2, size=(n, f.limbs), dtype=np.uint64)
    top = (f.bits - 1) - 64 * (f.limbs - 1)
    a[:, -1] &= np.uint64((1 << top) - 1)
    return a


def map_refs(mapper, fn, jobs):
    """mapper(fn, jobs) -> iterable of results, in order (map, or a process pool's map for the long references)"""
    return (mapper or map)(fn, jobs)


# ------------------------------------------------------------------------------------------
# A. the tile batch inversion as the Fr fp_inv
# ------------------------------------------------------------------------------------------


def check_batch_invert(c, invert, label, rng, log_t=9, threads=INV_THREADS, n_random=4096):
    """invert(A, in_place) returns gmsm_fr_batch_invert_device's output for the (n, w) limbs A (out of place, or in place).
    Every extreme alone in its own tile with every other leaf one (the tile root is the extreme: fp_inv of exactly that value),
    every extreme at n = 1, n_random random values one per tile, and dense tiles: all r - 1, all zero, zeros at the slots the
    thread mask splits on (j = 0, B - 1, B, T - 1 with j = tid + B q) among extremes"""
    f = fr(c)
    r, w, one = f.q, f.limbs, f.Rmod
    T = 1 << log_t
    E = extremes(c)
    ep = "%s %s gmsm_fr_batch_invert_device T=%d" % (label, c, T)

    def run(name, A, exp, ops):
        for in_place in (False, True):
            got = invert(A.copy(), in_place)
            compare_packed("%s %s (%s, n=%d)" % (ep, name, "in place" if in_place else "out of place", len(A)), got, exp, r, ops)

    def sparse(name, slots, vals):
        n = T * len(vals)
        A = np.tile(pack([one], w), (n, 1))
        X = A.copy()
        A[slots] = pack(vals, w)
        X[slots] = pack([inv_stored(f, v) for v in vals], w)
        at = dict(zip(slots.tolist(), vals))
        run(name, A, X, lambda i: (at.get(i, one),))

    slots = np.arange(len(E)) * T + (np.arange(len(E)) * 37) % T
    sparse("every extreme alone in its tile, other leaves one", slots, E)
    rnd = [rng.randrange(1, r) for _ in range(n_random)]
    slots = np.arange(n_random) * T + np.array([rng.randrange(T) for _ in range(n_random)])
    sparse("%d random values one per tile, other leaves one" % n_random, slots, rnd)
    for x in E:
        run("n=1", pack([x], w), pack([inv_stored(f, x)], w), lambda i: (x,))
    nz = [e for e in E if e]
    split = [j for j in (0, threads - 1, threads, T - 1) if j < T]
    dense = {"all r-1": [r - 1] * (2 * T + 3), "all zero": [0] * (T + 5), "all one": [one] * T,
             "zeros at j in %s among extremes" % split: [0 if j % T in split else nz[j % len(nz)] for j in range(2 * T)]}
    for name, vals in dense.items():
        run(name, pack(vals, w), pack([inv_stored(f, v) for v in vals], w), lambda i: (vals[i],))


# ------------------------------------------------------------------------------------------
# B. the permutation accumulation across scan levels
# ------------------------------------------------------------------------------------------


def level_positions(n, t):
    """k at the scan's level boundaries for a tile of t: T - 1, T, T^2 - 1, T^2, T^2 + T - 1, n - 2, n - 1 (those below n - 1)"""
    return sorted({k for k in (t - 1, t, t * t - 1, t * t, t * t + t - 1, n - 2, n - 1) if 0 <= k < n})


class Pools:
    """a vector of n stored values drawn from `vals` by the index array `idx`; special positions hold values of their own"""

    def __init__(self, r, n, rng, g, size, special=()):
        self.vals = [rng.randrange(1, r) for _ in range(size + len(special))]
        self.idx = g.integers(0, size, n)
        for s, k in enumerate(special):
            self.idx[k] = size + s

    def limbs(self, w):
        return pack(self.vals, w)[self.idx]

    def at(self, k):
        return self.vals[self.idx[k]]


def perm_accumulate_ref(job):
    """z_lin[k] = prod_{j<k} (E - t1[j]) (E - t2[j])^-1 (zero -> zero), stored, natural order: an (n, w) limb array"""
    r, w, one, v1, i1, v2, i2, E = job
    n, m = len(i1), len(v2)
    inv = [pow((E - b) % r, -1, r) if (E - b) % r else 0 for b in v2]
    tab = [(E - a) * y % r for a in v1 for y in inv]
    cidx = (i1 * m + i2).tolist()
    out = [0] * n
    acc = out[0] = one
    for j in range(n - 1):
        acc = acc * tab[cidx[j]] % r
        if not acc:
            break
        out[j + 1] = acc
    return pack(out, w)


def perm_cases(c, n, t, seed, forced=True, eps_extremes=()):
    """t1, t2 (Pools) and the cases (name, stored eps, k or None): random eps, then eps = t2[k] for every level position k and
    eps = t1[k] for k = T - 1, T, T^2 and n - 1 (no zero may appear at k = n - 1: r[n - 1] is never read), then the given stored
    eps"""
    f = fr(c)
    rng, g = random.Random(seed), np.random.default_rng(seed)
    ks = level_positions(n, t) if forced else []
    t1, t2 = Pools(f.q, n, rng, g, 64, ks), Pools(f.q, n, rng, g, 64, ks)
    cases = [("random eps", rng.randrange(f.q), None)]
    for k in ks:
        cases.append(("eps = t2[%d]" % k, t2.at(k), k))
        if k in (t - 1, t, t * t, n - 1):
            cases.append(("eps = t1[%d]" % k, t1.at(k), k))
    cases += [("eps extreme %d" % e, e, None) for e in eps_extremes]
    return t1, t2, cases


def check_perm_accumulate(c, n, t, accumulate, label, seed, mapper=None, forced=True, eps_extremes=()):
    """accumulate(T1, T2, E) returns gmsm_fr_permutation_accumulate_device's output (bit-reversed) for (n, w) limbs and the stored
    eps ((1, w) limbs).  The whole vector is compared with the sequential reference"""
    f = fr(c)
    r, w = f.q, f.limbs
    logn = n.bit_length() - 1
    t1, t2, cases = perm_cases(c, n, t, seed, forced, eps_extremes)
    refs = map_refs(mapper, perm_accumulate_ref, [(r, w, f.Rmod, t1.vals, t1.idx, t2.vals, t2.idx, E) for _, E, _ in cases])
    nat = bitrev(np.arange(n, dtype=np.int64), logn)
    A1, A2 = t1.limbs(w), t2.limbs(w)
    for (name, E, k), exp in zip(cases, refs):
        got = accumulate(A1, A2, pack([E], w))[nat]
        if k == n - 1:
            assert exp.any(axis=1).all(), "%s: the reference has a zero" % name
        compare_packed("%s %s gmsm_fr_permutation_accumulate_device n=%d scan tile %d, %s (z_lin[k] at d_z[rev(k)])" % (
            label, c, n, t, name), got, exp, r, lambda i: (E, t1.at(i - 1), t2.at(i - 1)) if i else (E,),
            kind="eps, t1[k - 1], t2[k - 1]")


# ------------------------------------------------------------------------------------------
# C. the plookup accumulation
# ------------------------------------------------------------------------------------------


def plookup_accumulate_ref(job):
    """z[0] = 1, z[i+1] = z[i] (1+b)(g+f[i])(g(1+b)+t[i]+b t[i+1]) / ((g(1+b)+h1[i]+b h1[i+1])(g(1+b)+h2[i]+b h2[i+1])) with
    zero -> zero inversion, on plain beta, gamma and stored vectors, stored output: an (n, w) limb array"""
    r, w, one, rinv, (vf, fi), (vt, ti), (v1, i1), (v2, i2), beta, gamma = job
    n = len(fi)
    pl = lambda vs: [v * rinv % r for v in vs]                 # noqa: E731
    vf, vt, v1, v2 = pl(vf), pl(vt), pl(v1), pl(v2)
    opb = (1 + beta) % r
    gopb = gamma * opb % r
    pair = lambda vs: [(gopb + a + beta * b) % r for a in vs for b in vs]   # noqa: E731
    num = [opb * (gamma + a) % r * u % r for a in vf for u in pair(vt)]
    inv1 = [pow(x, -1, r) if x else 0 for x in pair(v1)]
    inv2 = [pow(x, -1, r) if x else 0 for x in pair(v2)]
    mt, m1, m2 = len(vt), len(v1), len(v2)
    xi = ((fi[:-1] * mt + ti[:-1]) * mt + ti[1:]).tolist()
    yi = (i1[:-1] * m1 + i1[1:]).tolist()
    zi = (i2[:-1] * m2 + i2[1:]).tolist()
    out = [0] * n
    acc = out[0] = one
    for j in range(n - 1):
        acc = acc * num[xi[j]] % r * inv1[yi[j]] % r * inv2[zi[j]] % r
        if not acc:
            break
        out[j + 1] = acc
    return pack(out, w)


def plookup_cases(c, n, t, seed, edges=True):
    """(name, f, t, h1, h2 pools, plain beta, plain gamma, k or None): random challenges; with edges, beta = r - 1 (1 + beta = 0),
    beta = 0, gamma = 0, and gamma zeroing the h1 factor of the denominator at k = T^2 - 1 and at k = T^2"""
    f = fr(c)
    r = f.q
    rng, g = random.Random(seed), np.random.default_rng(seed)
    ks = [k for k in (t * t - 1, t * t) if k + 1 < n] if edges else []
    sp = sorted({j for k in ks for j in (k, k + 1)})
    vf, vt = Pools(r, n, rng, g, 16), Pools(r, n, rng, g, 16)
    v1, v2 = Pools(r, n, rng, g, 16, sp), Pools(r, n, rng, g, 16)
    beta, gamma = rng.randrange(r), rng.randrange(r)
    cases = [("random beta, gamma", beta, gamma, None)]
    if edges:
        cases += [("beta = r - 1", r - 1, gamma, None), ("beta = 0", 0, gamma, None), ("gamma = 0", beta, 0, None)]
        for k in ks:
            h, hn = v1.at(k) * f.Rinv % r, v1.at(k + 1) * f.Rinv % r
            cases.append(("gamma zeroes the h1 factor at k = %d" % k, beta, -(h + beta * hn) * pow(1 + beta, -1, r) % r, k))
    return vf, vt, v1, v2, cases


def check_plookup_accumulate(c, n, t, accumulate, label, seed, mapper=None, edges=True):
    """accumulate(F, T, H1, H2, B, G) returns gmsm_fr_plookup_accumulate_device's output (natural order) for (n, w) limbs and the
    stored beta and gamma ((1, w) limbs); the whole vector against the sequential reference"""
    fl = fr(c)
    r, w = fl.q, fl.limbs
    vf, vt, v1, v2, cases = plookup_cases(c, n, t, seed, edges)
    vecs = [(p.vals, p.idx) for p in (vf, vt, v1, v2)]
    refs = map_refs(mapper, plookup_accumulate_ref, [(r, w, fl.Rmod, fl.Rinv, *vecs, b, g) for _, b, g, _ in cases])
    L = [p.limbs(w) for p in (vf, vt, v1, v2)]
    for (name, b, g, k), exp in zip(cases, refs):
        got = accumulate(*L, pack([fl.to_mont(b)], w), pack([fl.to_mont(g)], w))
        if k is not None:
            assert not exp[k + 1].any() and exp[k].any(), "%s: the forced zero is not at %d" % (name, k)
        compare_packed("%s %s gmsm_fr_plookup_accumulate_device n=%d scan tile %d, %s (plain beta %d, gamma %d)" % (
            label, c, n, t, name, b, g), got, exp, r,
            lambda i: tuple(p.at(j) for p in (vf, vt, v1, v2) for j in (i - 1, i) if 0 <= j < n) if i else (),
            kind="f[i-1], f[i], t[i-1], t[i], h1[i-1], h1[i], h2[i-1], h2[i] stored")


# ------------------------------------------------------------------------------------------
# D. both numerators at per-position references
# ------------------------------------------------------------------------------------------


def numerator_positions(n, rng, count=4096, tile=INV_TILE):
    """storage positions p: every p whose i = rev(p) is in {0, 1, 2, half - 1, half, half + 1, n - 3, n - 2, n - 1}, every 2^b and
    2^b - 1, the first and last slot of sampled tiles, then random ones up to count (all of them when n <= count)"""
    if n <= count:
        return list(range(n))
    logn, half = n.bit_length() - 1, n // 2
    pos = {bitrev(i, logn) for i in (0, 1, 2, half - 1, half, half + 1, n - 3, n - 2, n - 1)}
    for b in range(logn):
        pos |= {1 << b, (1 << b) - 1}
    for s in rng.sample(range(n // tile), min(128, n // tile)):
        pos |= {s * tile, s * tile + tile - 1}
    while len(pos) < count:
        pos.add(rng.randrange(n))
    return sorted(pos)


def _plain_rows(f, arr, rows):
    return [v * f.Rinv % f.q for v in unpack(arr[rows])]


class PermNumRef:
    """per-position restatement of evaluateFirstPartNumReverse, evaluateSecondPartNumReverse and the omega-fold (permutation.go:
    78-121, 206-214) at storage positions p, i = rev(p): out[p] = (omega (lz[p] - 1) (g^n - 1) / (g w^i - 1) + (eps - lt2[p])
    lz[rev(i + 1 mod n)] - (eps - lt1[p]) lz[p]) / (g^n - 1), all plain"""

    def __init__(self, c, n, LT1, LT2, LZ, positions):
        f = self.f = fr(c)
        r = f.q
        od = domain(c, n)
        logn = n.bit_length() - 1
        self.positions = positions
        ii = [bitrev(p, logn) for p in positions]
        nb = [bitrev((i + 1) % n, logn) for i in ii]
        self.lt1, self.lt2, self.lz = (_plain_rows(f, A, positions) for A in (LT1, LT2, LZ))
        self.lzn = _plain_rows(f, LZ, nb)
        g, w = od.shift, od.generator
        self.tn = (pow(g, n, r) - 1) % r
        self.tninv = pow(self.tn, -1, r)
        self.u = [pow((g * pow(w, i, r) - 1) % r, -1, r) for i in ii]

    def __call__(self, eps, omega):
        """stored outputs at the positions for stored eps, omega"""
        f = self.f
        r = f.q
        e, o = eps * f.Rinv % r, omega * f.Rinv % r
        out = []
        for a, b, z, zn, u in zip(self.lt1, self.lt2, self.lz, self.lzn, self.u):
            second = (z - 1) * u % r * self.tn % r
            first = (zn * (e - b) - z * (e - a)) % r
            out.append((o * second + first) % r * self.tninv % r * f.R % r)
        return out


class PlookupNumRef:
    """per-position restatement of evaluateNumBitReversed, evaluateZStartsByOneBitReversed, evaluateZEndsByOneBitReversed,
    evaluateOverlapH1h2BitReversed and computeQuotientCanonical's fold (vector.go:106-335) at storage positions p of the big
    domain (n = 2s), i = rev(p), q = rev(i + 2 mod n), x = shift w^i, gg = (w^2)^(n/2 - 1), xn = x^(n/2) - 1 = shift^(n/2) (-1)^i - 1"""

    def __init__(self, c, n, LZ, LH1, LH2, LT, LF, positions):
        f = self.f = fr(c)
        r = f.q
        od = domain(c, n)
        logn = n.bit_length() - 1
        ii = [bitrev(p, logn) for p in positions]
        qq = [bitrev((i + 2) % n, logn) for i in ii]
        self.p = [_plain_rows(f, A, positions) for A in (LZ, LH1, LH2, LT, LF)]
        self.q = [_plain_rows(f, A, qq) for A in (LZ, LH1, LH2, LT)]
        w, sh = od.generator, od.shift
        gg = pow(w * w % r, n // 2 - 1, r)
        ss = pow(sh, n // 2, r)
        xn = [(ss - 1) % r, -(ss + 1) % r]
        self.ctx = []
        for i in ii:
            x = sh * pow(w, i, r) % r
            xi = xn[i % 2]
            self.ctx.append((x, (x - gg) % r, xi, pow((x - 1) % r, -1, r), pow((x - gg) % r, -1, r), pow(xi, -1, r)))

    def __call__(self, beta, gamma, alpha):
        """stored outputs at the positions for stored beta, gamma, alpha"""
        f = self.f
        r = f.q
        b, g, a = (v * f.Rinv % r for v in (beta, gamma, alpha))
        opb = (1 + b) % r
        gopb = opb * g % r
        out = []
        for (z, h1, h2, t, lf), (zq, h1q, h2q, tq), (x, xg, xi, d0, dn, xinv) in zip(zip(*self.p), zip(*self.q), self.ctx):
            m = opb * z % r * ((g + lf) % r) % r * ((b * tq + t + gopb) % r) % r
            nn = (b * h1q + h1 + gopb) * (b * h2q + h2 + gopb) % r * zq % r
            lh = (m - nn) * xg % r
            lh0 = (z - 1) * xi % r * d0 % r
            lhn = (z - 1) * xi % r * dn % r
            lh12 = (h1 - h2q) * xi % r * dn % r
            out.append((((lh12 * a + lhn) * a + lh0) * a + lh) % r * xinv % r * f.R % r)
        return out


def cycled_extremes(c, n, k):
    """k vectors of n stored values cycling the extremes with different strides and offsets"""
    E = extremes(c)
    m = len(E)
    return [[E[(p * (2 * v + 1) + 7 * v) % m] for p in range(n)] for v in range(k)]


def check_perm_numerator(c, n, numerator, label, rng, sweep=False):
    """numerator(LT1, LT2, LZ, E, O) returns gmsm_fft_permutation_numerator_device's output.  Random inputs at >= 4096 positions
    (all of them for n <= 4096); with sweep, inputs cycling the extremes and eps, then omega, through every extreme"""
    f = fr(c)
    r, w = f.q, f.limbs
    pos = numerator_positions(n, rng)
    if sweep:
        vecs = [pack(v, w) for v in cycled_extremes(c, n, 3)]
        chal = [(e, rng.randrange(r)) for e in extremes(c)] + [(rng.randrange(r), e) for e in extremes(c)]
    else:
        vecs = [random_canonical(c, n, rng.randrange(1 << 30)) for _ in range(3)]
        chal = [(rng.randrange(r), rng.randrange(r))]
    ref = PermNumRef(c, n, *vecs, pos)
    for eps, omega in chal:
        got = numerator(*vecs, pack([eps], w), pack([omega], w))[pos]
        logn = n.bit_length() - 1
        R.compare("%s %s gmsm_fft_permutation_numerator_device n=%d %s eps=%d omega=%d" % (
            label, c, n, "extreme inputs" if sweep else "random inputs", eps, omega), got, ref(eps, omega), r,
            lambda t: (ref.lt1[t], ref.lt2[t], ref.lz[t], ref.lzn[t]), index=lambda t: "p=%d i=%d" % (pos[t], bitrev(pos[t], logn)),
            kind="plain lt1[p], lt2[p], lz[p], lz[rev(i + 1)]")


def check_plookup_numerator(c, n, numerator, label, rng, sweep=False):
    """numerator(LZ, LH1, LH2, LT, LF, B, G, A) returns gmsm_fft_plookup_numerator_device's output; as check_perm_numerator with
    beta, gamma and alpha each swept through the extremes"""
    f = fr(c)
    r, w = f.q, f.limbs
    pos = numerator_positions(n, rng)
    if sweep:
        vecs = [pack(v, w) for v in cycled_extremes(c, n, 5)]
        base = [rng.randrange(r) for _ in range(3)]
        chal = [tuple(e if j == s else base[j] for j in range(3)) for s in range(3) for e in extremes(c)]
    else:
        vecs = [random_canonical(c, n, rng.randrange(1 << 30)) for _ in range(5)]
        chal = [tuple(rng.randrange(r) for _ in range(3))]
    ref = PlookupNumRef(c, n, *vecs, pos)
    logn = n.bit_length() - 1
    for beta, gamma, alpha in chal:
        got = numerator(*vecs, *(pack([v], w) for v in (beta, gamma, alpha)))[pos]
        R.compare("%s %s gmsm_fft_plookup_numerator_device n=%d %s beta=%d gamma=%d alpha=%d" % (
            label, c, n, "extreme inputs" if sweep else "random inputs", beta, gamma, alpha), got, ref(beta, gamma, alpha), r,
            lambda t: ref.p[0][t : t + 1] + ref.q[0][t : t + 1], index=lambda t: "p=%d i=%d" % (pos[t], bitrev(pos[t], logn)),
            kind="plain lz[p], lz[q]")


# ------------------------------------------------------------------------------------------
# E. the sort on adversarial keys
# ------------------------------------------------------------------------------------------


def top_full_byte(c):
    """the highest byte position at which all 256 digits give a value below r (the bytes above it zero)"""
    return (fr(c).bits - 1) // 8 - 1


def sort_pools(c, rng):
    """named pools of distinct canonical values, ascending: index = rank"""
    f = fr(c)
    r = f.q
    tb = top_full_byte(c)
    base = rng.randrange(1 << (8 * tb)) & ~0xFF & ~(0xFF << (8 * (tb // 2)))
    mid = tb // 2
    return {
        "two keys, differing in byte %d" % mid: [base, base + (1 << (8 * mid))],
        "byte %d varies (the top full byte: one pass)" % tb: [base + (d << (8 * tb)) for d in range(256)],
        "bytes 0 and %d vary (two passes)" % tb: [base + (d2 << (8 * tb)) + d1 for d2 in range(256) for d1 in range(256)],
        "byte 0 varies (one pass)": [base + d for d in range(256)],
        "0, 1, r - 1": [0, 1, r - 1],
        "random": sorted({rng.randrange(r) for _ in range(1 << 16)}),
    }


def sort_distributions(c, n, rng, g):
    """(name, pool name, idx) of adversarial key vectors of length n"""
    P = sort_pools(c, rng)
    names = list(P)
    two, one_top, two_b, low, sp, rnd = names
    out = []
    last_diff_tile = ((n - 1) >> 12) << 12
    for k in sorted({n - 1, last_diff_tile, max(n - 2, 0)}):
        idx = np.ones(n, dtype=np.int64)
        idx[k] = 0
        out.append(("all keys equal but the smaller one at %d" % k, two, idx))
    out += [("random digits", one_top, g.integers(0, 256, n)), ("random digits", two_b, g.integers(0, 1 << 16, n)),
            ("random", sp, g.integers(0, 3, n)), ("random", rnd, g.integers(0, len(P[rnd]), n))]
    s = np.sort(g.integers(0, len(P[rnd]), n))
    out += [("already sorted", rnd, s), ("reversed", rnd, s[::-1].copy())]
    j = np.arange(n)
    wp, lane = j // 32, j % 32
    pat = lambda wv: np.select([wv % 3 == 0, wv % 3 == 1], [(lane * 8 + wv) % 256, wv % 256], (wv + 128 * (lane & 1)) % 256)  # noqa
    out.append(("warps of 32 distinct / one / two alternating digits", low, pat(wp)))
    out.append(("warps of 32 distinct / one / two alternating digits in both passes", two_b, pat(wp + 1) * 256 + pat(wp)))
    idx = np.full(n, 7 * 256 + 7, dtype=np.int64)
    few = g.choice(n, size=min(32, n), replace=False)
    idx[few] = g.integers(0, 1 << 16, len(few))
    out.append(("one digit holds all keys but 32 in every pass", two_b, idx))
    return P, out


def check_sort(c, n, sort, label, seed, in_place_too=True, brief=False):
    """sort(A, in_place) returns gmsm_fr_sort_device's output for the (n, w) limbs A.  Keys index a pool of distinct canonical
    values converted once to Montgomery form; the expected output is pool_stored[sort(idx)].  The one- and two-byte keys (an odd
    and an even number of passes) also run in place; brief: only the single differing keys, the two-byte keys and the dominating
    digit"""
    f = fr(c)
    w = f.limbs
    rng, g = random.Random(seed), np.random.default_rng(seed)
    P, dists = sort_distributions(c, n, rng, g)
    one_top, two_b = list(P)[1:3]
    if brief:
        dists = [d for d in dists if d[0].startswith(("all keys equal", "one digit")) or (d[1] == two_b and d[0] == "random digits")]
    stored = {name: pack([f.to_mont(v) for v in vals], w) for name, vals in P.items() if any(d[1] == name for d in dists)}
    for name, pool, idx in dists:
        ps = stored[pool]
        A = ps[idx]
        exp = ps[np.sort(idx)]
        for in_place in (False, True) if in_place_too and pool in (one_top, two_b) else (False,):
            got = sort(A.copy(), in_place)
            what = "%s %s gmsm_fr_sort_device n=%d %s, keys from pool '%s' (%s)" % (
                label, c, n, name, pool, "in place" if in_place else "out of place")
            compare_packed(what, got, exp, f.q, lambda i: (), kind="output index; the pool and the distribution named above")
