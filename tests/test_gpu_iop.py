"""iop.py on the device for the seven pairing curves, limb for limb against the line-by-line restatement of tests/iop_ref.py and the
reference's own relational tests: every form change (with growth from a shorter buffer, host and device inputs), Polynomial.Evaluate
in all six forms and four shifts, Evaluate of traced expressions, BuildRatioShuffledVectors, BuildRatioCopyConstraint (k = 1 ... 5,
mixed layouts, ignored shifts, identity sigma, a zero denominator at a tile boundary, n = 1 and 2, sigma refused), DivideByXMinusOne,
and the copy constraint at production size."""
import random
from importlib import import_module

import numpy as np
import pytest

from tests import iop_ref as R
from tests.permutation_ref import domain as ref_domain

curves = import_module("gnark-crypto_b200.curves")

pytestmark = pytest.mark.gpu
CURVES = ["bn254", "bls12381", "bls12377", "bls24315", "bls24317", "bw6633", "bw6761"]
FORMS = [(b, l) for b in (1, 2, 4) for l in (8, 16)]


def _iop():
    return import_module("gnark-crypto_b200.iop")


def _fft():
    return import_module("gnark-crypto_b200.fft")


def _torch():
    return import_module("torch")


def _r(c):
    return curves.CURVE_PARAMS[c].r


def _enc(vals, c):
    return curves._fr_encode(vals, _r(c))


def _dec(a, c):
    a = a.cpu().numpy().view(np.uint64) if hasattr(a, "is_cuda") else a
    return curves._fr_decode(np.asarray(a, dtype=np.uint64), _r(c))


def _dev(a):
    return _torch().from_numpy(np.ascontiguousarray(a, dtype=np.uint64).view(np.int64).reshape(-1).copy()).cuda()


def _mk(c, vals, form, device=False, shift=0, size=None):
    iop = _iop()
    a = _enc(vals, c)
    p = iop.NewPolynomial(_dev(a) if device else a, iop.Form(*form), c)
    p.Shift(shift)
    if size is not None:
        p.SetSize(size)
    return p


def _same(p, q, c, what):
    assert (p.Basis, p.Layout) == (q["basis"], q["layout"]), what
    got = _dec(p.Coefficients(), c)
    assert got == q["c"], "%s %s: first mismatch at %d" % (c, what, next(i for i, (a, b) in enumerate(zip(got, q["c"])) if a != b))


@pytest.mark.parametrize("c", CURVES)
def test_form_changes(c):
    """every form change at 2^10 from every form (ToLagrange, ToCanonical, ToLagrangeCoset, ToRegular, ToBitReverse), including
    growth from 2^9 coefficients; host and device inputs give identical limbs; a shallow clone sees the change"""
    r = _r(c)
    rng = random.Random(5)
    n = 1 << 10
    d = _fft().Domain(c, n)
    rd = ref_domain(c, n)
    ops = [("ToLagrange", R.to_lagrange), ("ToCanonical", R.to_canonical), ("ToLagrangeCoset", R.to_lagrange_coset)]
    for form in FORMS:
        for name, fn in ops:
            m = n // 2 if name == "ToLagrangeCoset" and form == (1, 8) else n
            vals = [rng.randrange(r) for _ in range(m)]
            outs = []
            for device in (False, True):
                p = _mk(c, vals, form, device)
                sc = p.ShallowClone()
                getattr(p, name)(d)
                q = fn(R.poly(vals, *form), rd)
                _same(p, q, c, "%s from %s" % (name, form))
                assert (sc.Basis, sc.Layout) == (p.Basis, p.Layout) and _dec(sc.Coefficients(), c) == q["c"]
                outs.append(_dec(p.Coefficients(), c))
            assert outs[0] == outs[1]
    vals = [rng.randrange(r) for _ in range(n)]
    p = _mk(c, vals, (2, 8))
    p.ToBitReverse()
    _same(p, R.to_bit_reverse(R.poly(vals, 2, 8)), c, "ToBitReverse")
    p.ToRegular()
    _same(p, R.poly(vals, 2, 8), c, "ToRegular")


@pytest.mark.parametrize("c", CURVES)
def test_polynomial_evaluate(c):
    """Polynomial.Evaluate in the six forms with shift 0, 1, 5 and 6 (6: evaluated at 0, the reference's unset element), at a random
    x and at x on the domain (0 in Lagrange form), and with a zero coset"""
    r = _r(c)
    rng = random.Random(11)
    n = 1 << 8
    rd = ref_domain(c, n)
    for form in FORMS:
        vals = [rng.randrange(r) for _ in range(n)]
        for shift in (0, 1, 5, 6):
            for x in (rng.randrange(r), pow(rd.generator, 7, r), 1):
                for device in (False, True):
                    p = _mk(c, vals, form, device, shift)
                    q = R.poly(vals, *form, shift)
                    if form[0] == 4:
                        p.coset = q["coset"] = rd.shift if shift != 5 else 0
                    got = _dec(p.Evaluate(_enc([x], c)[0]), c)[0]
                    assert got == R.evaluate(q, x, c, r), (c, form, shift, x, device)
    p = _mk(c, vals, (2, 8))
    assert _dec(p.Evaluate(_enc([pow(rd.generator, 3, r)], c)[0]), c)[0] == 0


@pytest.mark.parametrize("c", CURVES)
def test_evaluate_expression(c):
    """Evaluate of a PLONK-like gate with constants, a power and the index, over inputs of mixed layouts and shifts, into a
    BitReverse and a Regular result, host and device"""
    iop = _iop()
    r = _r(c)
    rng = random.Random(17)
    n = 1 << 9
    vals = [[rng.randrange(r) for _ in range(n)] for _ in range(3)]
    lay = [(2, 8, 0), (2, 16, 1), (2, 8, 3)]

    def f(i, a, b, z):
        return a * b + 3 * a - b ** 5 + z * i - 7

    def fi(i, a, b, z):
        return (a * b + 3 * a - pow(b, 5, r) + z * i - 7) % r

    for out_layout in (8, 16):
        for device in (False, True):
            xs = [_mk(c, v, (b, l), device, s) for v, (b, l, s) in zip(vals, lay)]
            res = iop.Evaluate(f, None, iop.Form(2, out_layout), *xs)
            want = R.evaluate_expr(fi, (2, out_layout), [R.poly(v, b, l, s) for v, (b, l, s) in zip(vals, lay)], r)
            _same(res, want, c, "Evaluate layout %d" % out_layout)
            assert res.size == n and res.shift == 0
    with pytest.raises(iop.ErrInconsistentSize):
        iop.Evaluate(f, _enc([0] * 4, c), iop.Form(2, 8), *[_mk(c, v, (2, 8)) for v in vals])


@pytest.mark.parametrize("c", CURVES)
def test_ratio_shuffled(c):
    """TestBuildRatioShuffledVectors restated: the full product is 1 for shuffled vectors; bit-reversed inputs give the same ratio;
    every expected form agrees with the restatement bit for bit; inputs in mixed forms are put in Lagrange form in place"""
    iop = _iop()
    r = _r(c)
    rng = random.Random(23)
    n = 1 << 8
    beta = rng.randrange(r)
    num = [[rng.randrange(r) for _ in range(n)] for _ in range(4)]
    flat = [v for col in num for v in col]
    rng.shuffle(flat)
    den = [flat[j * n:(j + 1) * n] for j in range(4)]
    for device in (False, True):
        for form in FORMS:
            P = [_mk(c, v, (2, 8), device) for v in num]
            Q = [_mk(c, v, (2, 8), device) for v in den]
            z = iop.BuildRatioShuffledVectors(P, Q, _enc([beta], c)[0], iop.Form(*form))
            want = R.ratio_shuffled([R.poly(v, 2, 8) for v in num], [R.poly(v, 2, 8) for v in den], beta, form, c, r)
            _same(z, want, c, "shuffled form %s" % (form,))
        P = [_mk(c, R.bit_reverse(v), (2, 16), device) for v in num]
        Q = [_mk(c, R.bit_reverse(v), (2, 16), device) for v in den]
        z = iop.BuildRatioShuffledVectors(P, Q, _enc([beta], c)[0], iop.Form(2, 8))
        zl = _dec(z.Coefficients(), c)
        # Z[n-1] times the last ratio is the full product: 1
        last = 1
        for j in range(4):
            last = last * (beta - num[j][n - 1]) * pow(beta - den[j][n - 1], r - 2, r) % r
        assert zl[n - 1] * last % r == 1
    # mixed forms, shorter inputs grown
    vals = [[rng.randrange(r) for _ in range(n if j < 4 else n // 2)] for j in range(6)]   # checkSize reads P[0..1], Q[0..1]
    forms = [(1, 8), (4, 16), (1, 16), (2, 16), (4, 8), (2, 8)]
    d = _fft().Domain(c, n)
    rdom = ref_domain(c, n)
    P, Q, RP, RQ = [], [], [], []
    for j in range(3):
        for L, RL, v, f in ((P, RP, vals[2 * j], forms[2 * j]), (Q, RQ, vals[2 * j + 1], forms[2 * j + 1])):
            p = _mk(c, v, f)
            q = R.poly(v, *f)
            if f[0] == 4:   # a LagrangeCoset input: made by ToLagrangeCoset on the same domain
                p = _mk(c, v, (1, 8))
                p.ToLagrangeCoset(d)
                q = R.to_lagrange_coset(R.poly(v, 1, 8), rdom)
            L.append(p)
            RL.append(q)
    z = iop.BuildRatioShuffledVectors(P, Q, _enc([beta], c)[0], iop.Form(1, 8), d)
    _same(z, R.ratio_shuffled(RP, RQ, beta, (1, 8), c, r), c, "shuffled mixed forms")
    for p, q in zip(P + Q, RP + RQ):
        _same(p, q, c, "input put in Lagrange form")


def _cycles_sigma(k, n, rng):
    """a random permutation of [0, k n) and column values constant on its cycles"""
    perm = list(range(k * n))
    rng.shuffle(perm)
    sigma = [0] * (k * n)
    # one cycle through positions in the order perm[0], perm[1], ... split into cycles of random length
    pos = 0
    cyc = []
    while pos < k * n:
        ln = min(rng.randrange(1, 6), k * n - pos)
        cycle = perm[pos:pos + ln]
        for a, b in zip(cycle, cycle[1:] + cycle[:1]):
            sigma[a] = b
        cyc.append(cycle)
        pos += ln
    return sigma, cyc


@pytest.mark.parametrize("c", CURVES)
def test_ratio_copy(c):
    """TestBuildRatioCopyConstraint restated: Z(w^(n-1)) times the last ratio is 1 for values constant on sigma's cycles, k = 1 ... 5,
    bit-exact against the restatement in every expected form, with mixed layouts and shifts that are ignored; the identity sigma
    gives Z = 1; n = 1 and n = 2; sigma out of range is refused and the output left untouched"""
    iop = _iop()
    r = _r(c)
    rng = random.Random(29)
    n = 1 << 8
    for k in range(1, 6):
        sigma, cyc = _cycles_sigma(k, n, rng)
        flat = [0] * (k * n)
        for cycle in cyc:
            v = rng.randrange(r)
            for s in cycle:
                flat[s] = v
        cols = [flat[j * n:(j + 1) * n] for j in range(k)]
        beta, gamma = rng.randrange(r), rng.randrange(r)
        layouts = [8 if j % 2 == 0 else 16 for j in range(k)]
        for form in (FORMS if k == 3 else [(2, 8)]):
            for device in (False, True):
                E = [_mk(c, col if lay == 8 else R.bit_reverse(col), (2, lay), device, shift=j + 1) for j, (col, lay) in
                     enumerate(zip(cols, layouts))]
                sg = np.array(sigma, dtype=np.int64)
                z = iop.BuildRatioCopyConstraint(E, _dev(sg.view(np.uint64)) if device else sg, _enc([beta], c)[0], _enc([gamma], c)[0],
                                                 iop.Form(*form))
                want = R.ratio_copy([R.poly(col if lay == 8 else R.bit_reverse(col), 2, lay) for col, lay in zip(cols, layouts)], sigma,
                                    beta, gamma, form, c, r)
                _same(z, want, c, "copy k=%d form %s" % (k, form))
        z = iop.BuildRatioCopyConstraint([_mk(c, col, (2, 8)) for col in cols], np.array(sigma), _enc([beta], c)[0],
                                         _enc([gamma], c)[0], iop.Form(2, 8))
        d = ref_domain(c, n)
        bs, ds = R.factors_copy([R.poly(col, 2, 8) for col in cols], sigma, beta, gamma, d, r)
        zl = _dec(z.Coefficients(), c)
        tail = 1
        for j in range(k):
            tail = tail * (cols[j][n - 1] + beta * pow(d.shift, j, r) * pow(d.generator, n - 1, r) + gamma) % r
            s = sigma[j * n + n - 1]
            tail = tail * pow((cols[j][n - 1] + beta * pow(d.shift, s // n, r) * pow(d.generator, s % n, r) + gamma) % r, r - 2, r) % r
        assert zl[n - 1] * tail % r == 1, "full product k=%d" % k
    # identity sigma: Z = 1
    cols = [[rng.randrange(r) for _ in range(n)] for _ in range(3)]
    z = iop.BuildRatioCopyConstraint([_mk(c, col, (2, 8)) for col in cols], np.arange(3 * n), _enc([5], c)[0], _enc([7], c)[0],
                                     iop.Form(2, 8))
    assert _dec(z.Coefficients(), c) == [1] * n
    # n = 1, 2
    for m in (1, 2):
        cols = [[rng.randrange(r) for _ in range(m)] for _ in range(2)]
        sigma = list(range(2 * m))
        rng.shuffle(sigma)
        z = iop.BuildRatioCopyConstraint([_mk(c, col, (2, 8)) for col in cols], np.array(sigma), _enc([3], c)[0], _enc([4], c)[0],
                                         iop.Form(2, 8))
        want = R.ratio_copy([R.poly(col, 2, 8) for col in cols], sigma, 3, 4, (2, 8), c, r)
        _same(z, want, c, "copy n=%d" % m)
    # a zero denominator at a tile boundary (position 511 of 1024: the last leaf of tile 0) zeroes every later Z[k]
    m = 1 << 10
    cols = [[rng.randrange(r) for _ in range(m)] for _ in range(2)]
    sigma = list(range(2 * m))
    sigma[511], sigma[m + 600] = sigma[m + 600], sigma[511]
    d = ref_domain(c, m)
    beta = rng.randrange(1, r)
    s511 = sigma[511]
    idv = beta * pow(d.shift, s511 // m, r) * pow(d.generator, s511 % m, r) % r
    gamma = (-cols[0][511] - idv) % r
    for device in (False, True):
        E = [_mk(c, col, (2, 8), device) for col in cols]
        sg = np.array(sigma, dtype=np.int64)
        z = iop.BuildRatioCopyConstraint(E, _dev(sg.view(np.uint64)) if device else sg, _enc([beta], c)[0], _enc([gamma], c)[0],
                                         iop.Form(2, 8))
        want = R.ratio_copy([R.poly(col, 2, 8) for col in cols], sigma, beta, gamma, (2, 8), c, r)
        _same(z, want, c, "copy zero denominator")
        assert all(v == 0 for v in want["c"][512:])
    # sigma out of range: refused (device sigma: by the device check), the output untouched
    E = [_mk(c, col, (2, 8), True) for col in cols]
    for bad in (-1, 2 * m):
        sg = np.array(sigma, dtype=np.int64)
        sg[777] = bad
        with pytest.raises(import_module("gnark-crypto_b200.multiexp").MultiExpError, match="outside"):
            iop.BuildRatioCopyConstraint(E, _dev(sg.view(np.uint64)), _enc([1], c)[0], _enc([2], c)[0], iop.Form(2, 8))
        with pytest.raises(iop.IopError, match="outside"):
            iop.BuildRatioCopyConstraint([_mk(c, col, (2, 8)) for col in cols], sg, _enc([1], c)[0], _enc([2], c)[0], iop.Form(2, 8))


@pytest.mark.parametrize("c", CURVES)
def test_divide_by_x_minus_one(c):
    """TestDivideByXMinusOne restated: h = a b - c on the coset of the big domain (4 n), divided by X^n - 1, gives q with
    q(x) (x^n - 1) = h(a(x), b(x), c(x)) at a random x; bit-exact against the restatement, with a shifted input too"""
    iop = _iop()
    r = _r(c)
    rng = random.Random(31)
    n = 1 << 6
    small, big = _fft().Domain(c, n), _fft().Domain(c, 4 * n)
    va = [rng.randrange(r) for _ in range(n)]
    vb = [rng.randrange(r) for _ in range(n)]
    rs = ref_domain(c, n)        # c = a b on the small domain, so that a b - c is divisible by X^n - 1 (as in the reference's test)
    al, bl = (R.to_lagrange(R.poly(v, 1, 8), rs)["c"] for v in (va, vb))
    vc = R.to_canonical(R.poly([u * v % r for u, v in zip(al, bl)], 2, 16), rs)["c"]
    x = rng.randrange(r)
    for device in (False, True):
        A, B, C = (_mk(c, v, (1, 8), device) for v in (va, vb, vc))
        for p in (A, B, C):
            p.ToLagrangeCoset(big)
        h = iop.Evaluate(lambda i, a, b, cc: a * b - cc, None, iop.Form(4, 16), A, B, C)
        q = iop.DivideByXMinusOne(h, [small, big])
        assert (q.Basis, q.Layout, q.size) == (1, 8, n)
        qv = _dec(q.Coefficients(), c)
        ev = lambda cf: sum(v * pow(x, i, r) for i, v in enumerate(cf)) % r
        assert ev(qv) * (pow(x, n, r) - 1) % r == (ev(va) * ev(vb) - ev(vc)) % r
        ha = R.evaluate_expr(lambda i, a, b, cc: (a * b - cc) % r, (4, 16),
                             [R.to_lagrange_coset(R.poly(v, 1, 8), ref_domain(c, 4 * n)) for v in (va, vb, vc)], r)
        ha["size"] = n
        assert qv == R.divide_by_x_minus_one(ha, n, 4 * n, c, r)["c"]
        h.Shift(1)
        q = iop.DivideByXMinusOne(h, [small, big])
        ha["shift"] = 1
        assert _dec(q.Coefficients(), c) == R.divide_by_x_minus_one(ha, n, 4 * n, c, r)["c"]
    with pytest.raises(iop.ErrMustBeLagrangeCoset):
        iop.DivideByXMinusOne(_mk(c, va, (2, 8)), [small, big])


@pytest.mark.parametrize("c,logn", [("bn254", 22), ("bw6761", 20)])
def test_ratio_copy_production(c, logn):
    """k = 3 at production size with a random sigma whose cycles hold equal values: Z[n-1] times the last ratio is 1, and
    Z[k+1] d_k = Z[k] b_k at 4096 sampled k and every tile and scan-level boundary, b_k and d_k from the restatement"""
    iop = _iop()
    torch = _torch()
    r = _r(c)
    n = 1 << logn
    k = 3
    g = torch.Generator().manual_seed(7)
    perm = torch.randperm(k * n, generator=g).numpy()
    sigma = np.empty(k * n, dtype=np.int64)
    sigma[perm] = np.roll(perm, -1)           # one long cycle through perm: every value equal ...
    cuts = np.sort(np.random.default_rng(1).choice(k * n, size=k * n // 8, replace=False))
    starts = np.concatenate([[0], cuts])      # ... split into many cycles of random length
    ends = np.concatenate([cuts, [k * n]])
    for s0, e0 in zip(starts, ends):
        if e0 > s0:
            sigma[perm[e0 - 1]] = perm[s0]
    cyc_id = np.empty(k * n, dtype=np.int64)
    seg = np.repeat(np.arange(len(starts)), ends - starts)
    cyc_id[perm] = seg
    rng = random.Random(3)
    vals = curves._fr_encode([rng.randrange(r) for _ in range(len(starts))], r)
    cols = vals[cyc_id].reshape(k, n, -1)
    beta, gamma = rng.randrange(r), rng.randrange(r)
    E = [iop.NewPolynomial(_dev(cols[j]), iop.Form(2, 8), c) for j in range(k)]
    z = iop.BuildRatioCopyConstraint(E, torch.from_numpy(sigma).cuda(), _enc([beta], c)[0], _enc([gamma], c)[0], iop.Form(2, 8))
    zt = z.Coefficients().view(n, -1).cpu().numpy().view(np.uint64)
    d = ref_domain(c, n)

    def col(j, i):
        return curves._fr_decode(cols[j, i], r)[0]

    def bd(i):
        b = dd = 1
        for j in range(k):
            v = col(j, i)
            b = b * (v + beta * pow(d.shift, j, r) * pow(d.generator, i, r) + gamma) % r
            s = int(sigma[j * n + i])
            dd = dd * (v + beta * pow(d.shift, s // n, r) * pow(d.generator, s % n, r) + gamma) % r
        return b, dd

    zz = lambda i: curves._fr_decode(zt[i], r)[0]
    b, dd = bd(n - 1)
    assert zz(n - 1) * b * pow(dd, r - 2, r) % r == 1
    assert zz(0) == 1
    srng = random.Random(9)
    ks = {srng.randrange(n - 1) for _ in range(4096)}
    for t in range(512, n, 512):          # every inversion tile (512) and scan tile (512 or 1024) and every scan-level boundary
        for off in (-1, 0):
            if t + off < n - 1:
                ks.add(t + off)
    for kk in sorted(ks):
        b, dd = bd(kk)
        assert zz(kk + 1) * dd % r == zz(kk) * b % r, "k = %d" % kk
