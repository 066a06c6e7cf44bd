"""Test reference for iop.py on Python ints (regular, not Montgomery), restating ecc/bn254/fr/iop (polynomial.go, expressions.go,
ratios.go, quotient.go) line by line; the iop packages of the other six pairing curves are the same generated code.  A polynomial
is a dict {"c": [ints], "basis", "layout", "shift", "size", "coset"}; FFTs are the oracle's (tests/permutation_ref.domain).  Quirks
kept: Evaluate in Lagrange basis is 0 on the domain, shift > 5 (or < 0) evaluates at 0, a zero coset makes x = 0, every Z[k] past
the first zero denominator is 0, and checkSize compares pols[i][j] for i, j < len(pols) only."""
from tests.permutation_ref import batch_invert, domain, rev

CANONICAL, LAGRANGE, LAGRANGE_COSET = 1, 2, 4
REGULAR, BIT_REVERSE = 8, 16
DIT, DIF = 0, 1


def poly(c, basis, layout, shift=0, size=None, coset=0):
    return {"c": list(c), "basis": basis, "layout": layout, "shift": shift, "size": len(c) if size is None else size, "coset": coset}


def bit_reverse(a):
    n = len(a)
    return [a[rev(i, n)] for i in range(n)]


def _grow(p, n):
    if len(p["c"]) < n:
        p["c"] = p["c"] + [0] * (n - len(p["c"]))


def _fft(d, a, dec, coset=False):
    return d.fft(a, dec, coset)


def _ifft(d, a, dec, coset=False):
    return d.fft_inverse(a, dec, coset)


def to_lagrange(p, d):
    """ToLagrange (polynomial.go:287-318)"""
    f = (p["basis"], p["layout"])
    _grow(p, d.cardinality)
    if f == (CANONICAL, REGULAR):
        p["layout"], p["c"] = BIT_REVERSE, _fft(d, p["c"], DIF)
    elif f == (CANONICAL, BIT_REVERSE):
        p["layout"], p["c"] = REGULAR, _fft(d, p["c"], DIT)
    elif f[0] == LAGRANGE:
        return p
    elif f == (LAGRANGE_COSET, REGULAR):
        p["layout"], p["c"] = REGULAR, _fft(d, _ifft(d, p["c"], DIF, True), DIT)
    else:
        p["layout"], p["c"] = BIT_REVERSE, _fft(d, _ifft(d, p["c"], DIT, True), DIF)
    p["basis"] = LAGRANGE
    return p


def to_canonical(p, d):
    """ToCanonical (polynomial.go:322-349)"""
    f = (p["basis"], p["layout"])
    _grow(p, d.cardinality)
    if f[0] == CANONICAL:
        return p
    layout, dec = {REGULAR: (BIT_REVERSE, DIF), BIT_REVERSE: (REGULAR, DIT)}[f[1]]
    p["layout"], p["c"] = layout, _ifft(d, p["c"], dec, f[0] == LAGRANGE_COSET)
    p["basis"] = CANONICAL
    return p


def to_lagrange_coset(p, d):
    """ToLagrangeCoset (polynomial.go:359-390)"""
    p["coset"] = d.shift
    f = (p["basis"], p["layout"])
    _grow(p, d.cardinality)
    if f == (CANONICAL, REGULAR):
        p["layout"], p["c"] = BIT_REVERSE, _fft(d, p["c"], DIF, True)
    elif f == (CANONICAL, BIT_REVERSE):
        p["layout"], p["c"] = REGULAR, _fft(d, p["c"], DIT, True)
    elif f == (LAGRANGE, REGULAR):
        p["layout"], p["c"] = REGULAR, _fft(d, _ifft(d, p["c"], DIF), DIT, True)
    elif f == (LAGRANGE, BIT_REVERSE):
        p["layout"], p["c"] = BIT_REVERSE, _fft(d, _ifft(d, p["c"], DIT), DIF, True)
    else:
        return p
    p["basis"] = LAGRANGE_COSET
    return p


def to_regular(p):
    if p["layout"] != REGULAR:
        p["c"], p["layout"] = bit_reverse(p["c"]), REGULAR
    return p


def to_bit_reverse(p):
    if p["layout"] != BIT_REVERSE:
        p["c"], p["layout"] = bit_reverse(p["c"]), BIT_REVERSE
    return p


def _evaluate_inner(p, x, c, r):
    """polynomial.evaluate (polynomial.go:200-261)"""
    n = len(p["c"])
    res = 0
    if p["basis"] == CANONICAL:
        for i in range(n - 1, -1, -1):
            res = (res * x + p["c"][i if p["layout"] == REGULAR else rev(i, n)]) % r
        return res
    w = domain(c, n).generator
    accw, dens = 1, []
    for i in range(n):
        dens.append((x - accw) % r)
        accw = accw * w % r
    invdens = batch_invert(dens, r)
    li = (pow(x, n, r) - 1) * pow(n, r - 2, r) % r
    for i in range(n):
        li = li * invdens[i] % r
        res = (res + li * p["c"][i if p["layout"] == REGULAR else rev(i, n)]) % r
        li = li * dens[i] * w % r
    return res


def evaluate(p, x, c, r):
    """Polynomial.Evaluate (polynomial.go:106-132)"""
    if p["basis"] == LAGRANGE_COSET:
        x = x * (pow(p["coset"], r - 2, r) if p["coset"] else 0) % r
    s = p["shift"]
    if s == 0:
        return _evaluate_inner(p, x, c, r)
    if s <= 5:
        g = pow(domain(c, p["size"]).generator, s, r) if s > 0 else 0     # smallExp: fr.Element{} for a negative n
        return _evaluate_inner(p, x * g % r, c, r)
    return _evaluate_inner(p, 0, c, r)                                      # g.Exp(g, shift) of the zero g


def get_coeff(p, i):
    """GetCoeff (polynomial.go:151-163)"""
    n = len(p["c"])
    s = (i + (n // p["size"]) * p["shift"]) % n
    if p["layout"] == REGULAR:
        return p["c"][s]
    tz = (n & -n).bit_length() - 1
    return p["c"][int(bin(s)[2:].zfill(64)[::-1], 2) >> (64 - tz) if tz else 0]


def evaluate_expr(f, form, xs, r):
    """Evaluate (expressions.go:26-73) with f on Python ints"""
    n = len(xs[0]["c"])
    out = [0] * n
    for i in range(n):
        v = f(i, *[get_coeff(p, i) for p in xs]) % r
        out[i if form[1] == REGULAR else rev(i, n)] = v
    res = poly(out, form[0], form[1], 0, xs[0]["size"])
    return res


def check_size(*pols):
    """checkSize (ratios.go:277-291): True when accepted, False for ErrInconsistentSize, None where the reference panics"""
    m = len(pols)
    if any(j >= len(pols[i]) for i in range(m) for j in range(m)):
        return None
    n = len(pols[0][0]["c"])
    return all(len(pols[i][j]["c"]) == n for i in range(m) for j in range(m))


def put_in_expected_form(p, d, form):
    """putInExpectedFormFromLagrangeRegular (ratios.go:248-273)"""
    p["basis"], p["layout"] = form
    if form[0] == CANONICAL:
        p["c"] = _ifft(d, p["c"], DIF)
        if form[1] == REGULAR:
            p["c"] = bit_reverse(p["c"])
        return p
    if form[0] == LAGRANGE_COSET:
        p["c"] = _fft(d, _ifft(d, p["c"], DIF), DIT, True)
        if form[1] == BIT_REVERSE:
            p["c"] = bit_reverse(p["c"])
        return p
    if form[1] == BIT_REVERSE:
        p["c"] = bit_reverse(p["c"])
    return p


def _col(p, i, n):
    return p["c"][rev(i, n) if p["layout"] == BIT_REVERSE else i]


def ratio_shuffled(num, den, beta, form, c, r):
    """BuildRatioShuffledVectors (ratios.go:45-127) after the checks; mutates num and den to Lagrange form"""
    n = len(num[0]["c"])
    d = domain(c, n)
    for p, q in zip(num, den):
        to_lagrange(p, d)
        to_lagrange(q, d)
    coeffs, t = [1] + [0] * (n - 1), [1] + [0] * (n - 1)
    for i in range(n - 1):
        b = dd = 1
        for p, q in zip(num, den):
            b = b * (beta - _col(p, i, n)) % r
            dd = dd * (beta - _col(q, i, n)) % r
        coeffs[i + 1] = coeffs[i] * b % r
        t[i + 1] = t[i] * dd % r
    t = batch_invert(t, r)
    for i in range(1, n):
        coeffs[i] = coeffs[i] * t[i] % r
    return put_in_expected_form(poly(coeffs, *form), d, form)


def support(k, d, r):
    """getSupportIdentityPermutation (ratios.go:320-361)"""
    n = d.cardinality
    res = [pow(d.generator, i, r) for i in range(k * n)] if k else []
    res[:n] = [pow(d.generator, i, r) for i in range(n)]
    for j in range(1, k):
        cs = pow(d.shift, j, r)
        res[j * n:(j + 1) * n] = [v * cs % r for v in res[:n]]
    return res


def factors_copy(entries, sigma, beta, gamma, d, r):
    """the per-position numerator b_i and denominator d_i of BuildRatioCopyConstraint (ratios.go:174-206), entries in Lagrange form"""
    n = d.cardinality
    ids = support(len(entries), d, r)
    bs, ds = [], []
    for i in range(n - 1):
        b = dd = 1
        for j, p in enumerate(entries):
            v = _col(p, i, n)
            b = b * (beta * ids[i + j * n] + gamma + v) % r
            dd = dd * (beta * ids[sigma[i + j * n]] + gamma + v) % r
        bs.append(b)
        ds.append(dd)
    return bs, ds


def ratio_copy(entries, sigma, beta, gamma, form, c, r):
    """BuildRatioCopyConstraint (ratios.go:136-246) after the checks; mutates entries to Lagrange form"""
    n = len(entries[0]["c"])
    d = domain(c, n)
    for p in entries:
        to_lagrange(p, d)
    bs, ds = factors_copy(entries, sigma, beta, gamma, d, r)
    coeffs, t = [1] + bs, [1] + ds
    for i in range(2, n):
        coeffs[i] = coeffs[i] * coeffs[i - 1] % r
        t[i] = t[i] * t[i - 1] % r
    tinv = batch_invert(t[1:], r)
    for i in range(1, n):
        coeffs[i] = coeffs[i] * tinv[i - 1] % r
    return put_in_expected_form(poly(coeffs, *form), d, form)


def xn_minus_one_inverses(n_small, n_big, c, r):
    """evaluateXnMinusOneDomainBigCoset (quotient.go:56-79)"""
    big = domain(c, n_big)
    ratio = n_big // n_small
    res = [0] * ratio
    res[0] = pow(big.shift, n_small, r)
    t = pow(big.generator, n_small, r)
    for i in range(1, ratio):
        res[i] = res[i - 1] * t % r
        res[i - 1] = (res[i - 1] - 1) % r
    res[-1] = (res[-1] - 1) % r
    return batch_invert(res, r)


def divide_by_x_minus_one(a, n_small, n_big, c, r):
    """DivideByXMinusOne (quotient.go:21-53)"""
    inv = xn_minus_one_inverses(n_small, n_big, c, r)
    rho = len(a["c"]) // a["size"]
    n = len(a["c"])
    out = [0] * n
    for i in range(n):
        out[rev(i, n)] = get_coeff(a, i) * inv[i % rho] % r
    res = poly(out, LAGRANGE_COSET, BIT_REVERSE, 0, a["size"])
    return to_canonical(res, domain(c, n_big))
