"""shplonk.BatchOpen (ecc/bn254/shplonk/shplonk.go:43-172; the shplonk packages of the other six pairing curves are the same
generated code): one proof (W, W') for polynomials f_i opened on point sets S_i, T the multiset union of the S_i.

The reference builds W = Commit(sum_i gamma^i Z_{T\\S_i} (f_i - r_i) / Z_T) and W' = Commit(L / (X - z)) with naive products and
divisions.  On a single-device proving key the same digests come from three exact identities (DESIGN.md, "SHPLONK and FFLONK"):
  * W = sum_i gamma^i q_i, q_i the Euclidean quotient of f_i by Z_{S_i}: divide f_i by (X - a) once per point a of S_i
    (gmsm_fr_poly_div_x_minus_a_device, chained); the f(a) of the chain are the Newton coefficients of f_i on S_i, which give the
    claimed values on the host;
  * W' is the quotient of L by (X - z), which ignores L's constant term, so L = sum_i c_i f_i - Z_T(z) W with
    c_i = gamma^i Z_{T\\S_i}(z): one gmsm_fr_poly_lincomb_device and one more division;
  * FFLONK packs (fflonk.py) are never folded: the quotient of an interleave F = sum_i X^i p_i(X^t) by
    prod_s (X^t - s^t) is the interleave of the quotients of the p_i by prod_s (Y - s^t), so the chain runs on the p_i and the
    linear combination interleaves them with stride t.
The Euclidean quotients make these identities hold for any points, repeated ones included.  Only the claimed values (one copy),
W, W' and the challenges' inputs cross PCIe.  Proving keys sharded over several GPUs (device = -1) use `batch_open_host`, the
line-by-line restatement of the reference."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from . import kzg
from .curves import _challenge, _fr_decode, _fr_encode, _limbs, _params
from .kzg import _check_size, g1_raw_bytes
from .multiexp import MultiExpError
from .transcript import Transcript


class ErrInvalidNumberOfPoints(MultiExpError):
    """shplonk.ErrInvalidNumberOfPoints (shplonk.go:21)"""


class ErrInvalidNumberOfDigests(MultiExpError):
    """shplonk.ErrInvalidNumberOfDigests (shplonk.go:23)"""


@dataclass
class OpeningProof:
    """shplonk.OpeningProof{W, WPrime G1Affine; ClaimedValues [][]fr.Element} (shplonk.go:30-41): ClaimedValues[i] is a
    (len(points[i]), fr.Limbs) uint64 array of f_i on S_i"""

    W: np.ndarray
    WPrime: np.ndarray
    ClaimedValues: list


def BatchOpen(polynomials, digests, points, hf, pk: kzg.ProvingKey, *dataTranscript: bytes) -> OpeningProof:
    """shplonk.BatchOpen: polynomials[i] (numpy (n, fr.Limbs) limbs or a torch CUDA int64 tensor on the key's device, left
    unmodified) is opened on points[i] ((m, fr.Limbs) limbs, m >= 0).  `hf` is a hashlib constructor.  The work is ordered on the
    current stream of the key's device."""
    if len(polynomials) != len(points):
        raise ErrInvalidNumberOfPoints("number of digests should be equal to the number of points")
    if len(polynomials) != len(digests):
        raise ErrInvalidNumberOfDigests("number of digests should be equal to the number of polynomials")
    if not polynomials:
        raise ValueError("shplonk.BatchOpen needs at least one polynomial")
    cp = _params(pk.curve)
    r, w = cp.r, cp.fr_words
    pts = [_decode_points(S, r) for S in points]
    if pk.device < 0:
        polys = [_fr_decode(kzg._host_poly(p, w), r) for p in polynomials]
        W, WPrime, claimed, _, _ = batch_open_host(polys, pts, digests, hf, pk.curve, _host_commit(pk), *dataTranscript)
    else:
        W, WPrime, claimed, _ = open_packs([[p] for p in polynomials], pts, [1] * len(pts), pts, digests, hf, pk, dataTranscript)
    return OpeningProof(W=W, WPrime=WPrime, ClaimedValues=[_fr_encode(v, r).reshape(-1, w) for v in claimed])


def _decode_points(S, r: int) -> list:
    return _fr_decode(np.asarray(S, dtype=np.uint64).reshape(-1, _limbs(r)), r)


def _host_commit(pk: kzg.ProvingKey):
    r = _params(pk.curve).r
    return lambda coeffs: kzg.Commit(_fr_encode(coeffs, r), pk)


def _transcript(hf, ext_points, digests, curve: str, data) -> Transcript:
    """deriveChallenge("gamma", ...) (shplonk.go:278-308) up to the challenge: every point (fr.Marshal), every digest (RawBytes),
    the data transcript"""
    nb = _params(curve).fr_bytes
    fs = Transcript(hf, "gamma", "z")
    for S in ext_points:
        for x in S:
            fs.Bind("gamma", x.to_bytes(nb, "big"))
    for d in digests:
        fs.Bind("gamma", g1_raw_bytes(d, curve))
    for b in data:
        fs.Bind("gamma", b)
    return fs


def _sizes(lens_folded, ext_points):
    """(maxSizePolys, |T|) of shplonk.go:66-82"""
    max_size = max([*lens_folded, *(len(S) + 1 for S in ext_points)])
    return max_size, sum(len(S) for S in ext_points)


# ---- the device algorithm, over packs: plain SHPLONK is packs of one polynomial with t = 1 ----

def open_packs(packs, base_points, ts, ext_points, digests, hf, pk: kzg.ProvingKey, data):
    """shplonk.BatchOpen of the interleaves F_j = sum_i X^i packs[j][i](X^t_j) on ext_points[j] (base_points[j] extended by the
    t_j-th roots of unity, fflonk.extendSet) -> (W, W', claimed values of the F_j on ext_points[j], values of packs[j][i] on
    the s^t_j of base_points[j]), all values as Python ints."""
    import torch

    cp = _params(pk.curve)
    r, w = cp.r, cp.fr_words
    lens = [[kzg._poly_len(p, w) for p in pack] for pack in packs]
    max_size, nb_points = _sizes([t * max(ln, default=0) for t, ln in zip(ts, lens)], ext_points)
    n_srs = pk.G1.shape[0]
    # the reference's Commit checks: W has maxSizePolys coefficients, W' has maxSizePolys + |T| - 1 (zero past maxSizePolys - 1)
    _check_size(max_size, 0, n_srs)
    _check_size(max_size + nb_points - 1, 1, n_srs)
    fs = _transcript(hf, ext_points, digests, pk.curve, data)
    gamma = _challenge(fs, "gamma", r)
    enc = lambda v: _fr_encode([v % r], r)[0]          # noqa: E731
    ys = [[pow(s, t, r) for s in S] for S, t in zip(base_points, ts)]
    with torch.cuda.device(pk.device):
        dp = kzg._DevicePoly(pk.curve, pk.device, max_size)
        d_in = [[kzg._device_poly(p, w, pk.device) if n else None for p, n in zip(pack, ln)] for pack, ln in zip(packs, lens)]
        slots = sum(len(pack) * len(y) for pack, y in zip(packs, ys))
        d_newton = torch.zeros(max(slots, 1) * w, dtype=torch.int64, device=dp.dev)
        # chained divisions: q_i = f_i / prod_{a in Y_j} (X - a), f(a) of each step into its Newton slot (0 once f is empty)
        q, slot = [], 0
        for j, (ln, y) in enumerate(zip(lens, ys)):
            for i, (cur, n) in enumerate(zip(d_in[j], ln)):
                for a in y:
                    if n:
                        h = dp.empty(n - 1) if n > 1 else None
                        dp.div(cur, n, enc(a), h, d_newton[slot * w:(slot + 1) * w])
                        cur, n = h, n - 1
                    slot += 1
                if n:
                    q.append((cur, n, j, i))
        gam = [1]
        for _ in range(1, len(packs)):
            gam.append(gam[-1] * gamma % r)
        # W = sum_j gamma^j interleave_t_j(q_j,i)
        d_W = dp.empty(max_size)
        if q:
            dp.lincomb([d for d, _, _, _ in q], [n for _, n, _, _ in q], _fr_encode([gam[j] for _, _, j, _ in q], r),
                       [ts[j] for _, _, j, _ in q], [i for _, _, _, i in q], d_W, max_size)
        else:
            d_W.zero_()
        W = kzg._digest(pk._bases.MultiExpDevice(d_W, max_size, stream=dp.stream), pk.words)
        fs.Bind("z", g1_raw_bytes(W, pk.curve))
        z = _challenge(fs, "z", r)
        # L = sum_j c_j F_j - Z_T(z) W, c_j = gamma^j Z_{T\S_j}(z); W' = quotient of L by (X - z)
        zdiff = [[(z - x) % r for x in S] for S in ext_points]
        zt_z = 1
        for dz in zdiff:
            for v in dz:
                zt_z = zt_z * v % r
        coef = []
        for j in range(len(packs)):
            cj = gam[j]
            for k, dz in enumerate(zdiff):
                if k != j:
                    for v in dz:
                        cj = cj * v % r
            coef.append(cj)
        ins = [(d, n, coef[j], ts[j], i) for j in range(len(packs)) for i, (d, n) in enumerate(zip(d_in[j], lens[j])) if n]
        ins.append((d_W, max_size, -zt_z % r, 1, 0))
        d_L = dp.empty(max_size)
        dp.lincomb([e[0] for e in ins], [e[1] for e in ins], _fr_encode([e[2] for e in ins], r), [e[3] for e in ins],
                   [e[4] for e in ins], d_L, max_size)
        if max_size > 1:
            d_Wp, d_lz = dp.empty(max_size - 1), dp.empty(1)
            dp.div(d_L, max_size, enc(z), d_Wp, d_lz)
            WPrime = kzg._digest(pk._bases.MultiExpDevice(d_Wp, max_size - 1, stream=dp.stream), pk.words)
        else:                       # W' is the zero polynomial (its |T| coefficients are all past maxSizePolys - 1)
            WPrime = np.zeros(pk.words, dtype=np.uint64)
        newton = _fr_decode(d_newton[:slots * w].cpu().numpy().view(np.uint64), r) if slots else []
    # Newton form on Y: f(y_m) = sum_{l <= m} c_l prod_{u < l} (y_m - y_u)
    values, slot = [], 0
    for pack, y in zip(packs, ys):
        vals = []
        for _ in pack:
            c = newton[slot:slot + len(y)]
            slot += len(y)
            row = []
            for m, ym in enumerate(y):
                acc, basis = 0, 1
                for l in range(m + 1):
                    acc = (acc + c[l] * basis) % r
                    basis = basis * (ym - y[l]) % r
                row.append(acc)
            vals.append(row)
        values.append(vals)
    # claimed values of the interleaves: F_j(x) = sum_i x^i p_i(x^t), x^t = s^t for x = s omega^k
    claimed = []
    for vals, t, S in zip(values, ts, ext_points):
        cl = []
        for idx, x in enumerate(S):
            m, acc, xp = idx // t, 0, 1
            for row in vals:
                acc = (acc + xp * row[m]) % r
                xp = xp * x % r
            cl.append(acc)
        claimed.append(cl)
    return W, WPrime, claimed, values


# ---- host restatement of shplonk.go, line by line (sharded proving keys and the tests' reference) ----

def _eval(f, x, r):
    """eval (shplonk.go:332-338)"""
    y = 0
    for v in reversed(f):
        y = (y * x + v) % r
    return y


def _multiply_linear_factor(f, a, r):
    """multiplyLinearFactor (shplonk.go:350-361): (X - a) f"""
    s = len(f)
    f = list(f) + [0]
    f[s] = f[s - 1]
    for i in range(s - 1, 0, -1):
        f[i] = (f[i - 1] - f[i] * a) % r
    f[0] = -f[0] * a % r
    return f


def _vanishing(xs, r):
    """buildVanishingPoly (shplonk.go:381-388)"""
    res = [1]
    for x in xs:
        res = _multiply_linear_factor(res, x, r)
    return res


def _zt_minus_si(points, i, r):
    """buildZtMinusSi (shplonk.go:364-378)"""
    return _vanishing([x for j, S in enumerate(points) if j != i for x in S], r)


def _lagrange(x, i, r):
    """buildLagrangeFromDomain (shplonk.go:406-415); fr.Inverse(0) = 0, so repeated points give a zero basis polynomial"""
    res = _vanishing(x[:i] + x[i + 1:], r)
    d = pow(_eval(res, x[i], r), r - 2, r)
    return [v * d % r for v in res]


def _interpolate(x, y, r):
    """interpolate (shplonk.go:391-403)"""
    res = [0] * len(x)
    for i in range(len(x)):
        li = _lagrange(x, i, r)
        for j in range(len(x)):
            res[j] = (res[j] + li[j] * y[i]) % r
    return res


def _mul(f, g, r):
    """mul (shplonk.go:429-446)"""
    res = [0] * (len(f) + len(g) - 1)
    for i, gi in enumerate(g):
        for j, fj in enumerate(f):
            res[j + i] = (res[j + i] + fj * gi) % r
    return res


def _div(f, g, r):
    """div (shplonk.go:452-464): the Euclidean quotient of f by the monic g"""
    f = list(f)
    sf, sg = len(f), len(g)
    for i in range(sf - 2, sg - 2, -1):
        for j in range(sg - 1):
            f[i - j] = (f[i - j] - f[i + 1] * g[sg - 2 - j]) % r
    return f[sg - 1:]


def batch_open_host(polys, points, digests, hf, curve: str, commit, *data):
    """BatchOpen (shplonk.go:44-172) on Python ints: polys[i] and points[i] lists of ints; commit(coeffs) -> digest limbs (kzg.Commit
    and its errors).  Returns (W, W', claimed values, w, w') with w and w' the committed coefficient lists."""
    r = _params(curve).r
    fs = _transcript(hf, points, digests, curve, data)
    gamma = _challenge(fs, "gamma", r)
    max_size, nb_points = _sizes([len(p) for p in polys], points)
    total = max_size + nb_points
    f = [0] * total
    claimed, zt_minus, ri = [], [], []
    acc = 1
    for i, p in enumerate(polys):
        claimed.append([_eval(p, x, r) for x in points[i]])
        zt_minus.append(_zt_minus_si(points, i, r))
        buf = list(p) + [0] * (max_size - len(p))
        ri.append(_interpolate(points[i], claimed[i], r))
        for j, v in enumerate(ri[i]):
            buf[j] = (buf[j] - v) % r
        for j, v in enumerate(_mul(buf, zt_minus[i], r)):
            f[j] = (f[j] + v * acc) % r
        acc = acc * gamma % r
    zt = _vanishing([x for S in points for x in S], r)
    w = _div(f, zt, r)
    W = commit(w)
    fs.Bind("z", g1_raw_bytes(W, curve))
    z = _challenge(fs, "z", r)
    acc = 1
    lpoly = [0] * total
    for i, p in enumerate(polys):
        ci = acc * _eval(zt_minus[i], z, r) % r
        buf = list(p) + [0] * (max_size - len(p))
        buf[0] = (buf[0] - _eval(ri[i], z, r)) % r
        for j in range(len(p)):                 # mulByConstant(buf[:len(polynomials[i])], ...)
            buf[j] = buf[j] * ci % r
        for j in range(max_size):
            lpoly[j] = (lpoly[j] + buf[j]) % r
        acc = acc * gamma % r
    ztz = _eval(zt, z, r)
    buft = [v * ztz % r for v in w] + [0] * (total - len(w))
    for i in range(total - max_size):
        lpoly[total - 1 - i] = -buft[total - 1 - i] % r
    for i in range(max_size):
        lpoly[i] = (lpoly[i] - buft[i]) % r
    wprime = _div(lpoly, _vanishing([z], r), r)
    WPrime = commit(wprime)
    return W, WPrime, claimed, w, wprime
