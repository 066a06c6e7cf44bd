"""Big-int restatement of kzg.ToLagrangeG1 (ecc/bn254/kzg/utils.go:25-64; the kzg packages of the other pairing curves are the
same generated code) on the oracle's group operations (TEST INFRASTRUCTURE).

`to_lagrange_g1` follows the reference step by step: the power-of-two check, computeTwiddlesInv (fr.Generator(n) inverted, its
"too big" error), difFFTG1 (butterfly, then the twiddle multiplication for i >= 1, then the two halves at the next stage),
bitReverse, the scaling by 1/n and the affine normal form.  `to_lagrange_scalars` runs the same steps on discrete logarithms:
for points [a_j]G the result is [b_j]G with b = to_lagrange_scalars(a) -- a cheap reference for large n."""
from oracle import oracle as O

from tests import fft_more_fields

CURVES = ("bn254", "bls12381", "bls12377", "bls24315", "bls24317", "bw6633", "bw6761")
FFT_PARAMS = dict(O.FFT_PARAMS, **fft_more_fields.FFT_PARAMS)


class LagrangeError(ValueError):
    pass


def group(curve: str) -> O.Group:
    return O.GROUPS[curve + "_g1"]


def fr_modulus(curve: str) -> int:
    return group(curve).fr.q


def domain_inverses(curve: str, n: int):
    """(w^-1, 1/n) of fr.Generator(n) (generator.go:18-36), with the reference's errors"""
    if n <= 0 or n & (n - 1):
        raise LagrangeError("len(coeffs) must be a power of 2")
    P = FFT_PARAMS[curve + "_fr"]
    r = fr_modulus(curve)
    logn = n.bit_length() - 1
    if logn > P["max_order"]:
        raise LagrangeError("m (%d) is too big: the required root of unity does not exist" % n)
    w = pow(P["root"], 1 << (P["max_order"] - logn), r)
    return pow(w, -1, r), pow(n, -1, r)


def twiddles_inv(curve: str, n: int) -> list:
    """computeTwiddlesInv (utils.go:66-93): w^-j for j <= n / 2 (just [1] for n = 1)"""
    w_inv, _ = domain_inverses(curve, n)
    r = fr_modulus(curve)
    out = [1]
    for _ in range(n // 2):
        out.append(out[-1] * w_inv % r)
    return out


def dif_fft(a: list, tw: list, add, sub, mul, stage: int = 0) -> None:
    """difFFTG1 (utils.go:119-172) over any group given by add / sub / mul(x, k), in place"""
    n = len(a)
    if n == 1:
        return
    m = n >> 1
    stride = 1 << stage
    for i in range(m):
        x, y = a[i], a[i + m]
        a[i] = add(x, y)
        a[i + m] = sub(x, y)
        if i:
            a[i + m] = mul(a[i + m], tw[i * stride])
    if m == 1:
        return
    left, right = a[:m], a[m:]
    dif_fft(left, tw, add, sub, mul, stage + 1)
    dif_fft(right, tw, add, sub, mul, stage + 1)
    a[:m], a[m:] = left, right


def _run(curve: str, vals: list, add, sub, mul) -> list:
    n = len(vals)
    _, n_inv = domain_inverses(curve, n)
    tw = twiddles_inv(curve, n)
    a = list(vals)
    dif_fft(a, tw, add, sub, mul)
    O.bit_reverse(a)
    return [mul(v, n_inv) for v in a]


def to_lagrange_g1(curve: str, points: list) -> list:
    """ToLagrangeG1 on oracle affine points ((0, 0) = infinity); returns affine points"""
    G = group(curve)
    return _run(curve, points, G.aff_add, lambda p, q: G.aff_add(p, G.aff_neg(q)), G.scalar_mul)


def to_lagrange_scalars(curve: str, ks: list) -> list:
    """the same transform on the discrete logarithms of the points (integers mod r)"""
    r = fr_modulus(curve)
    return _run(curve, [k % r for k in ks], lambda x, y: (x + y) % r, lambda x, y: (x - y) % r, lambda x, k: x * k % r)
