"""The host side of iop.py, CPU only: the expression tracer (supported operations, powers, constants, the index, a constant-only
expression, rejected operations, programs at and over the limits), WriteTo / ReadFrom round trips and one stream built byte by byte
in the reference's format, and the errors raised before any device work."""
import io
import random
import struct
from importlib import import_module

import numpy as np
import pytest

curves = import_module("gnark-crypto_b200.curves")
CURVES = ["bn254", "bls12381", "bls12377", "bls24315", "bls24317", "bw6633", "bw6761"]


def _iop():
    return import_module("gnark-crypto_b200.iop")


def _run(prog, i, xs, r):
    """the interpreter of k_iop_evaluate on Python ints"""
    reg = [None] * 16
    for w in prog.code:
        op, dst, a, b = w & 0xFF, (w >> 8) & 0xFF, (w >> 16) & 0xFF, w >> 24
        reg[dst] = [lambda: xs[a], lambda: prog.consts[a], lambda: i, lambda: (reg[a] + reg[b]) % r, lambda: (reg[a] - reg[b]) % r,
                    lambda: reg[a] * reg[b] % r, lambda: -reg[a] % r][op]()
    return reg[prog.out]


R = curves.CURVE_PARAMS["bn254"].r


@pytest.mark.parametrize("f,g,m", [
    (lambda i, a, b: a + b, lambda i, a, b: a + b, 2),
    (lambda i, a, b: a - 3 * b + 5, lambda i, a, b: a - 3 * b + 5, 2),
    (lambda i, a, b: -(a * b) - 1 + a, lambda i, a, b: -(a * b) - 1 + a, 2),
    (lambda i, a: 7 - a * i, lambda i, a: 7 - a * i, 1),
    (lambda i, a: a ** 0 + a ** 1 + a ** 2 + a ** 13, lambda i, a: 1 + a + a ** 2 + a ** 13, 1),
    (lambda i, a: (a + 1) ** 5 * 2 ** 70, lambda i, a: (a + 1) ** 5 * 2 ** 70, 1),
    (lambda i, a: -5, lambda i, a: -5, 1),
    (lambda i, a: i, lambda i, a: i, 1),
    (lambda i, a, b, c: a * b * c - (a + b) * (b + c) + i * i * c, lambda i, a, b, c: a * b * c - (a + b) * (b + c) + i * i * c, 3),
])
def test_trace_semantics(f, g, m):
    """each traced program, run by a Python model of the device interpreter, equals f on random field values"""
    prog = _iop().trace(f, m, R)
    rng = random.Random(1)
    for _ in range(20):
        xs = [rng.randrange(R) for _ in range(m)]
        i = rng.randrange(1 << 22)
        assert _run(prog, i, xs, R) == g(i, *xs) % R
    assert all((w & 0xFF) <= 6 for w in prog.code) and prog.live <= 16


def test_trace_constants_and_registers():
    """constants are reduced mod r and shared; a constant-only expression is one instruction; dead inputs emit nothing"""
    iop = _iop()
    p = iop.trace(lambda i, a, b: a * (R + 3) + b * 3 + (-1), 2, R)
    assert sorted(p.consts) == [3, R - 1]
    p = iop.trace(lambda i, a: 42, 1, R)
    assert p.code == [1] and p.consts == [42]
    p = iop.trace(lambda i, a, b, c: b, 3, R)
    assert len(p.code) == 1 and p.code[0] & 0xFF == 0 and (p.code[0] >> 16) & 0xFF == 1


@pytest.mark.parametrize("bad,name", [
    (lambda i, a: a / 2, "/"), (lambda i, a: a // 2, "//"), (lambda i, a: a % 2, "%"), (lambda i, a: a < 1, "<"),
    (lambda i, a: a == 1, "=="), (lambda i, a: 1 if a else 0, "bool()"), (lambda i, a: a ** -1, "exponent"),
    (lambda i, a: a ** a, "exponent"), (lambda i, a: 2 ** a, "traced exponent"), (lambda i, a: a * 1.5, "float"),
    (lambda i, a: a + "x", "str"), (lambda i, a: int(a), "int()"), (lambda i, a: a & 1, "&"), (lambda i, a: a ** True, "exponent"),
])
def test_trace_rejects(bad, name):
    iop = _iop()
    with pytest.raises(iop.IopError, match="unsupported") as e:
        iop.trace(bad, 1, R)
    assert name in str(e.value)


def test_trace_limits():
    """256 instructions and 16 live values are accepted, one more of either is refused"""
    iop = _iop()

    def chain(steps):
        def f(i, a):
            x = a
            for _ in range(steps):
                x = x * a
            return x
        return f

    assert len(iop.trace(chain(255), 1, R).code) == 256           # 1 load + 255 products
    with pytest.raises(iop.IopError, match="instructions"):
        iop.trace(chain(256), 1, R)

    # a sum over all 32 inputs, with the index and a constant: each input is loaded right before its use, so few values are live
    p = iop.trace(lambda i, *xs: sum(xs[1:], xs[0]) * i + 5, 32, R)
    assert p.live <= 3 and len(p.code) == 32 + 31 + 4
    rng = random.Random(4)
    xs = [rng.randrange(R) for _ in range(32)]
    assert _run(p, 77, xs, R) == (sum(xs) * 77 + 5) % R

    # 16 values live at once: the 16 squares are all formed before the product consumes them
    def all_live(n):
        def f(i, *xs):
            ys = [x * x for x in xs]     # every square stays live until the product chain reaches it
            acc = ys[0]
            for y in ys[1:]:
                acc = acc * y
            return acc
        return f

    assert iop.trace(all_live(16), 16, R).live == 16
    with pytest.raises(iop.IopError, match="live values"):
        iop.trace(all_live(17), 17, R)
    with pytest.raises(iop.IopError, match="constants"):
        iop.trace(lambda i, a: sum((a * k for k in range(2, 36)), a), 1, R)


@pytest.mark.parametrize("c", CURVES)
def test_write_read_round_trip(c):
    iop = _iop()
    cp = curves.CURVE_PARAMS[c]
    rng = random.Random(2)
    vals = [rng.randrange(cp.r) for _ in range(17)] + [0, cp.r - 1]
    p = iop.NewPolynomial(curves._fr_encode(vals, cp.r), iop.Form(iop.LagrangeCoset, iop.BitReverse), c)
    p.Shift(7)
    p.SetSize(4)
    p.coset = rng.randrange(cp.r)
    buf = io.BytesIO()
    n = p.WriteTo(buf)
    assert n == len(buf.getvalue()) == 4 + len(vals) * cp.fr_bytes + 16 + cp.fr_bytes
    q = iop.Polynomial(c)
    assert q.ReadFrom(io.BytesIO(buf.getvalue())) == n
    assert (q.Basis, q.Layout, q.shift, q.size, q.coset) == (iop.LagrangeCoset, iop.BitReverse, 7, 4, p.coset)
    assert (q.Coefficients() == p.Coefficients()).all()


def test_stream_byte_by_byte():
    """a stream written by hand in the reference's format: fr.Vector (u32 BE length, big-endian elements), basis, layout, shift,
    size as u32 BE, the coset big-endian; an element >= r is refused"""
    iop = _iop()
    r = R
    b = struct.pack(">I", 3) + (1).to_bytes(32, "big") + (r - 1).to_bytes(32, "big") + (5).to_bytes(32, "big")
    b += struct.pack(">IIII", 2, 16, 1, 2) + (9).to_bytes(32, "big")
    p = iop.Polynomial("bn254")
    assert p.ReadFrom(io.BytesIO(b)) == len(b)
    assert curves._fr_decode(p.Coefficients(), r) == [1, r - 1, 5]
    assert (p.Basis, p.Layout, p.shift, p.size, p.coset) == (2, 16, 1, 2, 9)
    out = io.BytesIO()
    p.WriteTo(out)
    assert out.getvalue() == b
    bad = b[:4] + r.to_bytes(32, "big") + b[36:]
    with pytest.raises(iop.IopError, match="invalid fr.Element encoding"):
        iop.Polynomial("bn254").ReadFrom(io.BytesIO(bad))
    with pytest.raises(EOFError):
        iop.Polynomial("bn254").ReadFrom(io.BytesIO(b[:-1]))


def _p(n, form=(2, 8), c="bn254"):
    iop = _iop()
    return iop.NewPolynomial(np.zeros((n, 4), dtype=np.uint64), iop.Form(*form), c)


def test_errors_before_device_work():
    """the reference's errors and the refusals that stand in for its panics, all raised before any device work"""
    iop = _iop()
    one = curves._fr_encode([1], R)[0]
    F = iop.Form(2, 8)
    with pytest.raises(iop.ErrNumberPolynomials, match="^the number of polynomials"):
        iop.BuildRatioShuffledVectors([_p(8)], [_p(8), _p(8)], one, F)
    with pytest.raises(iop.IopError, match="index out of range"):       # checkSize reads [1] of a list of one: a panic
        iop.BuildRatioShuffledVectors([_p(8)], [_p(8)], one, F)
    with pytest.raises(iop.ErrInconsistentSize, match="^the sizes of the polynomial"):
        iop.BuildRatioShuffledVectors([_p(8), _p(4)], [_p(8), _p(8)], one, F)
    with pytest.raises(iop.ErrSizeNotPowerOfTwo):
        iop.BuildRatioShuffledVectors([_p(6), _p(6)], [_p(6), _p(6)], one, F)
    with pytest.raises(iop.ErrInconsistentSize):                         # unchecked by checkSize, longer than the domain
        iop.BuildRatioShuffledVectors([_p(8), _p(8), _p(16)], [_p(8), _p(8), _p(8)], one, F)
    with pytest.raises(iop.IopError, match="index out of range"):
        iop.BuildRatioCopyConstraint([], np.zeros(0, dtype=np.int64), one, one, F)
    with pytest.raises(iop.ErrSizeNotPowerOfTwo):
        iop.BuildRatioCopyConstraint([_p(6)], np.zeros(6, dtype=np.int64), one, one, F)
    with pytest.raises(iop.ErrInconsistentSize):                         # entries[1] is not checked by checkSize, but longer
        iop.BuildRatioCopyConstraint([_p(8), _p(16)], np.zeros(16, dtype=np.int64), one, one, F)
    sigma = np.arange(16, dtype=np.int64)
    for bad in (-1, 16):
        s = sigma.copy()
        s[5] = bad
        with pytest.raises(iop.IopError, match="outside"):
            iop.BuildRatioCopyConstraint([_p(8), _p(8)], s, one, one, F)
    with pytest.raises(iop.IopError, match="k n"):
        iop.BuildRatioCopyConstraint([_p(8), _p(8)], sigma[:15], one, one, F)
    with pytest.raises(iop.IopError, match="^need at lest one input$"):
        iop.Evaluate(lambda i: 1, None, F)
    with pytest.raises(iop.ErrInconsistentSize):
        iop.Evaluate(lambda i, a, b: a, None, F, _p(8), _p(4))
    with pytest.raises(iop.ErrInconsistentSize):
        iop.Evaluate(lambda i, a: a, np.zeros((4, 4), dtype=np.uint64), F, _p(8))
    with pytest.raises(iop.IopError, match="unsupported"):
        iop.Evaluate(lambda i, a: a / 3, None, F, _p(8))

    class Dom:
        Cardinality, device = 8, 0

    class Big:
        Cardinality, device = 32, 0

    with pytest.raises(iop.ErrMustBeLagrangeCoset, match="^the basis must be LagrangeCoset$"):
        iop.DivideByXMinusOne(_p(32, (1, 8)), [Dom(), Big()])
    q = _p(32, (4, 16))
    q.SetSize(16)            # len / size = 2, the domains' ratio is 4: the reference would index past its table
    with pytest.raises(iop.IopError, match="ratio"):
        iop.DivideByXMinusOne(q, [Dom(), Big()])
    assert issubclass(iop.IopError, import_module("gnark-crypto_b200.multiexp").MultiExpError)
