"""The iop package (ecc/bn254/fr/iop: polynomial.go, expressions.go, ratios.go, quotient.go; the iop packages of bls12-381, bls12-377,
bls24-315, bls24-317, bw6-633 and bw6-761 are the same generated code) with every O(n) step on the GPU.

  * Polynomial, Form, Basis, Layout; the form changes (ToRegular, ToBitReverse, ToLagrange, ToCanonical, ToLagrangeCoset) call
    fft.Domain's device FFTs with the decimation, inverse and coset flags of the reference (polynomial.go:263-390);
    Polynomial.Evaluate (polynomial.go:104-261) runs the opening scan (Canonical) or a barycentric reduction (Lagrange);
  * Evaluate(f, r, form, *x): f, a Python callable, is traced once into a straight-line program that one device kernel interprets
    at every position (csrc/iop_kernels.cuh, k_iop_evaluate);
  * BuildRatioShuffledVectors, BuildRatioCopyConstraint: one fused ratio kernel each, then the exclusive prefix product of
    permutation.Prove;
  * DivideByXMinusOne: one elementwise kernel, then the inverse FFT.
Coefficients are numpy (n, fr.Limbs) uint64 arrays or contiguous torch int64 CUDA tensors (the layout of kzg._device_poly).  A host
array is uploaded once and downloaded once per call, in place when its length does not change (a growing buffer is replaced, as
Go's append replaces a full slice); a device tensor never leaves its device.  The inputs of one call are all on the host or all on
one device."""
from __future__ import annotations

import struct
from dataclasses import dataclass

import numpy as np

from . import _native
from .curves import CURVE_PARAMS, _fr_decode, _fr_encode, _params
from .fft import DIF, DIT, Domain
from .kzg import _DevicePoly, _device_poly, _is_device
from .multiexp import MultiExpError

Canonical, Lagrange, LagrangeCoset = 1, 2, 4   # iop.Basis
Regular, BitReverse = 8, 16                    # iop.Layout

# limits of the device kernels (include/gmsm.h)
MAX_COLUMNS, MAX_PROGRAM, MAX_REGISTERS, MAX_INPUTS, MAX_CONSTS, MAX_RHO = 32, 256, 16, 32, 32, 64


class IopError(MultiExpError):
    """an error of the iop package"""

    message = "iop error"

    def __init__(self, *args):
        super().__init__(*(args or (self.message,)))


class ErrMustBeRegular(IopError):
    message = "the layout must be Regular"


class ErrMustBeCanonical(IopError):
    message = "the basis must be Canonical"


class ErrMustBeLagrangeCoset(IopError):
    message = "the basis must be LagrangeCoset"


class ErrInconsistentFormat(IopError):
    message = "the format of the polynomials must be the same"


class ErrInconsistentSize(IopError):
    message = "the sizes of the polynomial must be the same as the size of the domain"


class ErrNumberPolynomials(IopError):
    message = "the number of polynomials in the denominator and the numerator must be the same"


class ErrSizeNotPowerOfTwo(IopError):
    message = "the size of the polynomials must be a power of two"


class ErrInconsistentSizeDomain(IopError):
    message = "the size of the domain must be consistent with the size of the polynomials"


class ErrIncorrectNumberOfVariables(IopError):
    message = "the number of variables is incorrect"


@dataclass(frozen=True)
class Form:
    Basis: int
    Layout: int


def _curve_name(curve: str) -> str:
    c = curve[:-3] if curve.endswith("_g1") else curve
    if c not in CURVE_PARAMS:
        raise IopError("unknown curve %r (iop: %s)" % (curve, ", ".join(CURVE_PARAMS)))
    return c


_DOMAINS: dict = {}
_MAX_DOMAINS = 2


def _domain(curve: str, n: int, device: int) -> Domain:
    """fft.NewDomain(n) of the curve's scalar field on `device` for the Lagrange evaluation and for the ratio builders called without
    a domain; the last two are kept for later calls (ClearDomainCache releases them)"""
    key = (curve, n, device)
    if key not in _DOMAINS:
        if len(_DOMAINS) >= _MAX_DOMAINS:
            _DOMAINS.pop(next(iter(_DOMAINS))).close()
        _DOMAINS[key] = Domain(curve, n, device=device)
    return _DOMAINS[key]


def ClearDomainCache():
    """frees the device twiddle tables of the domains iop built for itself"""
    while _DOMAINS:
        _DOMAINS.popitem()[1].close()


def _generator(curve: str, m: int) -> int:
    """fr.Generator(m) (generator.go:18-36) on the host, as a regular integer"""
    from .multiexp import _check

    cp = _params(curve)
    out = np.zeros(cp.fr_words, dtype=np.uint64)
    _check(_native.lib().gmsm_fr_generator(cp.fr_id, m, out.ctypes.data))
    return _fr_decode(out, cp.r)[0]


class _Inner:
    """iop.polynomial: the coefficient buffer and the form, shared by ShallowClone"""

    def __init__(self, coefficients, basis: int, layout: int):
        self.coefficients = coefficients
        self.Basis = basis
        self.Layout = layout


def _length(c, words: int) -> int:
    return c.numel() // words if _is_device(c) else c.shape[0]


def _host_array(c, words: int) -> np.ndarray:
    a = np.asarray(c)
    if a.dtype == np.uint64 and a.ndim == 2 and a.shape[1] == words and a.flags["C_CONTIGUOUS"] and a.flags.writeable:
        return a
    return np.ascontiguousarray(a, dtype=np.uint64).reshape(-1, words).copy()


def _device_of(inners) -> int | None:
    """None when every buffer is on the host, the device index when every buffer is a tensor on it; a mixed call raises"""
    devs = {c.coefficients.device.index if _is_device(c.coefficients) else None for c in inners}
    if len(devs) != 1:
        raise IopError("the polynomials of one call must all be host arrays or all be tensors on one device")
    return devs.pop()


class _Staged:
    """the buffers of a call on the device: host arrays uploaded once on entry and written back once on exit (in place when the
    length did not change)"""

    def __init__(self, inners, device: int, words: int):
        self.words = words
        self.host = []
        seen = set()
        for p in inners:
            if id(p) in seen or _is_device(p.coefficients):
                continue
            seen.add(id(p))
            self.host.append((p, p.coefficients))
            p.coefficients = _device_poly(p.coefficients, words, device)

    def done(self):
        for p, arr in self.host:
            h = p.coefficients.cpu().numpy().view(np.uint64).reshape(-1, self.words)
            if h.shape == arr.shape:
                np.copyto(arr, h)
                p.coefficients = arr
            else:
                p.coefficients = h.copy()
        self.host = []


def _torch():
    import torch

    return torch


def _check_rev(n: int):
    if n & (n - 1) or n == 0:
        raise ErrSizeNotPowerOfTwo()


class Polynomial:
    """iop.Polynomial: P'(X) = P(w^shift X), of real size `size`; `coset` is set by ToLagrangeCoset"""

    def __init__(self, curve: str, inner: _Inner = None, shift: int = 0, size: int = 0, coset: int = 0):
        self.curve = _curve_name(curve)
        self._cp = _params(self.curve)
        self._p = inner
        self.shift = shift
        self.size = size
        self.coset = coset   # regular (not Montgomery) integer

    # -- accessors --
    @property
    def Basis(self) -> int:
        return self._p.Basis

    @Basis.setter
    def Basis(self, v: int):
        self._p.Basis = v

    @property
    def Layout(self) -> int:
        return self._p.Layout

    @Layout.setter
    def Layout(self, v: int):
        self._p.Layout = v

    @property
    def Form(self) -> Form:
        return Form(self._p.Basis, self._p.Layout)

    def _words(self) -> int:
        return self._cp.fr_words

    def _len(self) -> int:
        return _length(self._p.coefficients, self._words())

    def Shift(self, shift: int) -> "Polynomial":
        self.shift = shift
        return self

    def Size(self) -> int:
        return self.size

    def SetSize(self, size: int):
        self.size = size

    def Coefficients(self):
        return self._p.coefficients

    def ShallowClone(self) -> "Polynomial":
        return Polynomial(self.curve, self._p, self.shift, self.size, self.coset)

    def Clone(self, *capacity: int) -> "Polynomial":
        c = self._p.coefficients
        c = c.clone() if _is_device(c) else c.copy()
        res = self.ShallowClone()
        res._p = _Inner(c, self._p.Basis, self._p.Layout)
        return res

    def GetCoeff(self, i: int) -> np.ndarray:
        n = self._len()
        rho = n // self.size
        s = (i + rho * self.shift) % n
        if self.Layout != Regular:
            tz = (n & -n).bit_length() - 1
            s = int(bin(s)[2:].zfill(64)[::-1], 2) >> (64 - tz) if tz else 0
        c = self._p.coefficients
        if _is_device(c):
            w = self._words()
            return c[s * w:(s + 1) * w].cpu().numpy().view(np.uint64).copy()
        return np.array(c[s], dtype=np.uint64)

    # -- form changes (polynomial.go:263-390) --
    def _grow(self, n: int):
        c, w = self._p.coefficients, self._words()
        m = _length(c, w)
        if m < n:
            if _is_device(c):
                torch = _torch()
                self._p.coefficients = torch.cat([c, torch.zeros((n - m) * w, dtype=torch.int64, device=c.device)])
            else:
                self._p.coefficients = np.concatenate([c, np.zeros((n - m, w), dtype=np.uint64)])

    def _transform(self, d: Domain, steps, grow: int = None):
        """runs `steps` on the coefficients: ("fft", inverse, decimation, coset) on `d`, ("br",) a bit reversal of the whole buffer"""
        dev = _device_of([self._p])
        device = d.device if d is not None else (0 if dev is None else dev)
        if dev is not None and d is not None and dev != d.device:
            raise IopError("the polynomial is on cuda:%d, the domain on cuda:%d" % (dev, d.device))
        if grow is not None:
            self._grow(grow)
        if not steps:
            return
        n = self._len()
        if d is not None and n != d.Cardinality:
            raise ErrInconsistentSize()
        _check_rev(n)
        torch = _torch()
        with torch.cuda.device(device):
            st = _Staged([self._p], device, self._words())
            try:
                _run_steps(self._p.coefficients, self.curve, d, steps, device)
            finally:
                st.done()

    def ToRegular(self) -> "Polynomial":
        if self.Layout == Regular:
            return self
        self._transform(None, [("br",)])
        self.Layout = Regular
        return self

    def ToBitReverse(self) -> "Polynomial":
        if self.Layout == BitReverse:
            return self
        self._transform(None, [("br",)])
        self.Layout = BitReverse
        return self

    def ToLagrange(self, d: Domain) -> "Polynomial":
        f = self.Form
        card = d.Cardinality
        if f == Form(Canonical, Regular):
            self._transform(d, [("fft", False, DIF, False)], card)
            self.Layout = BitReverse
        elif f == Form(Canonical, BitReverse):
            self._transform(d, [("fft", False, DIT, False)], card)
            self.Layout = Regular
        elif f in (Form(Lagrange, Regular), Form(Lagrange, BitReverse)):
            self._transform(d, [], card)
            return self
        elif f == Form(LagrangeCoset, Regular):
            self._transform(d, [("fft", True, DIF, True), ("fft", False, DIT, False)], card)
            self.Layout = Regular
        elif f == Form(LagrangeCoset, BitReverse):
            self._transform(d, [("fft", True, DIT, True), ("fft", False, DIF, False)], card)
            self.Layout = BitReverse
        else:
            raise IopError("unknown ID")
        self.Basis = Lagrange
        return self

    def ToCanonical(self, d: Domain) -> "Polynomial":
        f = self.Form
        card = d.Cardinality
        if f in (Form(Canonical, Regular), Form(Canonical, BitReverse)):
            self._transform(d, [], card)
            return self
        table = {Form(Lagrange, Regular): (BitReverse, DIF, False), Form(Lagrange, BitReverse): (Regular, DIT, False),
                 Form(LagrangeCoset, Regular): (BitReverse, DIF, True), Form(LagrangeCoset, BitReverse): (Regular, DIT, True)}
        if f not in table:
            raise IopError("unknown ID")
        layout, dec, coset = table[f]
        self._transform(d, [("fft", True, dec, coset)], card)
        self.Layout = layout
        self.Basis = Canonical
        return self

    def ToLagrangeCoset(self, d: Domain) -> "Polynomial":
        self.coset = _fr_decode(d.FrMultiplicativeGen, self._cp.r)[0]   # CosetTable()[1]
        f = self.Form
        card = d.Cardinality
        table = {Form(Canonical, Regular): (BitReverse, [("fft", False, DIF, True)]),
                 Form(Canonical, BitReverse): (Regular, [("fft", False, DIT, True)]),
                 Form(Lagrange, Regular): (Regular, [("fft", True, DIF, False), ("fft", False, DIT, True)]),
                 Form(Lagrange, BitReverse): (BitReverse, [("fft", True, DIT, False), ("fft", False, DIF, True)])}
        if f in (Form(LagrangeCoset, Regular), Form(LagrangeCoset, BitReverse)):
            self._transform(d, [], card)
            return self
        if f not in table:
            raise IopError("unknown ID")
        layout, steps = table[f]
        self._transform(d, steps, card)
        self.Layout = layout
        self.Basis = LagrangeCoset
        return self

    # -- evaluation (polynomial.go:104-261) --
    def Evaluate(self, x) -> np.ndarray:
        """p(x) as fr.Element limbs: x is divided by the coset in LagrangeCoset basis (a zero coset gives x = 0) and multiplied by
        Generator(size)^shift for 0 < shift <= 5; for shift > 5 (and shift < 0) the reference multiplies by an unset (zero) element,
        so p is evaluated at 0"""
        r = self._cp.r
        xv = _fr_decode(np.asarray(x, dtype=np.uint64), r)[0]
        if self.Basis == LagrangeCoset:
            xv = xv * (pow(self.coset, r - 2, r)) % r          # x.Div(x, coset): Inverse(0) = 0
        dev = _device_of([self._p])
        device = 0 if dev is None else dev
        if self.shift != 0:
            if 0 < self.shift <= 5:
                if self.size <= 0:
                    raise IopError("size (%d) must be positive" % self.size)
                g = _generator(self.curve, self.size)
                xv = xv * pow(g, self.shift, r) % r
            else:
                xv = 0                                         # smallExp(..) / g.Exp(g, shift) of a zero g
        return self._evaluate(xv, device)

    def _evaluate(self, xv: int, device: int) -> np.ndarray:
        cp = self._cp
        n, w = self._len(), cp.fr_words
        if n == 0:
            return np.zeros(w, dtype=np.uint64)
        x = _fr_encode([xv], cp.r)[0]
        torch = _torch()
        with torch.cuda.device(device):
            dp = _DevicePoly(self.curve, device, n)
            d = _device_poly(self._p.coefficients, w, device)
            out = dp.empty(1)
            bitrev = self.Layout != Regular
            if self.Basis == Canonical:
                if bitrev:
                    _check_rev(n)
                    d = d.clone()
                    dp.bit_reverse(d, n)
                dp.div(d, n, x, None, out)
            else:
                _check_rev(n)
                dp.iop_lagrange_eval(_domain(self.curve, n, device), d, bitrev, x, out)
            return out.cpu().numpy().view(np.uint64).copy()

    # -- serialisation (polynomial.go:392-471) --
    def WriteTo(self, w) -> int:
        cp = self._cp
        vals = _fr_decode(_host_array(_to_host(self._p.coefficients, cp.fr_words), cp.fr_words), cp.r) if self._len() else []
        nb = 8 * cp.fr_words
        buf = bytearray(struct.pack(">I", len(vals)))
        for v in vals:
            buf += v.to_bytes(nb, "big")
        buf += struct.pack(">IIII", self.Basis & 0xFFFFFFFF, self.Layout & 0xFFFFFFFF, self.shift & 0xFFFFFFFF, self.size & 0xFFFFFFFF)
        buf += self.coset.to_bytes(nb, "big")
        w.write(bytes(buf))
        return len(buf)

    def ReadFrom(self, r) -> int:
        cp = self._cp
        nb = 8 * cp.fr_words

        def read(k):
            b = r.read(k)
            if len(b) != k:
                raise EOFError("unexpected EOF")
            return b

        def element(b):
            v = int.from_bytes(b, "big")
            if v >= cp.r:
                raise IopError("invalid fr.Element encoding")
            return v

        (m,) = struct.unpack(">I", read(4))
        vals = [element(read(nb)) for _ in range(m)]
        basis, layout, shift, size = struct.unpack(">IIII", read(16))
        coset = element(read(nb))
        self._p = _Inner(_fr_encode(vals, cp.r), basis, layout)
        self.shift = shift          # int(uint32) on a 64-bit Go int keeps the value
        self.size = size
        self.coset = coset
        return 4 + m * nb + 16 + nb


def _to_host(c, words: int):
    return c.cpu().numpy().view(np.uint64).reshape(-1, words) if _is_device(c) else c


def _run_steps(d_a, curve: str, d: Domain, steps, device: int):
    from .kzg import _stream

    st = _stream(device)
    for s in steps:
        if s[0] == "br":
            _DevicePoly(curve, device, 1).bit_reverse(d_a, _length(d_a, _params(curve).fr_words))
        else:
            _, inverse, dec, coset = s
            d.fft_device(d_a, inverse, dec, coset, st)


def NewPolynomial(coeffs, form: Form, curve: str) -> Polynomial:
    """iop.NewPolynomial: the coefficients are not copied (a host array is used in place when it is a C-contiguous (n, fr.Limbs)
    uint64 array; a device tensor must be a contiguous int64 CUDA tensor)"""
    cp = _params(_curve_name(curve))
    w = cp.fr_words
    if _is_device(coeffs):
        torch = _torch()
        if not coeffs.is_cuda or coeffs.dtype != torch.int64 or not coeffs.is_contiguous() or coeffs.numel() % w:
            raise IopError("a device polynomial must be a contiguous torch.int64 CUDA tensor of whole fr.Elements")
        c = coeffs.view(-1)
    else:
        c = _host_array(coeffs, w)
    return Polynomial(curve, _Inner(c, form.Basis, form.Layout), 0, _length(c, w))


# ---------------------------------------------------------------------------------------------------------------------------
# Evaluate (expressions.go): a traced straight-line program
# ---------------------------------------------------------------------------------------------------------------------------
_OP_INPUT, _OP_CONST, _OP_INDEX, _OP_ADD, _OP_SUB, _OP_MUL, _OP_NEG = range(7)


class _Tracer:
    def __init__(self, r: int):
        self.r = r
        self.nodes = []       # (op, a, b): a, b node ids (ADD/SUB/MUL/NEG), input j (INPUT), value (CONST)
        self.consts = {}

    def node(self, op, a=0, b=0) -> "_Sym":
        self.nodes.append((op, a, b))
        return _Sym(self, len(self.nodes) - 1)

    def const(self, v: int) -> "_Sym":
        v %= self.r
        if v not in self.consts:
            self.consts[v] = self.node(_OP_CONST, v)
        return self.consts[v]

    def operand(self, v, what: str) -> int:
        if isinstance(v, _Sym) and v.t is self:
            return v.i
        if isinstance(v, int) and not isinstance(v, bool):
            return self.const(v).i
        raise IopError("iop.Evaluate: unsupported operand %r for %s in the expression" % (type(v).__name__, what))


def _unsupported(name):
    def f(self, *args):
        raise IopError("iop.Evaluate: unsupported operation %s in the expression (supported: +, -, *, unary -, ** int)" % name)

    return f


class _Sym:
    """a traced value: the index i, an input, or an expression over them"""

    __slots__ = ("t", "i")
    __array_ufunc__ = None
    __hash__ = object.__hash__

    def __init__(self, t: _Tracer, i: int):
        self.t, self.i = t, i

    def __add__(self, o):
        return self.t.node(_OP_ADD, self.i, self.t.operand(o, "+"))

    def __radd__(self, o):
        return self.t.node(_OP_ADD, self.t.operand(o, "+"), self.i)

    def __sub__(self, o):
        return self.t.node(_OP_SUB, self.i, self.t.operand(o, "-"))

    def __rsub__(self, o):
        return self.t.node(_OP_SUB, self.t.operand(o, "-"), self.i)

    def __mul__(self, o):
        return self.t.node(_OP_MUL, self.i, self.t.operand(o, "*"))

    def __rmul__(self, o):
        return self.t.node(_OP_MUL, self.t.operand(o, "*"), self.i)

    def __neg__(self):
        return self.t.node(_OP_NEG, self.i)

    def __pow__(self, e, mod=None):
        if mod is not None or not isinstance(e, int) or isinstance(e, bool) or e < 0:
            raise IopError("iop.Evaluate: unsupported operation ** with exponent %r (a non-negative int is required)" % (e,))
        if e == 0:
            return self.t.const(1)
        res, base = None, self
        while e:                                  # square-and-multiply from the low bit
            if e & 1:
                res = base if res is None else res * base
            e >>= 1
            if e:
                base = base * base
        return res

    __truediv__ = __rtruediv__ = _unsupported("/")
    __floordiv__ = __rfloordiv__ = _unsupported("//")
    __mod__ = __rmod__ = __divmod__ = __rdivmod__ = _unsupported("%")
    __rpow__ = _unsupported("** (with a traced exponent)")
    __lt__ = _unsupported("<")
    __le__ = _unsupported("<=")
    __gt__ = _unsupported(">")
    __ge__ = _unsupported(">=")
    __eq__ = _unsupported("==")
    __ne__ = _unsupported("!=")
    __bool__ = _unsupported("bool()")
    __int__ = __index__ = _unsupported("int()")
    __float__ = _unsupported("float()")
    __pos__ = _unsupported("unary +")
    __abs__ = _unsupported("abs()")
    __invert__ = _unsupported("~")
    __lshift__ = __rlshift__ = _unsupported("<<")
    __rshift__ = __rrshift__ = _unsupported(">>")
    __and__ = __rand__ = _unsupported("&")
    __or__ = __ror__ = _unsupported("|")
    __xor__ = __rxor__ = _unsupported("^")
    __matmul__ = __rmatmul__ = _unsupported("@")


@dataclass
class Program:
    """a lowered expression: instruction words (op | dst << 8 | a << 16 | b << 24), the register of the result, the constants
    (regular integers) and the peak number of live values"""

    code: list
    out: int
    consts: list
    live: int


def trace(f, nb_inputs: int, r: int) -> Program:
    """calls f(i, x_0, ..., x_{m-1}) once on symbols and lowers the result to a straight-line program over at most MAX_REGISTERS
    registers (slots assigned by liveness, each leaf loaded right before its first use); raises IopError for an unsupported operation or a program over the limits"""
    t = _Tracer(r)
    idx = t.node(_OP_INDEX)
    xs = [t.node(_OP_INPUT, j) for j in range(nb_inputs)]
    res = f(idx, *xs)
    out = t.operand(res, "the result")
    # the nodes the result depends on, in creation (topological) order
    need, stack = set(), [out]
    while stack:
        k = stack.pop()
        if k in need:
            continue
        need.add(k)
        op, a, b = t.nodes[k]
        if op in (_OP_ADD, _OP_SUB, _OP_MUL):
            stack += [a, b]
        elif op == _OP_NEG:
            stack.append(a)
    # operations in creation (topological) order; each leaf (input, index, constant) just before its first use, so that it is live
    # only from there to its last use
    order, placed = [], set()
    for k in sorted(need):
        op, a, b = t.nodes[k]
        if op not in (_OP_ADD, _OP_SUB, _OP_MUL, _OP_NEG):
            continue
        for u in (a, b) if op != _OP_NEG else (a,):
            if u not in placed and t.nodes[u][0] in (_OP_INPUT, _OP_INDEX, _OP_CONST):
                placed.add(u)
                order.append(u)
        order.append(k)
    if out not in placed and t.nodes[out][0] in (_OP_INPUT, _OP_INDEX, _OP_CONST):
        order.append(out)                              # the result is a leaf: one load
    if len(order) > MAX_PROGRAM:
        raise IopError("iop.Evaluate: the expression needs %d instructions (at most %d)" % (len(order), MAX_PROGRAM))
    last = {}
    for pos, k in enumerate(order):
        op, a, b = t.nodes[k]
        for u in ((a, b) if op in (_OP_ADD, _OP_SUB, _OP_MUL) else (a,) if op == _OP_NEG else ()):
            last[u] = pos
    last[out] = len(order)
    consts, cidx = [], {}
    reg, free, code, live, peak = {}, list(range(MAX_REGISTERS)), [], 0, 0
    for pos, k in enumerate(order):
        op, a, b = t.nodes[k]
        ra = rb = 0
        if op in (_OP_ADD, _OP_SUB, _OP_MUL, _OP_NEG):
            ra = reg[a]
            rb = reg[b] if op != _OP_NEG else 0
            for u in {a, b} if op != _OP_NEG else {a}:
                if last[u] == pos:                     # the operand dies here: its slot can take the result
                    free.append(reg.pop(u))
                    live -= 1
            free.sort()
        elif op == _OP_CONST:
            if a not in cidx:
                if len(consts) == MAX_CONSTS:
                    raise IopError("iop.Evaluate: the expression has more than %d distinct constants" % MAX_CONSTS)
                cidx[a] = len(consts)
                consts.append(a)
            ra = cidx[a]
        elif op == _OP_INPUT:
            ra = a
        if not free:
            raise IopError("iop.Evaluate: the expression needs more than %d live values" % MAX_REGISTERS)
        dst = free.pop(0)
        reg[k] = dst
        live += 1
        peak = max(peak, live)
        code.append(op | dst << 8 | ra << 16 | rb << 24)
    return Program(code, reg[out], consts, peak)


def _offset(p: Polynomial, n: int) -> int:
    """(rho shift) mod n of GetCoeff, rho = len / size"""
    if p.size <= 0:
        raise IopError("size (%d) must be positive" % p.size)
    s = (n // p.size) * p.shift
    if s < 0:
        raise IopError("shift %d reads before the start of the coefficients" % p.shift)
    return s % n


def Evaluate(f, r, form: Form, *x: Polynomial) -> Polynomial:
    """iop.Evaluate: the polynomial whose coefficient idx(i) is f(i, x_0.GetCoeff(i), ...), idx(i) = i for a Regular form and
    the bit reversal of i otherwise; size = x[0].size, shift = 0.  `r`: None or a host array / device tensor of n elements that
    becomes the result's buffer.  `f` is traced once (trace) and run by the device interpreter."""
    if len(x) == 0:
        raise IopError("need at lest one input")
    cp = x[0]._cp
    w = cp.fr_words
    n = x[0]._len()
    for p in x[1:]:
        if p._len() != n:
            raise ErrInconsistentSize()
    if r is not None and (_length(r, w) if _is_device(r) else _host_array(r, w).shape[0]) != n:
        raise ErrInconsistentSize()
    if len(x) > MAX_INPUTS:
        raise IopError("iop.Evaluate: %d inputs (at most %d)" % (len(x), MAX_INPUTS))
    if n == 0:
        raise IopError("empty polynomials")
    prog = trace(f, len(x), cp.r)
    offsets = [_offset(p, n) for p in x]
    res_inner = _Inner(r if _is_device(r) or r is None else _host_array(r, w), form.Basis, form.Layout)
    dev = _device_of([p._p for p in x] + ([res_inner] if r is not None else []))
    device = 0 if dev is None else dev
    torch = _torch()
    with torch.cuda.device(device):
        dp = _DevicePoly(x[0].curve, device, 1)
        st = _Staged([p._p for p in x], device, w)
        try:
            d_r = r.view(-1) if _is_device(r) else dp.empty(n)
            dp.iop_evaluate(np.array(prog.code, dtype=np.uint32), prog.out, _fr_encode(prog.consts, cp.r).reshape(-1, w),
                            [p._p.coefficients for p in x], offsets, [p.Layout != Regular for p in x], n, form.Layout != Regular, d_r)
        finally:
            st.done()
        if dev is None:
            h = d_r.cpu().numpy().view(np.uint64).reshape(-1, w)
            if res_inner.coefficients is not None:
                np.copyto(res_inner.coefficients, h)
            else:
                res_inner.coefficients = h.copy()
        else:
            res_inner.coefficients = d_r
    return Polynomial(x[0].curve, res_inner, 0, x[0].size)


# ---------------------------------------------------------------------------------------------------------------------------
# ratios.go
# ---------------------------------------------------------------------------------------------------------------------------
def _check_size(*pols) -> int:
    """checkSize (ratios.go:277-291): compares pols[i][j] for i, j < len(pols) only; an index the reference reads past the end of
    a list (where it panics) raises IopError"""
    m = len(pols)
    for i in range(m):
        for j in range(m):
            if j >= len(pols[i]):
                raise IopError("checkSize: index out of range [%d] with length %d" % (j, len(pols[i])))
    n = pols[0][0]._len()
    for i in range(m):
        for j in range(m):
            if pols[i][j]._len() != n:
                raise ErrInconsistentSize()
    return n


def _build_domain(n: int, domain: Domain, curve: str, device: int) -> Domain:
    """buildDomain (ratios.go:295-313)"""
    if n & (n - 1):
        raise ErrSizeNotPowerOfTwo()
    if domain is None:
        domain = _domain(curve, n, device)
    elif getattr(domain, "curve", curve) != curve:
        raise IopError("the domain is over the scalar field of %s, the polynomials over that of %s" % (domain.curve, curve))
    if domain.Cardinality != n:
        raise ErrInconsistentSizeDomain()
    if domain.device != device:
        raise IopError("the polynomials are on cuda:%d, the domain on cuda:%d" % (device, domain.device))
    return domain


def _put_in_expected_form(d_z, domain: Domain, form: Form, curve: str, device: int):
    """putInExpectedFormFromLagrangeRegular (ratios.go:248-273) on a device tensor"""
    steps = []
    if form.Basis == Canonical:
        steps = [("fft", True, DIF, False)] + ([("br",)] if form.Layout == Regular else [])
    elif form.Basis == LagrangeCoset:
        steps = [("fft", True, DIF, False), ("fft", False, DIT, True)] + ([("br",)] if form.Layout == BitReverse else [])
    elif form.Layout == BitReverse:
        steps = [("br",)]
    _run_steps(d_z, curve, domain, steps, device)


def _ratio_checks(lists):
    """the checks of a ratio builder that come before its domain, and the placement of its inputs (no device work)"""
    n = _check_size(*lists)
    curve = lists[0][0].curve
    for lst in lists:
        for p in lst:
            if p.curve != curve:
                raise IopError("the polynomials of one call must be over one curve")
    if n & (n - 1):
        raise ErrSizeNotPowerOfTwo()
    for lst in lists:
        if len(lst) > MAX_COLUMNS:
            raise IopError("%d polynomials per list (at most %d)" % (len(lst), MAX_COLUMNS))
        for p in lst:
            if p._len() > n:   # the reference would run an FFT over a slice longer than its domain
                raise ErrInconsistentSize()
    inners = [p._p for lst in lists for p in lst]
    return curve, n, _device_of(inners), inners


def _ratio_domain(curve, n, dev, domain):
    device = (domain.device if domain is not None else 0) if dev is None else dev
    return _build_domain(n, domain, curve, device), device


def _ratio_result(d_z, n, curve, dev, expectedForm) -> Polynomial:
    w = _params(curve).fr_words
    c = d_z if dev is not None else d_z.cpu().numpy().view(np.uint64).reshape(-1, w).copy()
    return Polynomial(curve, _Inner(c, expectedForm.Basis, expectedForm.Layout), 0, n)


def BuildRatioShuffledVectors(numerator, denominator, beta, expectedForm: Form, domain: Domain = None) -> Polynomial:
    """iop.BuildRatioShuffledVectors: Z(w^k) = prod_{i<k} prod_j (beta - P_j(w^i)) / (beta - Q_j(w^i)).  The inputs are put in
    Lagrange form in place first, as in the reference; `beta`: fr.Element limbs."""
    if len(numerator) != len(denominator):
        raise ErrNumberPolynomials()
    curve, n, dev, inners = _ratio_checks([list(numerator), list(denominator)])
    domain, device = _ratio_domain(curve, n, dev, domain)
    cp = _params(curve)
    b = _fr_encode([_fr_decode(np.asarray(beta, dtype=np.uint64), cp.r)[0]], cp.r)[0]
    torch = _torch()
    with torch.cuda.device(device):
        st = _Staged(inners, device, cp.fr_words)
        try:
            for p, q in zip(numerator, denominator):
                p.ToLagrange(domain)
                q.ToLagrange(domain)
            dp = _DevicePoly(curve, device, 1)
            d_z = dp.empty(n)
            dp.iop_ratio_shuffled([p._p.coefficients for p in numerator], [p.Layout == BitReverse for p in numerator],
                                  [q._p.coefficients for q in denominator], [q.Layout == BitReverse for q in denominator], n, b, d_z)
            _put_in_expected_form(d_z, domain, expectedForm, curve, device)
        finally:
            st.done()
        return _ratio_result(d_z, n, curve, dev, expectedForm)


def BuildRatioCopyConstraint(entries, permutation, beta, gamma, expectedForm: Form, domain: Domain = None) -> Polynomial:
    """iop.BuildRatioCopyConstraint: Z(w^k) = prod_{i<k} prod_j (P_j(w^i) + beta g^j w^i + gamma) / (P_j(w^i) + beta ID[sigma(jn+i)]
    + gamma), ID[s] = g^(s / n) w^(s mod n).  `permutation`: k n int64 entries, a host array or a device tensor; an entry outside
    [0, k n) is refused before the result is written."""
    entries = list(entries)
    curve, n, dev, inners = _ratio_checks([entries])
    cp = _params(curve)
    k = len(entries)
    if _is_device(permutation):
        torch = _torch()
        device = 0 if dev is None else dev
        if not permutation.is_cuda or permutation.device.index != device or permutation.dtype != torch.int64 or not permutation.is_contiguous():
            raise IopError("the permutation must be a contiguous torch.int64 tensor on cuda:%d" % device)
        if permutation.numel() != k * n:
            raise IopError("the permutation has %d entries, not k n = %d" % (permutation.numel(), k * n))
        sigma = permutation
    else:
        s = np.ascontiguousarray(permutation, dtype=np.int64).reshape(-1)
        if s.shape[0] != k * n:
            raise IopError("the permutation has %d entries, not k n = %d" % (s.shape[0], k * n))
        if s.size and (s.min() < 0 or s.max() >= k * n):
            raise IopError("the permutation has an entry outside [0, %d)" % (k * n))
        sigma = None
        s_host = s
    domain, device = _ratio_domain(curve, n, dev, domain)
    torch = _torch()
    b = _fr_encode([_fr_decode(np.asarray(beta, dtype=np.uint64), cp.r)[0]], cp.r)[0]
    g = _fr_encode([_fr_decode(np.asarray(gamma, dtype=np.uint64), cp.r)[0]], cp.r)[0]
    with torch.cuda.device(device):
        if sigma is None:
            sigma = torch.from_numpy(s_host.copy()).to(torch.device("cuda", device))
        st = _Staged(inners, device, cp.fr_words)
        try:
            for p in entries:
                p.ToLagrange(domain)
            dp = _DevicePoly(curve, device, 1)
            d_z = dp.empty(n)
            dp.iop_ratio_copy(domain, [p._p.coefficients for p in entries], [p.Layout == BitReverse for p in entries], sigma, b, g, d_z)
            _put_in_expected_form(d_z, domain, expectedForm, curve, device)
        finally:
            st.done()
        return _ratio_result(d_z, n, curve, dev, expectedForm)


# ---------------------------------------------------------------------------------------------------------------------------
# quotient.go
# ---------------------------------------------------------------------------------------------------------------------------
def _xn_minus_one_inverses(domains, r: int) -> list:
    """evaluateXnMinusOneDomainBigCoset (quotient.go:56-79): (g^s (w_big^s)^j - 1)^-1 for j < rho, zero -> zero"""
    s = domains[0].Cardinality
    ratio = domains[1].Cardinality // s
    g = _fr_decode(domains[1].FrMultiplicativeGen, r)[0]
    wb = _fr_decode(domains[1].Generator, r)[0]
    v, t, res = pow(g, s, r), pow(wb, s, r), []
    for _ in range(ratio):
        res.append((v - 1) % r)
        v = v * t % r
    return [pow(x, r - 2, r) if x else 0 for x in res]


def DivideByXMinusOne(a: Polynomial, domains) -> Polynomial:
    """iop.DivideByXMinusOne: the quotient of a (LagrangeCoset, on the coset of domains[1]) by X^s - 1, s = |domains[0]|, in
    Canonical Regular form with size = a.size"""
    if a.Basis != LagrangeCoset:
        raise ErrMustBeLagrangeCoset()
    cp = a._cp
    n, w = a._len(), cp.fr_words
    ratio = domains[1].Cardinality // domains[0].Cardinality
    if a.size <= 0 or n // a.size != ratio or ratio == 0:
        raise IopError("len / size = %s does not match the ratio %d of the domains" % (n // a.size if a.size > 0 else "?", ratio))
    if ratio > MAX_RHO:
        raise IopError("the ratio of the domains (%d) is over %d" % (ratio, MAX_RHO))
    if n > domains[1].Cardinality:
        raise ErrInconsistentSize()
    _check_rev(n)
    offset = _offset(a, n)
    inv = _fr_encode(_xn_minus_one_inverses(domains, cp.r), cp.r)
    dev = _device_of([a._p])
    device = domains[1].device if dev is None else dev
    torch = _torch()
    with torch.cuda.device(device):
        dp = _DevicePoly(a.curve, device, 1)
        d_a = _device_poly(a._p.coefficients, w, device)
        d_out = dp.empty(n)
        dp.iop_divide_by_xn_minus_one(d_a, n, offset, a.Layout != Regular, inv, d_out)
        res = Polynomial(a.curve, _Inner(d_out, LagrangeCoset, BitReverse), 0, a.size)
        res.ToCanonical(domains[1])
        if dev is None:
            res._p.coefficients = res._p.coefficients.cpu().numpy().view(np.uint64).reshape(-1, w).copy()
    return res
