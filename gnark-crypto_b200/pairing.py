"""Pairings of bn254 and bls12-381 on the GPU: MillerLoop, FinalExponentiation, Pair and PairingCheck (ecc/bn254/pairing.go,
ecc/bls12-381/pairing.go).

P is n G1Affine and Q n G2Affine points in the reference's memory layout (Montgomery u64 limbs, infinity = zeroes), as host numpy
arrays or contiguous torch.int64 CUDA tensors (both of one kind).  A GT element is 12 Montgomery fp.Elements, E12{C0, C1} of
E6{B0, B1, B2} of E2{A0, A1}: 48 u64 for bn254, 72 for bls12-381.  Results are host numpy arrays for host inputs and CUDA tensors
for device inputs; device work is ordered on the current torch stream of the inputs' device.  The other pairing curves raise
ValueError."""
from __future__ import annotations

import ctypes

import numpy as np

from . import _native
from .kzg import _device_poly, _host_poly, _is_device, _stream
from .multiexp import _check

# curve -> (G1 id of the C ABI, u64 words of an fp.Element)
_CURVES = {"bn254": (0, 4), "bls12381": (2, 6), "bls12-381": (2, 6)}


def _curve(curve: str):
    if curve not in _CURVES:
        raise ValueError("pairing: bn254 and bls12-381 only (got %r)" % (curve,))
    return _CURVES[curve]


def gt_words(curve: str) -> int:
    return 12 * _curve(curve)[1]


def _count(a, words: int, what: str) -> int:
    """points in a host array or CUDA tensor of whole points (`words` u64 each)"""
    size = a.numel() if _is_device(a) else np.asarray(a).size
    if size % words:
        raise ValueError("a buffer of %s holds whole points (%d int64 each)" % (what, words))
    return size // words


def _pairs(curve: str, P, Q):
    cid, L = _curve(curve)
    if _is_device(P) != _is_device(Q):
        raise ValueError("P and Q must both be host arrays or both CUDA tensors")
    n, m = _count(P, 2 * L, "G1Affine"), _count(Q, 4 * L, "G2Affine")
    if n == 0 or n != m:
        raise ValueError("invalid inputs sizes")
    return cid, L, n


def _run_pairs(entry: str, curve: str, P, Q):
    import torch

    cid, L, n = _pairs(curve, P, Q)
    on_device = _is_device(P)
    dev = P.device.index if on_device else torch.cuda.current_device()
    dP, dQ = _device_poly(P, 2 * L, dev), _device_poly(Q, 4 * L, dev)
    lib = _native.lib()
    ws = torch.empty((lib.gmsm_pairing_workspace_bytes(cid, n) + 7) // 8, dtype=torch.int64, device=torch.device("cuda", dev))
    out = torch.empty(12 * L, dtype=torch.int64, device=torch.device("cuda", dev))
    with torch.cuda.device(dev):
        _check(getattr(lib, entry)(cid, ctypes.c_void_p(dP.data_ptr()), ctypes.c_void_p(dQ.data_ptr()), n,
                                   ctypes.c_void_p(out.data_ptr()), ctypes.c_void_p(ws.data_ptr()), ctypes.c_void_p(_stream(dev))))
    if on_device:
        return out
    return out.cpu().numpy().view(np.uint64)


def MillerLoop(curve: str, P, Q):
    """MillerLoop(P, Q): the product of the Miller functions of the pairs, limb-identical to the reference"""
    return _run_pairs("gmsm_pairing_miller_loop_device", curve, P, Q)


def Pair(curve: str, P, Q):
    """Pair(P, Q) = FinalExponentiation(MillerLoop(P, Q))"""
    return _run_pairs("gmsm_pair_device", curve, P, Q)


def FinalExponentiation(curve: str, z, *zs):
    """FinalExponentiation(z, zs...): the product of the arguments raised to the reference's exponent"""
    import torch

    cid, L = _curve(curve)
    W = 12 * L
    args = (z,) + zs
    if len({_is_device(a) for a in args}) != 1:
        raise ValueError("the GT elements must all be host arrays or all CUDA tensors")
    on_device = _is_device(z)
    dev = z.device.index if on_device else torch.cuda.current_device()
    if on_device:
        for a in args:
            if a.numel() != W:
                raise ValueError("a GT element of %s is %d int64" % (curve, W))
        dz = torch.cat([a.reshape(-1) for a in args]).to(torch.device("cuda", dev)) if len(args) > 1 else _device_poly(z, W, dev)
    else:
        h = np.concatenate([_host_poly(a, W) for a in args])
        if h.shape[0] != len(args):
            raise ValueError("a GT element of %s is %d u64" % (curve, W))
        dz = _device_poly(h, W, dev)
    out = torch.empty(W, dtype=torch.int64, device=torch.device("cuda", dev))
    with torch.cuda.device(dev):
        _check(_native.lib().gmsm_pairing_final_exp_device(cid, ctypes.c_void_p(dz.data_ptr()), len(args), ctypes.c_void_p(out.data_ptr()),
                                                           ctypes.c_void_p(_stream(dev))))
    if on_device:
        return out
    return out.cpu().numpy().view(np.uint64)


_FP = {0: 0x30644E72E131A029B85045B68181585D97816A916871CA8D3C208C16D87CFD47,
       2: 0x1A0111EA397FE69A4B1BA7B6434BACD764774B84F38512BF6730D2A0F6B0F6241EABFFFEB153FFFFB9FEFFFFFFFFAAAB}


def is_one(curve: str, e) -> bool:
    """e == 1 in GT: C0.B0.A0 is R mod p (Montgomery one), everything else zero"""
    cid, L = _curve(curve)
    h = _host_poly(e, 12 * L).reshape(-1)
    r = (1 << (64 * L)) % _FP[cid]
    one = np.zeros(12 * L, dtype=np.uint64)
    one[:L] = [(r >> (64 * i)) & (2**64 - 1) for i in range(L)]
    return bool(np.array_equal(h, one))


def PairingCheck(curve: str, P, Q) -> bool:
    """PairingCheck(P, Q): Pair(P, Q) == 1"""
    return is_one(curve, Pair(curve, P, Q))
