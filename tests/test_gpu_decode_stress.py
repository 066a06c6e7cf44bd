"""The sm_90a G1 point decoder (k_g1_decode through gmsm_g1_decode_device and gmsm_g1_decode, csrc/decode.cu) at every
square-root depth, sign boundary, element boundary and flag pattern, and at production sizes (generators and the big-int
reference in tests/decode_stress.py; the CPU twin is tests/test_decode_stress_cpu.py):

A-E. the families of decode_stress.py for the seven pairing curves, one device call per stream on torch tensors, every row limb
     for limb and the first error; one device error word serves every call of a curve, so each call after a failing one must
     start from a clean word;
E.   a first error past index 2^24 (the (i << 8) | code key above 2^32), then the same error word on a clean stream;
F.   a block of 2^16 distinct encodings (the accepted points of A to C, an infinity, subgroup points) tiled to bn254 compressed
     at 2^26 + 3 (a 2 GiB input: byte offsets past 2^31), bw6-761 raw at 2^24 + 1 (3 GiB) and bls24-315 compressed at 2^24 + 5
     (40-byte elements) on a non-default stream; the bls24-315 stream also through the host entry gmsm_g1_decode."""
import time
from importlib import import_module

import numpy as np
import pytest

from tests import decode_stress as S

pytestmark = pytest.mark.gpu
NONE = (1 << 64) - 1


def _torch():
    return import_module("torch")


def _native():
    return import_module("gnark-crypto_b200._native")


def _dev_bytes(data: bytes):
    torch = _torch()
    return torch.from_numpy(np.frombuffer(data, dtype=np.uint8).copy()).cuda()


def _first(err):
    e = int(err.cpu().numpy().view(np.uint64)[0])
    return None if e == NONE else (e >> 8, e & 0xFF)


def decode_device(name, d_bytes, n, is_raw, check, d_out, d_err, stream):
    """gmsm_g1_decode_device on device tensors, enqueued on `stream` (a torch.cuda.Stream)"""
    rc = _native().lib().gmsm_g1_decode_device(S.GID[name], d_bytes.data_ptr(), n, int(is_raw), int(check), d_out.data_ptr(),
                                                d_err.data_ptr(), stream.cuda_stream)
    assert rc == 0, _native().last_error()


@pytest.mark.parametrize("name", S.CURVES)
def test_decode_families_device(name):
    """families A to E, one call per stream on a non-default stream; the device error word is shared by all the calls"""
    torch = _torch()
    c = S.curve(name)
    fams = S.families(name)
    st = torch.cuda.Stream()
    d_err = torch.zeros(1, dtype=torch.int64, device="cuda")
    times = {}
    for letter, streams in fams.items():
        for s in streams:
            s.expected()
        t0 = time.perf_counter()
        for s in streams:
            d_in = _dev_bytes(s.data())
            d_out = torch.full((s.n * c.words,), -1, dtype=torch.int64, device="cuda")
            st.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(st):
                decode_device(name, d_in, s.n, s.raw, s.check, d_out, d_err, st)
            st.synchronize()
            S.compare(s, d_out.cpu().numpy().view(np.uint64).reshape(s.n, c.words), _first(d_err))
        times[letter] = time.perf_counter() - t0
    print("%s device: %s" % (name, ", ".join("%s %.2f s" % kv for kv in times.items())))


def _tiled_input(block: np.ndarray, n: int):
    """n encodings on the device: the (B, size) uint8 block repeated, then its head"""
    torch = _torch()
    B, size = block.shape
    full = n // B * B
    blk = torch.from_numpy(np.ascontiguousarray(block).reshape(-1).copy()).cuda()
    d = torch.empty(n * size, dtype=torch.uint8, device="cuda")
    d[: full * size].view(n // B, B * size).copy_(blk.view(1, -1).expand(n // B, -1))
    d[full * size:] = blk[: (n - full) * size]
    return d


def _compare_tiled(title, got, want, labels, n):
    """got: (n * words) int64 device tensor or (n, words) uint64 array; want: the (B, words) block.  Compared in chunks of 64
    blocks with numpy; the message names the index and the block entry"""
    B, w = want.shape
    chunk = 64 * B
    for lo in range(0, n, chunk):
        hi = min(n, lo + chunk)
        g = got[lo * w: hi * w] if not isinstance(got, np.ndarray) else got[lo:hi]
        g = (g.cpu().numpy() if not isinstance(g, np.ndarray) else g).view(np.uint64).reshape(hi - lo, w)
        m = hi - lo
        exp = want[np.arange(m) % B] if m % B else None
        bad = (g != exp).any(axis=1) if exp is not None else (g.reshape(-1, B, w) != want[None]).any(axis=2).reshape(-1)
        if bad.any():
            i = lo + int(np.nonzero(bad)[0][0])
            raise AssertionError("%s: index %d (block entry %d, %s): %d rows differ in [%d, %d)\n got  %s\n want %s" % (
                title, i, i % B, labels[i % B], int(bad.sum()), lo, hi, g[i - lo].tolist(), want[i % B].tolist()))


def test_first_error_past_2_24_and_error_word_reuse():
    """E on the device: bn254 compressed, 2^24 + 1024 points, DEC_BAD_FLAGS at 2^24 + 3 and DEC_BAD_INFINITY at 2^24 + 700
    (the lower index with the higher code, keys above 2^32); then the same error word on the stream with both points restored
    must report none, and every row must match"""
    torch = _torch()
    name = "bn254"
    c = S.curve(name)
    B = 1024
    rows, pts = S.subgroup_rows(name, B, 17)
    block = np.frombuffer(b"".join(S.compress(c, *p) for p in pts), dtype=np.uint8).reshape(B, c.nb)
    n = (1 << 24) + B
    d_in = _tiled_input(block, n)
    d_out = torch.empty(n * c.words, dtype=torch.int64, device="cuda")
    d_err = torch.zeros(1, dtype=torch.int64, device="cuda")
    st = torch.cuda.Stream()
    i1, i2 = (1 << 24) + 3, (1 << 24) + 700
    saved = (d_in[i1 * c.nb:(i1 + 1) * c.nb].clone(), d_in[i2 * c.nb:(i2 + 1) * c.nb].clone())
    d_in[i1 * c.nb] = (int(block[i1 % B, 0]) & ~c.mask & 0xFF) | c.flag(0b00)               # uncompressed in a compressed stream
    d_in[i2 * c.nb:(i2 + 1) * c.nb] = _dev_bytes(bytes([c.inf]) + bytes(c.nb - 2) + b"\x01")
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        decode_device(name, d_in, n, False, True, d_out, d_err, st)
    st.synchronize()
    assert _first(d_err) == (i1, S.BAD_FLAGS), ("bn254 E past 2^24", _first(d_err))
    o = d_out.view(n, c.words)
    assert not o[i1].any() and not o[i2].any(), "bn254 E past 2^24: rejected rows are not zero"
    assert torch.equal(o[i1 - 1].cpu(), torch.from_numpy(rows[(i1 - 1) % B].view(np.int64))), "bn254 E past 2^24: row before"
    d_in[i1 * c.nb:(i1 + 1) * c.nb] = saved[0]
    d_in[i2 * c.nb:(i2 + 1) * c.nb] = saved[1]
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        decode_device(name, d_in, n, False, True, d_out, d_err, st)
    st.synchronize()
    assert _first(d_err) is None, ("bn254 E: the error word after a failing call", _first(d_err))
    _compare_tiled("bn254 E clean stream of 2^24 + 1024 after a failing call", d_out, rows, ["subgroup point"] * B, n)


@pytest.mark.parametrize("name,is_raw,n", [("bn254", False, (1 << 26) + 3), ("bw6761", True, (1 << 24) + 1),
                                          ("bls24315", False, (1 << 24) + 5)])
def test_production_size(name, is_raw, n):
    """F: a tiled block of 2^16 distinct encodings through gmsm_g1_decode_device on a non-default stream, the whole output against
    the tiled expectation; bls24-315 also through the host entry gmsm_g1_decode"""
    torch = _torch()
    c = S.curve(name)
    block, want, labels = S.production_block(name, is_raw)
    title = "%s F %s n=%d" % (name, "raw" if is_raw else "compressed", n)
    d_in = _tiled_input(block, n)
    d_out = torch.empty(n * c.words, dtype=torch.int64, device="cuda")
    d_err = torch.zeros(1, dtype=torch.int64, device="cuda")
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    t0 = time.perf_counter()
    with torch.cuda.stream(st):
        decode_device(name, d_in, n, is_raw, True, d_out, d_err, st)
    st.synchronize()
    dt = time.perf_counter() - t0
    assert _first(d_err) is None, (title, _first(d_err))
    del d_in
    _compare_tiled(title, d_out, want, labels, n)
    print("%s: device decode %.1f ms" % (title, 1e3 * dt))
    del d_out
    if name == "bls24315":
        host = np.tile(block.reshape(-1), n // block.shape[0] + 1)[: n * block.shape[1]]
        out = np.zeros((n, c.words), dtype=np.uint64)
        t0 = time.perf_counter()
        rc = _native().lib().gmsm_g1_decode(S.GID[name], host.ctypes.data, n, int(is_raw), 1, out.ctypes.data)
        assert rc == 0, _native().last_error()
        print("%s: host entry %.1f ms" % (title, 1e3 * (time.perf_counter() - t0)))
        _compare_tiled(title + " (host entry)", out, want, labels, n)
