"""Point (de)serialisation on the device (gmsm_g2_decode_device, gmsm_points_encode_device and the kzg.py layer on top), against
the big-int restatement of tests/marshal_ref.py (the CPU twin is tests/test_marshal_cpu.py):

  * every decoder family of marshal_ref.decode_cases for the five G2 groups, and the encoder families for all twelve groups;
  * a first error at index 2^24 + 5, and a clean call on the same error word after it;
  * production sizes built on the device (gmsm_generate_multiples_device): bn254 and bls12-381 G2 at 2^22 + 3 points, bn254 G1
    encode at 2^26 + 3.  Each is encoded and decoded back on the device and compared whole with the original; 4096 sampled
    indices (first and last included) are compared with the reference's encoding;
  * one contribution without leaving the device: G2 decode -> UpdateMonomialsG2 -> encode, against the big-int codec and
    mpcsetup_ref.update_monomials;
  * the slice helpers (mixed streams of both orders refused) and ProvingKey.WriteTo / WriteRawTo / UnsafeReadFrom;
  * buffers that are not 16-byte aligned refused with GMSM_EINVAL."""
import ctypes
import io
import random
from importlib import import_module

import numpy as np
import pytest

from tests import marshal_ref as R

pytestmark = pytest.mark.gpu


def _torch():
    return import_module("torch")


def _lib():
    return import_module("gnark-crypto_b200._native").lib()


def _stream():
    return _torch().cuda.current_stream().cuda_stream


def _err():
    return _torch().empty(1, dtype=_torch().int64, device="cuda")


def _first(err):
    e = int(err.cpu().numpy().view(np.uint64)[0])
    return None if e == (1 << 64) - 1 else (e >> 8, e & 0xFF)


def dev_decode(G, data, n, raw, check=True, err=None):
    """bytes (host bytes or a device uint8 tensor) -> (device rows (n * words int64), first error)"""
    torch = _torch()
    d = data if torch.is_tensor(data) else torch.frombuffer(bytearray(data or b"\0"), dtype=torch.uint8).cuda()
    out = torch.empty(max(n, 1) * G.words, dtype=torch.int64, device="cuda")
    err = _err() if err is None else err
    fn = _lib().gmsm_g1_decode_device if G.name.endswith("_g1") else _lib().gmsm_g2_decode_device
    assert fn(G.id, d.data_ptr(), n, int(raw), int(check), out.data_ptr(), err.data_ptr(), _stream()) == 0
    return out, _first(err)


def dev_encode(G, rows, raw):
    """device rows (int64 tensor) -> device uint8 tensor of the n encodings"""
    torch = _torch()
    n = rows.numel() // G.words
    size = (2 if raw else 1) * G.comp_bytes()
    out = torch.empty(max(n * size, 4), dtype=torch.uint8, device="cuda")
    assert _lib().gmsm_points_encode_device(G.id, rows.data_ptr(), n, int(raw), out.data_ptr(), _stream()) == 0
    return out[:n * size]


def _to_dev(rows):
    return _torch().from_numpy(np.ascontiguousarray(rows, dtype=np.uint64).view(np.int64).reshape(-1).copy()).cuda()


def _host(t, w):
    return t.cpu().numpy().view(np.uint64).reshape(-1, w)


@pytest.mark.parametrize("name", R.G2_GROUPS)
def test_g2_decode_families_device(name):
    """every decoder family on the device: rows limb for limb and the first error, with one error word for all calls"""
    G = R.group(name)
    err = _err()
    for c in R.decode_cases(G):
        rows, first = dev_decode(G, c.data, c.n, c.raw, c.check, err)
        want, wfirst = G.decode_stream(c.data, c.n, c.raw, c.check)
        assert first == wfirst, (name, c.title, first, wfirst)
        assert np.array_equal(_host(rows, G.words)[:c.n], want), (name, c.title)


def test_bls12377_square_root_depths_device():
    G = R.group("bls12377_g2")
    pts = R.depth_points(G, random.Random(11), per=4)
    allp = [q for d in pts for p in pts[d] for q in (p, (p[0], G.neg(p[1])))]
    rows, first = dev_decode(G, G.encode(allp, False), len(allp), False)
    assert first is None and np.array_equal(_host(rows, G.words), np.stack([G.row(p) for p in allp]))


@pytest.mark.parametrize("name", R.ALL_GROUPS)
def test_encode_families_device(name):
    """the encoder families on the device over 3 blocks and a partial one, both kinds, and the round trip through the decoder"""
    G = R.group(name)
    base = R.encode_points(G, random.Random(17))
    pts = [base[i % len(base)] for i in range(3 * 128 + 77)]
    rows = np.stack([G.row(p) for p in pts])
    d = _to_dev(rows)
    for raw in (False, True):
        got = dev_encode(G, d, raw).cpu().numpy().tobytes()
        assert got == R.encode_ref(G, pts, raw), (name, raw)
    cur = [p for p in G.random_points(50, random.Random(2))] + [None]
    rows = np.stack([G.row(p) for p in cur])
    for raw in (False, True):
        b = dev_encode(G, _to_dev(rows), raw)
        back, first = dev_decode(G, b, len(cur), raw)
        assert first is None and np.array_equal(_host(back, G.words), rows), (name, raw)


def test_first_error_past_2_24():
    """a compressed bn254 G2 stream of infinity points with one bad flag at index 2^24 + 5 and a bad infinity past it: the
    first-error word holds the index in full; a clean call on the same word resets it"""
    torch = _torch()
    G = R.group("bn254_g2")
    n = (1 << 24) + 9
    size = G.comp_bytes()
    data = torch.zeros(n * size, dtype=torch.uint8, device="cuda")
    data[::size] = G.flags["inf"]
    bad = (1 << 24) + 5
    data[bad * size] = G.flags["unc"]                 # an uncompressed flag in a compressed stream
    data[(bad + 2) * size + 7] = 1                    # a later, lower code
    err = _err()
    _, first = dev_decode(G, data, n, False, err=err)
    assert first == (bad, R.BAD_FLAGS)
    _, first = dev_decode(G, data[:bad * size], bad, False, err=err)
    assert first is None


def _production(name, n, raw, seed):
    """points [1 + i]G built on the device -> encode -> decode -> compare whole, and 4096 sampled indices against the reference"""
    torch = _torch()
    O = import_module("oracle.oracle")
    G = R.group(name)
    OG = O.GROUPS[name]
    gen = OG.encode_affine([OG.gen])[0]
    pts = torch.empty(n * G.words, dtype=torch.int64, device="cuda")
    assert _lib().gmsm_generate_multiples_device(G.id, gen.ctypes.data, 1, n, pts.data_ptr(), _stream()) == 0
    enc = dev_encode(G, pts, raw)
    back, first = dev_decode(G, enc, n, raw)
    assert first is None
    assert torch.equal(back, pts), name
    del back
    rng = random.Random(seed)
    idx = sorted({0, n - 1} | {rng.randrange(n) for _ in range(4094)})
    it = torch.tensor(idx, dtype=torch.int64, device="cuda")
    rows = _host(pts.view(n, G.words)[it], G.words)
    size = (2 if raw else 1) * G.comp_bytes()
    encs = enc.view(n, size)[it].cpu().numpy()
    sample = [G.unrow(r) for r in rows]
    for k, (i, p) in enumerate(zip(idx, sample)):
        assert encs[k].tobytes() == R.encode_ref(G, [p], raw), (name, i)
    for k in range(0, len(idx), 64):                  # the reference's decoder on a subset (a Python square root each)
        assert np.array_equal(G.decode_stream(encs[k].tobytes(), 1, raw)[0][0], rows[k]), (name, idx[k])


@pytest.mark.parametrize("name", ["bn254_g2", "bls12381_g2"])
def test_g2_production_size(name):
    _production(name, (1 << 22) + 3, False, 31)


def test_bn254_g1_encode_2_26():
    _production("bn254_g1", (1 << 26) + 3, False, 37)


@pytest.mark.parametrize("curve", ["bn254", "bls12381", "bls12377"])
def test_contribution_on_device(curve):
    """G2 decode -> UpdateMonomialsG2 -> encode without leaving the device equals the host path: the big-int decoder,
    mpcsetup_ref.update_monomials on the oracle's points (big-int scalar multiplications) and the big-int encoder"""
    torch = _torch()
    K = R.kzg()
    mpc = import_module("gnark-crypto_b200.mpcsetup")
    C = import_module("gnark-crypto_b200.curves")
    MR = import_module("tests.mpcsetup_ref")
    G = R.group(curve + "_g2")
    OG = MR.group(curve + "_g2")
    rng = random.Random(41)
    pts = G.random_points(120, rng) + [None]
    data = G.encode(pts, False)
    rv = rng.randrange(1, C.CURVE_PARAMS[curve].r)
    r = C._fr_encode([rv], C.CURVE_PARAMS[curve].r)[0]
    d = K.decode_g2_points(curve, torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda(), len(pts))
    mpc.UpdateMonomialsG2(curve, d.view(-1), r)
    got = K.encode_g2_points(curve, d.view(-1), raw=False).cpu().numpy().tobytes()
    rows, first = G.decode_stream(data, len(pts), False)
    assert first is None
    want = OG.encode_affine(MR.update_monomials(OG, OG.decode_affine(rows), rv))
    assert got == G.encode([G.unrow(x) for x in want], False)


@pytest.mark.parametrize("curve", ["bn254", "bls12381", "bw6761"])
def test_slices_and_proving_key(curve):
    """write_points / read_points (the Encoder / Decoder slice framing), a mixed stream refused, and ProvingKey.WriteTo /
    WriteRawTo / UnsafeReadFrom round trips"""
    K = R.kzg()
    mx = import_module("gnark-crypto_b200.multiexp")
    G1 = R.group(curve + "_g1")
    pts = G1.random_points(200, random.Random(5)) + [None]
    rows = np.stack([G1.row(p) for p in pts])
    pk = K.ProvingKey(curve, rows)
    try:
        for raw, write in ((False, pk.WriteTo), (True, pk.WriteRawTo)):
            buf = io.BytesIO()
            nb = write(buf)
            assert buf.getvalue() == len(pts).to_bytes(4, "big") + R.encode_ref(G1, pts, raw) and nb == len(buf.getvalue())
            buf.seek(0)
            pk2, nr = K.ProvingKey.UnsafeReadFrom(curve, buf)
            assert nr == nb and np.array_equal(pk2.G1, rows)
            pk2.close()
    finally:
        pk.close()
    G2 = R.group(curve + "_g2")
    p2 = G2.random_points(20, random.Random(6)) + [None]
    r2 = np.stack([G2.row(p) for p in p2])
    for raw in (False, True):
        buf = io.BytesIO()
        K.write_points(buf, curve + "_g2", r2, raw)
        buf.seek(0)
        assert np.array_equal(K.read_points(buf, curve + "_g2"), r2)
    # mixed: a raw point after a compressed one
    mixed = len(pts[:3]).to_bytes(4, "big") + G1.encode(pts[:2], False) + G1.encode(pts[2:3], True)
    with pytest.raises(mx.MultiExpError, match="point 2: invalid point encoding"):
        K.read_points(io.BytesIO(mixed), curve + "_g1")
    # mixed the other way: compressed points after a raw one (a stream shorter than three raw strides)
    mixed = len(pts[:3]).to_bytes(4, "big") + G1.encode(pts[:1], True) + G1.encode(pts[1:3], False)
    with pytest.raises(mx.MultiExpError, match="point 1: invalid point encoding"):
        K.read_points(io.BytesIO(mixed), curve + "_g1")
    # an empty slice read onto a device is an empty device tensor
    empty = K.read_points(io.BytesIO(bytes(4)), curve + "_g2", device=0)
    assert _torch().is_tensor(empty) and empty.is_cuda and tuple(empty.shape) == (0, G2.words)


def test_misaligned_buffers_refused():
    """points that are 8-byte but not 16-byte aligned (the kernels load and store points in 16-byte granules) are refused with
    GMSM_EINVAL before any launch, through the C entries and through kzg; the context stays usable"""
    torch = _torch()
    K = R.kzg()
    mx = import_module("gnark-crypto_b200.multiexp")
    G = R.group("bn254_g2")
    pts = G.random_points(8, random.Random(9))
    rows = np.stack([G.row(p) for p in pts])
    flat = torch.zeros(rows.size + 1, dtype=torch.int64, device="cuda")
    flat[1:] = _to_dev(rows)
    shifted = flat[1:]                                 # 8 bytes past a 256-byte aligned allocation
    assert shifted.data_ptr() % 16 == 8
    out = torch.empty(len(pts) * G.comp_bytes(), dtype=torch.uint8, device="cuda")
    L = _lib()
    assert L.gmsm_points_encode_device(G.id, shifted.data_ptr(), len(pts), 0, out.data_ptr(), _stream()) == 1
    with pytest.raises(mx.MultiExpError, match="16-byte"):
        K.encode_g2_points("bn254", shifted)
    enc = dev_encode(G, _to_dev(rows), False)
    err = _err()
    assert L.gmsm_g2_decode_device(G.id, enc.data_ptr(), len(pts), 0, 1, shifted.data_ptr(), err.data_ptr(), _stream()) == 1
    torch.cuda.synchronize()
    assert enc.cpu().numpy().tobytes() == G.encode(pts, False)


def test_host_entries_and_refusals():
    """the host entries agree with the device ones; unknown and unsupported ids are GMSM_EINVAL"""
    K = R.kzg()
    mx = import_module("gnark-crypto_b200.multiexp")
    G = R.group("bls12377_g2")
    pts = G.random_points(10, random.Random(8)) + [None]
    rows = np.stack([G.row(p) for p in pts])
    for raw in (False, True):
        b = K.encode_g2_points("bls12377", rows, raw)
        assert b == G.encode(pts, raw)
        assert np.array_equal(K.decode_g2_points("bls12377", b, len(pts), raw), rows)
    bad = bytearray(G.encode(pts, False))
    bad[3 * G.comp_bytes()] = 0
    with pytest.raises(mx.MultiExpError, match="point 3: invalid point encoding"):
        K.decode_g2_points("bls12377", bytes(bad), len(pts))
    L = _lib()
    buf = np.zeros(4096, dtype=np.uint8)
    out = np.zeros(64, dtype=np.uint64)
    for gid in (0, 2, 6, 9, 13, -1):              # G1 groups, secp256k1, bls24-315 G1, unknown
        assert L.gmsm_g2_decode(gid, buf.ctypes.data, 1, 0, 1, out.ctypes.data) == 1
    for gid in (6, 13, -1):
        assert L.gmsm_points_encode(gid, out.ctypes.data, 1, 0, buf.ctypes.data) == 1
