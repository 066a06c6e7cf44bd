"""Kernel time of point (de)serialisation on device-resident data, with CUDA events: G1 decode and encode at 2^24 points for bn254
and bls12-381, G2 decode and encode at 2^22 points for bn254, bls12-381 and bls12-377, both wire kinds (Bytes, RawBytes).  Points
are [1 + i]G built on the device; the bytes to decode are their encoding.  For each step the rate is the bytes it moves (points
read and bytes written for encode, the reverse for decode) over the kernel time, against the H100's 3.35 TB/s: encode is bound by
memory bandwidth, decode of compressed points by the square root.  Prints the card name and power limit read in the same run,
then one JSON line per step.

  python tools/time_marshal.py [--repeat 5] [--g1-log 24] [--g2-log 22]"""
import argparse
import json
import os
import subprocess
import sys
from importlib import import_module

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
HBM_BYTES_PER_S = 3.35e12       # H100 SXM data sheet


def _card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 else "unknown"


def _events_ms(fn, repeat, torch):
    """median of `repeat` timings of fn() between two CUDA events on the current stream, after one warm-up call"""
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(repeat):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=5)
    ap.add_argument("--g1-log", type=int, default=24)
    ap.add_argument("--g2-log", type=int, default=22)
    a = ap.parse_args()
    import torch

    L = import_module("gnark-crypto_b200._native").lib()
    C = import_module("gnark-crypto_b200.curves")
    O = import_module("oracle.oracle")
    card = _card()
    print("card:", card, flush=True)
    st = torch.cuda.current_stream().cuda_stream
    groups = [("bn254_g1", a.g1_log), ("bls12381_g1", a.g1_log), ("bn254_g2", a.g2_log), ("bls12381_g2", a.g2_log),
              ("bls12377_g2", a.g2_log)]
    for name, logn in groups:
        g = C.GROUPS[name]
        n = 1 << logn
        words = 2 * g.words
        gen = O.GROUPS[name].encode_affine([O.GROUPS[name].gen])[0]
        pts = torch.empty(n * words, dtype=torch.int64, device="cuda")
        assert L.gmsm_generate_multiples_device(g.id, gen.ctypes.data, 1, n, pts.data_ptr(), st) == 0
        out = torch.empty(n * words, dtype=torch.int64, device="cuda")
        err = torch.empty(1, dtype=torch.int64, device="cuda")
        decode = L.gmsm_g2_decode_device if name.endswith("_g2") else L.gmsm_g1_decode_device
        for raw in (0, 1):
            size = (2 if raw else 1) * 8 * g.words
            enc = torch.empty(n * size, dtype=torch.uint8, device="cuda")
            moved = n * (8 * words + size)
            ms = _events_ms(lambda: L.gmsm_points_encode_device(g.id, pts.data_ptr(), n, raw, enc.data_ptr(), st), a.repeat, torch)
            dms = _events_ms(lambda: decode(g.id, enc.data_ptr(), n, raw, 1, out.data_ptr(), err.data_ptr(), st), a.repeat, torch)
            assert torch.equal(out, pts) and int(err.cpu()[0]) == -1, name
            for step, t in (("encode", ms), ("decode", dms)):
                gbs = moved / (t * 1e-3) / 1e9
                print(json.dumps({"group": name, "log_n": logn, "step": step, "raw": raw, "ms": round(t, 3), "bytes": moved,
                                  "GB_s": round(gbs, 1), "share_of_hbm": round(gbs * 1e9 / HBM_BYTES_PER_S, 3),
                                  "points_per_s": round(n / (t * 1e-3)), "card": card}), flush=True)
            del enc
        del pts, out
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
