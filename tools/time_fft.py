"""Times the device Fr FFT (Domain.fft_device: FFT DIF then FFTInverse DIT, the round trip gnark's provers use) for the
seven scalar fields at 2^20, and at 2^22 where the field's maxOrderRoot allows it, with CUDA events after a warm-up.  Prints
the card's name and power limit first, then one JSON line per (field, size).  Needs a GPU and a built library.

    python tools/time_fft.py [--reps 20] [--warmup 3]"""
import argparse
import importlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CURVES = [("bn254", 28), ("bls12381", 32), ("bls12377", 47), ("bls24315", 22), ("bls24317", 60), ("bw6633", 20), ("bw6761", 46)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import numpy as np
    import torch

    import gnark_crypto_b200  # noqa: F401

    fft = importlib.import_module("gnark-crypto_b200.fft")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"card": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}), flush=True)
    for curve, max_order in CURVES:
        for logn in (20, 22):
            if logn > max_order:
                continue
            n = 1 << logn
            d = fft.NewDomain(curve, n)
            rng = np.random.default_rng(logn)
            a = rng.integers(0, 2**62, size=(n, d.words), dtype=np.uint64)
            a[:, d.words - 1] = 0                       # < r: arbitrary Montgomery residues
            da = torch.from_numpy(a.view(np.int64)).cuda()
            orig = da.clone()
            for _ in range(args.warmup):
                d.fft_device(da, False, fft.DIF)
                d.fft_device(da, True, fft.DIT)
            torch.cuda.synchronize()
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(args.reps):
                d.fft_device(da, False, fft.DIF)
                d.fft_device(da, True, fft.DIT)
            t1.record()
            torch.cuda.synchronize()
            ms = t0.elapsed_time(t1) / args.reps
            assert torch.equal(da, orig), "round trip changed the vector"
            print(json.dumps({"curve": curve, "logn": logn, "fr_bytes": 8 * d.words, "fft_plus_inverse_ms": round(ms, 3)}), flush=True)
            d.close()
            del da, orig


if __name__ == "__main__":
    main()
