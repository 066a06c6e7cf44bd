"""Times MillerLoop, FinalExponentiation and Pair on the GPU for bn254 and bls12-381 at n in {1, 2, 64, 2^10, 2^14, 2^16}: one JSON
line per (curve, entry, n) with the median of CUDA-event timings, and the card's name and power limit read in the same run.
First, one line per curve with the device memory the driver reserves for the kernels' per-thread stacks (local memory) at their
first launch: the drop of free device memory over a one-pair Pair, less what the torch allocator took.
`python tools/time_pairing.py [--reps R] [--out FILE]`."""
import argparse
import ctypes
import importlib
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sizes", default="1,2,64,1024,16384,65536")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch

    import gnark_crypto_b200  # noqa: F401
    from tests import pairing_cases as PC

    nat = importlib.import_module("gnark-crypto_b200._native")
    L = nat.lib()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    card, power = [s.strip() for s in smi.splitlines()[0].split(",")] if smi else ("unknown", "unknown")
    lines = []
    torch.empty(1, device="cuda")
    torch.cuda.synchronize()
    for curve, cid in (("bn254", 0), ("bls12381", 2)):
        P, Q = PC.random_pairs(curve, 1, seed=6)
        pa, qa = PC.encode_pairs(curve, P, Q)
        dP, dQ = torch.from_numpy(pa.view(np.int64).copy()).cuda(), torch.from_numpy(qa.view(np.int64).copy()).cuda()
        ws = torch.empty((L.gmsm_pairing_workspace_bytes(cid, 1) + 7) // 8, dtype=torch.int64, device="cuda")
        out = torch.empty(128, dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        free0, res0 = torch.cuda.mem_get_info()[0], torch.cuda.memory_reserved()
        v = lambda t: ctypes.c_void_p(t.data_ptr())
        assert L.gmsm_pair_device(cid, v(dP), v(dQ), 1, v(out), v(ws), None) == 0, nat.last_error()
        torch.cuda.synchronize()
        free1, res1 = torch.cuda.mem_get_info()[0], torch.cuda.memory_reserved()
        rec = {"curve": curve, "entry": "local_memory_reserved_at_first_launch", "MiB": ((free0 - free1) - (res1 - res0)) / 2**20,
               "card": card, "power_limit": power}
        print(json.dumps(rec), flush=True)
        lines.append(rec)
    for curve, cid in (("bn254", 0), ("bls12381", 2)):
        P, Q = PC.random_pairs(curve, 64, seed=5)
        pa, qa = PC.encode_pairs(curve, P, Q)
        for n in [int(s) for s in a.sizes.split(",")]:
            reps = max(1, n // 64)
            dP = torch.from_numpy(np.tile(pa, (reps, 1))[:n].view(np.int64).copy()).cuda()
            dQ = torch.from_numpy(np.tile(qa, (reps, 1))[:n].view(np.int64).copy()).cuda()
            ws = torch.empty((L.gmsm_pairing_workspace_bytes(cid, n) + 7) // 8, dtype=torch.int64, device="cuda")
            out = torch.empty(128, dtype=torch.int64, device="cuda")
            st = torch.cuda.current_stream().cuda_stream
            v = lambda t: ctypes.c_void_p(t.data_ptr())
            calls = {
                "MillerLoop": lambda: L.gmsm_pairing_miller_loop_device(cid, v(dP), v(dQ), n, v(out), v(ws), ctypes.c_void_p(st)),
                "FinalExponentiation": lambda: L.gmsm_pairing_final_exp_device(cid, v(ws), 1, v(out), ctypes.c_void_p(st)),
                "Pair": lambda: L.gmsm_pair_device(cid, v(dP), v(dQ), n, v(out), v(ws), ctypes.c_void_p(st)),
            }
            for entry, fn in calls.items():
                if entry == "FinalExponentiation" and n != 1:
                    continue
                assert fn() == 0, nat.last_error()       # warm-up
                torch.cuda.synchronize()
                ts = []
                for _ in range(a.reps):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    assert fn() == 0, nat.last_error()
                    e1.record()
                    e1.synchronize()
                    ts.append(e0.elapsed_time(e1))
                rec = {"curve": curve, "entry": entry, "n": n, "ms_median": float(np.median(ts)), "ms_min": float(min(ts)),
                       "reps": a.reps, "card": card, "power_limit": power}
                print(json.dumps(rec), flush=True)
                lines.append(rec)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write("".join(json.dumps(r) + "\n" for r in lines))


if __name__ == "__main__":
    main()
