"""Times kzg.Open and kzg.BatchOpenSinglePoint (k polynomials) on one GPU, split into their device steps, with CUDA events after
a warm-up: the upload of numpy coefficients, the Fr scan (gmsm_fr_poly_div_x_minus_a_device: f(a) and the quotient), the
evaluation-only scans and the gamma-fold of the batch, and the MultiExp of the quotient; plus the whole call with numpy and with
device-tensor (torch) polynomials.  The scan's algorithmic traffic is 3 n fr.Bytes (the heads pass reads f, the write pass reads
f and writes h); its rate is printed against the H100 SXM data-sheet HBM3 bandwidth of 3.35 TB/s.  The bases are [1..n] G.
Prints the card's name and power limit first, then one JSON line per (curve, n).  Needs a GPU and a built library.

    python tools/time_kzg_open.py [--reps 5] [--warmup 2] [--k 8] [--host-ref]

--host-ref also times the host Fr loops that Open used before (decode, eval, divide, encode) once, at 2^20."""
import argparse
import hashlib
import importlib
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CASES = [("bn254", 20), ("bn254", 22), ("bn254", 24), ("bls12381", 20), ("bls12381", 22), ("bls12381", 24), ("bw6761", 20)]
HBM_TBS = 3.35


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--k", type=int, default=8)
    ap.add_argument("--host-ref", action="store_true")
    args = ap.parse_args()
    import numpy as np
    import torch

    import gnark_crypto_b200  # noqa: F401

    kzg = importlib.import_module("gnark-crypto_b200.kzg")
    curves = importlib.import_module("gnark-crypto_b200.curves")
    mx = importlib.import_module("gnark-crypto_b200.multiexp")
    gens = json.load(open(os.path.join(ROOT, "gnark-crypto_b200", "generators.json")))
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"card": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}), flush=True)
    st = torch.cuda.current_stream().cuda_stream

    def timed(fn):
        """mean ms of fn over the repetitions, CUDA events on the current stream"""
        for _ in range(args.warmup):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.reps

    def wall(fn):
        """mean ms of a call that ends in a device synchronise (the proof comes back to the host)"""
        for _ in range(args.warmup):
            fn()
        t0 = time.perf_counter()
        for _ in range(args.reps):
            fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / args.reps

    for curve, logn in CASES:
        n = 1 << logn
        cp = kzg.CURVE_PARAMS[curve]
        w, S = cp.fr_words, cp.fr_bytes
        g = curve + "_g1"
        eng = mx.Engine(g, 1 << 10)
        pts = eng.generate_multiples(np.array([int(x, 16) for x in gens[g]], dtype=np.uint64), 1, n).cpu().numpy().view(np.uint64).copy()
        eng.close()
        pk = kzg.ProvingKey(curve, pts)
        del pts
        rng = np.random.default_rng(logn)
        p = rng.integers(0, 2**62, size=(n, w), dtype=np.uint64)
        p[:, w - 1] = 0                                     # < r: arbitrary Montgomery residues
        a = p[12345].copy()
        d_p = kzg._device_poly(p, w, 0)
        dp = kzg._DevicePoly(curve, 0, n)
        d_h, d_fa = dp.empty(n - 1), dp.empty(1)
        d_fold = dp.empty(n)
        d_claimed = dp.empty(args.k)
        polys_t = [d_p] * args.k
        gamma = curves._reduced(p[777], cp.r)
        res = {"curve": curve, "logn": logn, "fr_bytes": S, "k": args.k, "reps": args.reps}
        res["upload_ms"] = timed(lambda: kzg._device_poly(p, w, 0))
        res["scan_ms"] = timed(lambda: dp.div(d_p, n, a, d_h, d_fa))
        res["eval_scan_ms"] = timed(lambda: dp.div(d_p, n, a, None, d_claimed[:w]))
        res["fold_ms"] = timed(lambda: dp.fold(polys_t, [n] * args.k, gamma, d_fold, n))
        res["msm_ms"] = timed(lambda: pk._bases.MultiExpDevice(d_h, n - 1, stream=st))
        res["scan_TBps"] = 3 * n * S / (res["scan_ms"] * 1e-3) / 1e12
        res["scan_share_of_hbm_peak"] = res["scan_TBps"] / HBM_TBS
        res["eval_scan_TBps"] = n * S / (res["eval_scan_ms"] * 1e-3) / 1e12
        res["fold_TBps"] = (args.k + 1) * n * S / (res["fold_ms"] * 1e-3) / 1e12
        digest = kzg.Commit(d_p, pk)
        digests = [digest] * args.k
        res["open_numpy_ms"] = wall(lambda: kzg.Open(p, a, pk))
        res["open_tensor_ms"] = wall(lambda: kzg.Open(d_p, a, pk))
        res["batch_open_numpy_ms"] = wall(lambda: kzg.BatchOpenSinglePoint([p] * args.k, digests, a, hashlib.sha256, pk))
        res["batch_open_tensor_ms"] = wall(lambda: kzg.BatchOpenSinglePoint(polys_t, digests, a, hashlib.sha256, pk))
        if args.host_ref and logn == 20:
            t0 = time.perf_counter()
            coeffs = curves._fr_decode(p, cp.r)
            av = curves._fr_decode(a, cp.r)[0]
            fa = kzg._eval(coeffs, av, cp.r)
            h = kzg._divide_by_x_minus_a(coeffs, fa, av, cp.r)
            curves._fr_encode(h, cp.r)
            res["host_fr_loops_ms"] = (time.perf_counter() - t0) * 1e3
        print(json.dumps({k: (round(v, 4) if isinstance(v, float) else v) for k, v in res.items()}), flush=True)
        pk.close()
        del d_p, d_h, d_fa, d_fold, d_claimed, polys_t, dp, p
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
