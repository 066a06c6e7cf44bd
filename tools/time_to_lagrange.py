"""Times kzg.ToLagrangeG1 on one GPU: gmsm_g1_to_lagrange_device on a device-resident SRS-like input ([1..n] G, from
gmsm_generate_multiples_device), output to a separate device buffer, CUDA events around each call after a warm-up.

Reported per (curve, n): the call time; the time per twiddle multiplication, over the (n/2) log2 n - (n - 1) twiddle
multiplications and n multiplications by 1/n of the transform; and the achieved share of the INT32 multiplier pipe, counted
as bench.py counts it for k_accumulate: Fp products x (2 N^2 + N) IMAD.WIDE (N 32-bit limbs) against 132 SMs x 32 IMAD.WIDE per
clock at the card's maximum SM clock.  The Fp products are the textbook count of the kernels in csrc/lagrange_kernels.cuh
(window width W, lag_w there): per window a conversion to Jacobian (4), W doublings (7 each), a conversion back (2) and, for a
non-zero digit, one extended-Jacobian addition (14); the table of 2^(W-1) multiples; the two additions of each butterfly.
Prints the card's name and power limit first, then one JSON line per case.  Needs a GPU and a built library; GMSM_LIB=<tag> times
a variant build (build.py's GMSM_BUILD_TAG with GMSM_NVCC_EXTRA=-DGMSM_LAG_W=w), whose window width is then given with --lag-w.

    python tools/time_to_lagrange.py [--reps 3] [--warmup 1] [--cases bn254:16,bw6761:16] [--lag-w w] [--big]"""
import argparse
import importlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CURVES = ["bn254", "bls12381", "bls12377", "bls24315", "bls24317", "bw6633", "bw6761"]
DEFAULT = [(c, 16) for c in CURVES] + [("bn254", 20), ("bls12381", 20), ("bw6761", 20)]
BIG = [("bn254", 22), ("bn254", 24)]
FR_BITS = {"bn254": 254, "bls12381": 255, "bls12377": 253, "bls24315": 253, "bls24317": 255, "bw6633": 315, "bw6761": 377}
H100_SMS = 132


def lag_w(curve):
    """the library's window width (lag_w in csrc/lagrange_kernels.cuh)"""
    return 5 if FR_BITS[curve] > 300 else 4


def fp_products(curve, n, w):
    """Fp products of one transform of n points with window width w (textbook count, see the module docstring)"""
    logn = n.bit_length() - 1
    nwin = FR_BITS[curve] // w + 1
    per_mul = (nwin - 1) * (4 + 7 * w + 2) + (nwin - 1) * (1 - 2.0 ** -w) * 14 + ((1 << (w - 1)) - 1) * 14
    twiddle_muls = (n // 2) * logn - (n - 1)
    return (twiddle_muls + n) * per_mul + (n // 2) * logn * 2 * 14, twiddle_muls + n, per_mul


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--cases", default="")
    ap.add_argument("--lag-w", type=int, default=0, help="window width of a GMSM_LIB variant (default: the library's)")
    ap.add_argument("--big", action="store_true", help="also bn254 at 2^22 and 2^24")
    args = ap.parse_args()
    import numpy as np
    import torch

    import gnark_crypto_b200  # noqa: F401
    from oracle import oracle as O

    native = importlib.import_module("gnark-crypto_b200._native")
    mx = importlib.import_module("gnark-crypto_b200.multiexp")
    L = native.lib()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True)
    smi = q.stdout.strip().splitlines()[0] if q.stdout.strip() else ""
    print(json.dumps({"card": torch.cuda.get_device_name(0), "nvidia_smi": smi, "lib": os.environ.get("GMSM_LIB", "")}), flush=True)
    try:
        sm_mhz = float(smi.split(",")[2])
    except (IndexError, ValueError):
        sm_mhz = None
    cases = [(c.split(":")[0], int(c.split(":")[1])) for c in args.cases.split(",") if c] or DEFAULT + (BIG if args.big else [])
    dev = torch.device("cuda", 0)
    for curve, logn in cases:
        g = curve + "_g1"
        cid = mx.CURVES[g]
        G = O.GROUPS[g]
        n = 1 << logn
        words = G.aff_words
        base = G.encode_affine([G.gen])[0]
        pts = torch.empty(n * words, dtype=torch.int64, device=dev)
        out = torch.empty_like(pts)
        work = torch.empty(int(L.gmsm_g1_to_lagrange_workspace_bytes(cid, n)) // 8, dtype=torch.int64, device=dev)
        st = torch.cuda.current_stream(dev).cuda_stream
        mx._check(L.gmsm_generate_multiples_device(cid, base.ctypes.data, 1, n, pts.data_ptr(), st))
        torch.cuda.synchronize()

        def call():
            mx._check(L.gmsm_g1_to_lagrange_device(cid, pts.data_ptr(), n, out.data_ptr(), work.data_ptr(), st))

        for _ in range(args.warmup):
            call()
        torch.cuda.synchronize()
        ms = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            call()
            e1.record()
            e1.synchronize()
            ms.append(e0.elapsed_time(e1))
        t = sorted(ms)[len(ms) // 2]
        w = args.lag_w or lag_w(curve)
        prods, muls, per_mul = fp_products(curve, n, w)
        limbs = words   # 32-bit limbs of one Fp element (2 x fp.Limbs) = u64 words of an affine point
        wide = prods * (2 * limbs * limbs + limbs)
        rec = {"curve": curve, "logn": logn, "n": n, "lag_w": w, "ms_median": round(t, 3), "ms_all": [round(x, 3) for x in ms],
               "scalar_muls": muls, "fp_products_per_mul": round(per_mul, 1), "ns_per_scalar_mul": round(t * 1e6 / muls, 2),
               "wide_mads_per_s": wide / (t * 1e-3)}
        if sm_mhz:
            rec["int_pipe_frac_at_max_clock"] = round(wide / (t * 1e-3) / (H100_SMS * 32 * sm_mhz * 1e6), 4)
        digest = np.frombuffer(out[:8 * words].cpu().numpy().tobytes(), dtype=np.uint64)
        rec["out_head_sum"] = int(digest.sum() & 0xFFFFFFFF)
        print(json.dumps(rec), flush=True)
        del pts, out, work
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
