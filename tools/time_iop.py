"""Kernel time of each new iop step on device-resident inputs, with CUDA events: the copy-constraint ratio (k = 3, with its sigma
check and prefix product), the shuffled-vectors ratio (two polynomials per list), Evaluate of the PLONK gate ql a + qr b + qm a b +
qo c + qk, the Lagrange evaluation and the elementwise step of DivideByXMinusOne.  bn254 and bls12-381 at 2^20 and 2^22 by default,
the copy constraint also at 2^24.  The copy-constraint window includes its sigma check, whose flag read back is a host
synchronisation; the workspace is allocated once, before the window.  Inputs are already in Lagrange Regular form, so no FFT is timed.  For each step the rate is the
bytes it must move (columns, sigma, output) over the kernel time, against the H100's 3.35 TB/s.  Prints the card name and power
limit read in the same run, then one JSON line per step.

  python tools/time_iop.py [--repeat 5] [--curves bn254,bls12381] [--logs 20,22] [--copy-logs 24]"""
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


def _report(curve, logn, step, ms, nbytes, card):
    gbs = nbytes / (ms * 1e-3) / 1e9
    print(json.dumps({"curve": curve, "log_n": logn, "step": step, "ms": round(ms, 3), "bytes": nbytes, "GB_s": round(gbs, 1),
                      "share_of_hbm": round(gbs * 1e9 / HBM_BYTES_PER_S, 3), "card": card}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=5)
    ap.add_argument("--curves", default="bn254,bls12381")
    ap.add_argument("--logs", default="20,22")
    ap.add_argument("--copy-logs", default="24")
    a = ap.parse_args()
    import torch

    iop = import_module("gnark-crypto_b200.iop")
    kzg = import_module("gnark-crypto_b200.kzg")
    fft = import_module("gnark-crypto_b200.fft")
    card = _card()
    print("card:", card, flush=True)
    logs = [int(x) for x in a.logs.split(",") if x]
    copy_logs = [int(x) for x in a.copy_logs.split(",") if x]
    for curve in a.curves.split(","):
        cp = kzg.CURVE_PARAMS[curve]
        w, fb = cp.fr_words, cp.fr_bytes
        for logn in sorted(set(logs + copy_logs)):
            n = 1 << logn
            g = torch.Generator(device="cuda").manual_seed(logn)

            def rand():
                # random limbs reduced below r by clearing the top bits: values need not be uniform here
                t = torch.randint(-(1 << 62), 1 << 62, (n, w), dtype=torch.int64, device="cuda", generator=g)
                t[:, w - 1] &= (1 << (cp.r.bit_length() - 64 * (w - 1) - 2)) - 1
                return t.reshape(-1)

            d = fft.Domain(curve, n)
            dp = kzg._DevicePoly(curve, 0, 1)
            beta, gamma = curves_enc(curve, 5), curves_enc(curve, 7)
            cols = [rand() for _ in range(3)]
            sigma = torch.randperm(3 * n, device="cuda", generator=g)
            z = dp.empty(n)
            ms = _events_ms(lambda: dp.iop_ratio_copy(d, cols, [False] * 3, sigma, beta, gamma, z), a.repeat, torch)
            _report(curve, logn, "ratio_copy_k3", ms, 3 * n * fb + 2 * 3 * n * 8 + n * fb, card)   # sigma is read twice: check, ratio
            if logn in logs:
                ms = _events_ms(lambda: dp.iop_ratio_shuffled(cols[:2], [False, False], [cols[2], cols[0]], [False, False], n, beta, z),
                                a.repeat, torch)
                _report(curve, logn, "ratio_shuffled_2", ms, 4 * n * fb + n * fb, card)
                prog = iop.trace(lambda i, ql, qr, qm, qo, qk, xa, xb, xc: ql * xa + qr * xb + qm * xa * xb + qo * xc + qk, 8, cp.r)
                ins = [rand() for _ in range(5)] + cols
                consts = curves_enc(curve, *prog.consts).reshape(-1, w)
                ms = _events_ms(lambda: dp.iop_evaluate(np.array(prog.code, dtype=np.uint32), prog.out, consts, ins, [0] * 8,
                                                        [False] * 8, n, True, z), a.repeat, torch)
                _report(curve, logn, "evaluate_gate", ms, 8 * n * fb + n * fb, card)
                one = dp.empty(1)
                x = curves_enc(curve, 123456789)
                ms = _events_ms(lambda: dp.iop_lagrange_eval(d, cols[0], False, x, one), a.repeat, torch)
                _report(curve, logn, "lagrange_eval", ms, n * fb, card)
                inv = curves_enc(curve, *range(2, 6)).reshape(-1, w)
                ms = _events_ms(lambda: dp.iop_divide_by_xn_minus_one(cols[0], n, 0, True, inv, z), a.repeat, torch)
                _report(curve, logn, "divide_xn_minus_one", ms, 2 * n * fb, card)
            del cols, sigma, z
            d.close()
            torch.cuda.empty_cache()


def curves_enc(curve, *vals):
    kzg = import_module("gnark-crypto_b200.kzg")
    c = import_module("gnark-crypto_b200.curves")
    out = c._fr_encode(list(vals), kzg.CURVE_PARAMS[curve].r)
    return out[0] if len(vals) == 1 else out


if __name__ == "__main__":
    main()
