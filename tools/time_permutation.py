"""Wall time of permutation.Prove on device-resident inputs (bn254 and bls12-381 at 2^20 and 2^22 by default), and the same work broken
into its parts, each timed alone with CUDA events on vectors of the same length:
  * ffts: the seven transforms of Prove (FFTInverse DIF + BitReverse of t1 and t2, FFTInverse DIT of Z, FFT DIF on the coset of
    cz, ct1 and ct2, FFTInverse DIT on the coset of the numerator);
  * multiexps: the six MultiExps (Commit of t1, t2, Z and q on n scalars, the quotients of BatchOpenSinglePoint and Open on n - 1);
  * accumulate / numerator: the two new entry points, with their rate as the bytes the step must move (accumulate: read t1 and t2,
    write z; numerator: read lt1, lt2 and lz, write the numerator) over the kernel time, against the H100's 3.35 TB/s.
What Prove adds to the parts is the transcript, the copies of the digests and claimed values, the openings' Fr scans and the
allocations.  Prints the card name and power limit read in the same run, then one JSON line per workload.

  python tools/time_permutation.py [--repeat 5] [--curves bn254,bls12381] [--logs 20,22]"""
import argparse
import json
import os
import subprocess
import sys
import time
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


def _wall_ms(fn, repeat, torch):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(repeat):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=5)
    ap.add_argument("--curves", default="bn254,bls12381")
    ap.add_argument("--logs", default="20,22")
    a = ap.parse_args()
    import torch

    kzg = import_module("gnark-crypto_b200.kzg")
    perm = import_module("gnark-crypto_b200.permutation")
    fft = import_module("gnark-crypto_b200.fft")
    curves = import_module("gnark-crypto_b200.curves")
    from oracle import oracle as O

    print("card:", _card(), flush=True)
    logs = [int(x) for x in a.logs.split(",")]
    for c in a.curves.split(","):
        cp = kzg.CURVE_PARAMS[c]
        r, w, fb = cp.r, cp.fr_words, cp.fr_bytes
        G = O.GROUPS[c + "_g1"]
        gen = G.encode_affine([G.gen])[0]
        pk = kzg.ProvingKey(c, kzg.new_srs_g1(c, 1 << max(logs), 0xC0FFEE % r, gen, r, G.encode_scalars))
        gen_t = torch.Generator(device="cuda").manual_seed(1)
        for logn in logs:
            n = 1 << logn

            def rand():         # reduced limbs: the top limb below 2^61 keeps every element under r
                x = torch.randint(-(1 << 62), 1 << 62, (n, w), dtype=torch.int64, device="cuda", generator=gen_t)
                x[:, -1] &= (1 << 61) - 1
                return x.reshape(-1)

            t1 = rand()
            t2 = t1.reshape(n, w)[torch.randperm(n, device="cuda", generator=gen_t)].reshape(-1).contiguous()
            prove_ms = _wall_ms(lambda: perm.Prove(pk, t1, t2), a.repeat, torch)

            st = torch.cuda.current_stream().cuda_stream
            dom = fft.NewDomain(c, n)
            bufs = [rand() for _ in range(4)]

            def ffts():
                for v in bufs[:2]:
                    dom.fft_device(v, True, fft.DIF, False, st)
                    dom.bit_reverse_device(v, st)
                dom.fft_device(bufs[2], True, fft.DIT, False, st)
                for v in bufs[:3]:
                    dom.fft_device(v, False, fft.DIF, True, st)
                dom.fft_device(bufs[3], True, fft.DIT, True, st)

            def msms():
                for v in bufs:
                    pk._bases.MultiExpDevice(v, n, stream=st)
                for v in bufs[:2]:
                    pk._bases.MultiExpDevice(v, n - 1, stream=st)

            eps, om = curves._fr_encode([0x1234567 % r], r)[0], curves._fr_encode([0x7654321 % r], r)[0]
            dp = kzg._DevicePoly(c, 0, n)
            d_z, d_out = torch.empty_like(t1), torch.empty_like(t1)

            def accumulate():
                dp.permutation_accumulate(t1, t2, n, eps, d_z)

            def numerator():
                dp.permutation_numerator(dom, bufs[0], bufs[1], bufs[2], eps, om, d_out)

            fft_ms = _events_ms(ffts, a.repeat, torch)
            msm_ms = _events_ms(msms, a.repeat, torch)
            acc_ms = _events_ms(accumulate, a.repeat, torch)
            num_ms = _events_ms(numerator, a.repeat, torch)
            acc_b, num_b = 3 * n * fb, 4 * n * fb
            print(json.dumps({
                "workload": "permutation.Prove %s 2^%d, device inputs" % (c, logn), "prove_ms": round(prove_ms, 3),
                "ffts_ms": round(fft_ms, 3), "multiexps_ms": round(msm_ms, 3), "accumulate_ms": round(acc_ms, 3),
                "numerator_ms": round(num_ms, 3),
                "accumulate_TBps": round(acc_b / acc_ms / 1e9, 3), "accumulate_share_of_3.35TBps": round(acc_b / acc_ms / 1e9 / (HBM_BYTES_PER_S / 1e12), 3),
                "numerator_TBps": round(num_b / num_ms / 1e9, 3), "numerator_share_of_3.35TBps": round(num_b / num_ms / 1e9 / (HBM_BYTES_PER_S / 1e12), 3),
            }), flush=True)
            dom.close()
            del t1, t2, bufs, d_z, d_out, dp
            torch.cuda.empty_cache()
        pk.close()


if __name__ == "__main__":
    main()
