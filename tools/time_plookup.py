"""Wall time of plookup.ProveLookupVector on device-resident inputs (bn254 and bls12-381 at s = 2^20 and 2^22 by default: a table of s
random entries and a vector of s - 1 values drawn from it), and the same work broken into its parts, each timed alone with CUDA
events on vectors of the same length:
  * sorts: the two sorts of ProveLookupVector (the table lt, s keys, and lt || lf, 2s - 1 keys);
  * sort_table / sort_merged: each of them alone, with the sort rate as the bytes of the keys over the time;
  * ffts: the eleven transforms (FFTInverse DIF + BitReverse of lt, lf, h1, h2 and z on s points, FFT DIF on the coset of the five
    on 2s points, FFTInverse DIT on the coset of the numerator);
  * multiexps: the eight MultiExps (Commit of t, f, h1, h2, z on s scalars and of h on 2s, the quotients of the two
    BatchOpenSinglePoint on 2s - 1 and s - 1);
  * accumulate / numerator: the two new Fr entry points.
What ProveLookupVector adds to the parts is the padding and copies, the transcript, the openings' Fr scans and folds, the copies of
the digests and claimed values, and the allocations.  Prints the card name and power limit read in the same run, then one JSON
line per workload.

  python tools/time_plookup.py [--repeat 5] [--curves bn254,bls12381] [--logs 20,22]"""
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
    pl = import_module("gnark-crypto_b200.plookup")
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
        pk = kzg.ProvingKey(c, kzg.new_srs_g1(c, 2 << max(logs), 0xC0FFEE % r, gen, r, G.encode_scalars))
        gen_t = torch.Generator(device="cuda").manual_seed(1)
        for logn in logs:
            s = 1 << logn

            def rand(n):        # reduced limbs: the top limb below 2^61 keeps every element under r
                x = torch.randint(-(1 << 62), 1 << 62, (n, w), dtype=torch.int64, device="cuda", generator=gen_t)
                x[:, -1] &= (1 << 61) - 1
                return x.reshape(-1)

            t = rand(s)
            f = t.reshape(s, w)[torch.randint(0, s, (s - 1,), device="cuda", generator=gen_t)].reshape(-1).contiguous()
            prove_ms = _wall_ms(lambda: pl.ProveLookupVector(pk, f, t), a.repeat, torch)

            st = torch.cuda.current_stream().cuda_stream
            dom, big = fft.NewDomain(c, s), fft.NewDomain(c, 2 * s)
            small = [rand(s) for _ in range(5)]
            large = [rand(2 * s) for _ in range(6)]
            merged = rand(2 * s - 1)
            dp = kzg._DevicePoly(c, 0, 2 * s)
            d_out = torch.empty_like(merged)

            def sort_table():
                dp.sort(t, s, d_out)

            def sort_merged():
                dp.sort(merged, 2 * s - 1, d_out)

            def sorts():
                sort_table()
                sort_merged()

            def ffts():
                for v in small:
                    dom.fft_device(v, True, fft.DIF, False, st)
                    dom.bit_reverse_device(v, st)
                for v in large[:5]:
                    big.fft_device(v, False, fft.DIF, True, st)
                big.fft_device(large[5], True, fft.DIT, True, st)

            def msms():
                for v in small:
                    pk._bases.MultiExpDevice(v, s, stream=st)
                pk._bases.MultiExpDevice(large[0], 2 * s, stream=st)
                pk._bases.MultiExpDevice(large[1], 2 * s - 1, stream=st)
                pk._bases.MultiExpDevice(small[0], s - 1, stream=st)

            beta, gamma, alpha = (curves._fr_encode([v % r], r)[0] for v in (0x1234567, 0x7654321, 0xABCDEF))
            d_z, d_num = torch.empty_like(t), torch.empty_like(large[0])

            def accumulate():
                dp.plookup_accumulate(small[0], small[1], small[2], small[3], s, beta, gamma, d_z)

            def numerator():
                dp.plookup_numerator(big, *large[:5], beta, gamma, alpha, d_num)

            sort_t_ms = _events_ms(sort_table, a.repeat, torch)
            sort_m_ms = _events_ms(sort_merged, a.repeat, torch)
            sorts_ms = _events_ms(sorts, a.repeat, torch)
            fft_ms = _events_ms(ffts, a.repeat, torch)
            msm_ms = _events_ms(msms, a.repeat, torch)
            acc_ms = _events_ms(accumulate, a.repeat, torch)
            num_ms = _events_ms(numerator, a.repeat, torch)
            print(json.dumps({
                "workload": "plookup.ProveLookupVector %s s=2^%d, random table, device inputs" % (c, logn), "prove_ms": round(prove_ms, 3),
                "sorts_ms": round(sorts_ms, 3), "sort_table_ms": round(sort_t_ms, 3), "sort_merged_ms": round(sort_m_ms, 3),
                "sort_merged_GBps": round((2 * s - 1) * fb / sort_m_ms / 1e6, 1),
                "ffts_ms": round(fft_ms, 3), "multiexps_ms": round(msm_ms, 3), "accumulate_ms": round(acc_ms, 3),
                "numerator_ms": round(num_ms, 3),
            }), flush=True)
            dom.close()
            big.close()
            del t, f, small, large, merged, d_out, d_z, d_num, dp
            torch.cuda.empty_cache()
        pk.close()


if __name__ == "__main__":
    main()
