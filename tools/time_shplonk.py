"""Wall time of shplonk.BatchOpen and fflonk.BatchOpen on bn254 with device-tensor inputs, against the two MultiExps (W and W') they
contain, timed alone on scalars of the same lengths.  The difference is the Fr work (chained divisions by (X - a), two linear
combinations, one division by (X - z)), the transcript and the one copy of the claimed values.

  python tools/time_shplonk.py [--repeat 3] [--log-shplonk 22] [--log-fflonk 20]

Workloads: SHPLONK, 8 polynomials of 2^22 coefficients, 7 opened at {z} and 1 at {z, z w} (PLONK-style); FFLONK, one pack of 9 at {z}
and one pack of 3 at {z, z w}, 2^20 coefficients each.  The SRS is [alpha^i]G from new_srs_g1 on the device.  Prints the card name
and power limit read in the same run, then one JSON line per workload."""
import argparse
import hashlib
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


def _timed(fn, repeat, torch):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(repeat):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return min(ts), float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--log-shplonk", type=int, default=22)
    ap.add_argument("--log-fflonk", type=int, default=20)
    a = ap.parse_args()
    import torch

    kzg = import_module("gnark-crypto_b200.kzg")
    curves = import_module("gnark-crypto_b200.curves")
    shplonk = import_module("gnark-crypto_b200.shplonk")
    fflonk = import_module("gnark-crypto_b200.fflonk")
    from oracle import oracle as O

    c = "bn254"
    cp = kzg.CURVE_PARAMS[c]
    r, w = cp.r, cp.fr_words
    print("card:", _card(), flush=True)
    ns, nf = 1 << a.log_shplonk, 1 << a.log_fflonk
    t9 = fflonk._next_divisor_r_minus_one(9, r)
    srs_n = max(ns, t9 * nf) + 32
    G = O.GROUPS[c + "_g1"]
    gen = G.encode_affine([G.gen])[0]
    pk = kzg.ProvingKey(c, kzg.new_srs_g1(c, srs_n, 0xC0FFEE % r, gen, r, G.encode_scalars))
    gen_t = torch.Generator(device="cuda").manual_seed(1)

    def rand(n):        # reduced limbs: the top limb below 2^61 keeps every element under r
        x = torch.randint(-(1 << 62), 1 << 62, (n, w), dtype=torch.int64, device="cuda", generator=gen_t)
        x[:, -1] &= (1 << 61) - 1
        return x.reshape(-1)

    zeta = 0x1234567 % r
    omega = fflonk._ith_root_one(2, c)
    enc = lambda S: curves._fr_encode(S, r).reshape(-1, w)          # noqa: E731
    st = torch.cuda.current_stream().cuda_stream

    polys = [rand(ns) for _ in range(8)]
    digests = [kzg.Commit(p, pk) for p in polys]
    sets = [[zeta]] * 7 + [[zeta, zeta * omega % r]]
    pts = [enc(S) for S in sets]
    nT = 9
    wl, wpl = ns, ns - 1
    d_w, d_wp = rand(wl), rand(wpl)
    b_open = _timed(lambda: shplonk.BatchOpen(polys, digests, pts, hashlib.sha256, pk), a.repeat, torch)
    b_msm = _timed(lambda: (pk._bases.MultiExpDevice(d_w, wl, stream=st), pk._bases.MultiExpDevice(d_wp, wpl, stream=st)), a.repeat, torch)
    print(json.dumps({"workload": "shplonk bn254 8 x 2^%d, 7 at {z}, 1 at {z, zw}" % a.log_shplonk, "batch_open_s": b_open,
                      "two_multiexps_s": b_msm, "W_len": wl, "Wprime_len": wpl, "T": nT}), flush=True)
    del polys, d_w, d_wp

    packs = [[rand(nf) for _ in range(9)], [rand(nf) for _ in range(3)]]
    fdig = [fflonk.FoldAndCommit(p, pk) for p in packs]
    fsets = [enc([zeta]), enc([zeta, zeta * omega % r])]
    t3 = fflonk._next_divisor_r_minus_one(3, r)
    wl = max(t9 * nf, t3 * nf)
    d_w, d_wp = rand(wl), rand(wl - 1)
    f_open = _timed(lambda: fflonk.BatchOpen(packs, fdig, fsets, hashlib.sha256, pk), a.repeat, torch)
    f_msm = _timed(lambda: (pk._bases.MultiExpDevice(d_w, wl, stream=st), pk._bases.MultiExpDevice(d_wp, wl - 1, stream=st)), a.repeat, torch)
    f_commit = _timed(lambda: fflonk.FoldAndCommit(packs[0], pk), a.repeat, torch)
    print(json.dumps({"workload": "fflonk bn254 pack 9 at {z} (t=%d), pack 3 at {z, zw} (t=%d), 2^%d each" % (t9, t3, a.log_fflonk),
                      "batch_open_s": f_open, "two_multiexps_s": f_msm, "fold_and_commit_9_s": f_commit, "W_len": wl,
                      "T": t9 + 2 * t3}), flush=True)
    pk.close()


if __name__ == "__main__":
    main()
