"""Times mpcsetup.UpdateMonomialsG1 / G2 on one GPU: device-resident points ([1 + i]g, from gmsm_generate_multiples_device), updated in
place on the current stream, CUDA events around each call after a warm-up.

Reported per (group, n): the call time, points per second, and the output checked against its closed form: after one update by r
of [1 + i]g, A[0] is unchanged and A[i] = [(1 + i) r^i]g, compared limb for limb with BatchScalarMultiplication (the fixed-base
kernels) at 4096 random indices, the first 8 and the last 8.  Prints the card's name and power limit first, then one JSON line per
case.

--ab runs the A/B timing of the window width of the kernel's ladder: this script at the --ab-cases sizes under the library (its
default width, scale_w in csrc/mpc_kernels.cuh) and under the variant builds GMSM_LIB=w3 and w5 (build.py with GMSM_BUILD_TAG=w3,
GMSM_NVCC_EXTRA=-DGMSM_SCALE_W=3; w5 likewise), alternated twice in one run, then one summary line per case.  Needs a GPU and the
built libraries.

    python tools/time_mpcsetup.py [--reps 3] [--warmup 1] [--cases bn254_g1:22,bls12381_g1:24] [--ab] [--ab-cases bn254_g1:22]"""
import argparse
import importlib
import json
import os
import random
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DEFAULT = [("bn254_g1", 22), ("bn254_g1", 24), ("bls12381_g1", 22), ("bls12381_g1", 24), ("bn254_g2", 22)]
AB_DEFAULT = [("bn254_g1", 22), ("bls12381_g1", 22), ("bn254_g2", 20)]


def _cases(s, default):
    return [(c.split(":")[0], int(c.split(":")[1])) for c in s.split(",") if c] or default


def card():
    import torch

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return {"card": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[0] if q.stdout.strip() else "",
            "lib": os.environ.get("GMSM_LIB", "")}


def time_cases(cases, reps, warmup):
    import numpy as np
    import torch

    import gnark_crypto_b200  # noqa: F401
    from oracle import oracle as O

    native = importlib.import_module("gnark-crypto_b200._native")
    mx = importlib.import_module("gnark-crypto_b200.multiexp")
    mpc = importlib.import_module("gnark-crypto_b200.mpcsetup")
    curves = importlib.import_module("gnark-crypto_b200.curves")
    L = native.lib()
    dev = torch.device("cuda", 0)
    for name, logn in cases:
        curve, g = name.split("_")
        upd = mpc.UpdateMonomialsG1 if g == "g1" else mpc.UpdateMonomialsG2
        G = O.GROUPS[name]
        q = G.fr.q
        cid = curves.GROUPS[name].id
        n = 1 << logn
        words = G.aff_words
        base = G.encode_affine([G.gen])[0]
        rng = random.Random(logn * 100 + cid)
        r = rng.randrange(2, q)
        rl = curves._fr_encode([r], q)[0]
        pts = torch.empty(n * words, dtype=torch.int64, device=dev)
        st = torch.cuda.current_stream(dev).cuda_stream
        mx._check(L.gmsm_generate_multiples_device(cid, base.ctypes.data, 1, n, pts.data_ptr(), st))
        first = pts[:words].clone()
        # closed-form check of one update
        upd(curve, pts, rl)
        idx = sorted(set(list(range(8)) + list(range(n - 8, n)) + [rng.randrange(n) for _ in range(4096)]))
        got = pts.view(n, words)[torch.tensor(idx, device=dev)].cpu().numpy().view(np.uint64)
        want = mx.BatchScalarMultiplication(name, base, curves._fr_encode([(1 + i) * pow(r, i, q) % q for i in idx], q))
        ok = bool(np.array_equal(got, want)) and bool(torch.equal(pts[:words], first))
        # timing: further updates of the same (valid) points
        for _ in range(warmup):
            upd(curve, pts, rl)
        torch.cuda.synchronize()
        ms = []
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            upd(curve, pts, rl)
            e1.record()
            e1.synchronize()
            ms.append(e0.elapsed_time(e1))
        t = sorted(ms)[len(ms) // 2]
        rec = {"group": name, "logn": logn, "n": n, "ms_median": round(t, 2), "ms_all": [round(x, 2) for x in ms],
               "points_per_s": round((n - 1) / (t * 1e-3)), "closed_form_ok": ok, "checked_indices": len(idx), "lib": os.environ.get("GMSM_LIB", "")}
        print(json.dumps(rec), flush=True)
        if not ok:
            raise SystemExit("closed-form check failed: %s 2^%d" % (name, logn))
        del pts
        torch.cuda.empty_cache()


def ab(cases, reps, warmup):
    libs = [("", "default"), ("w3", "W=3"), ("w5", "W=5")]
    spec = ",".join("%s:%d" % c for c in cases)
    res = {}
    for rnd in range(2):
        for tag, label in libs:
            env = dict(os.environ, GMSM_LIB=tag)
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--cases", spec, "--reps", str(reps), "--warmup", str(warmup),
                                "--no-card"], env=env, capture_output=True, text=True)
            if p.returncode:
                raise SystemExit("A/B run %s failed:\n%s%s" % (label, p.stdout, p.stderr))
            for line in p.stdout.splitlines():
                rec = json.loads(line)
                rec["round"], rec["variant"] = rnd, label
                print(json.dumps(rec), flush=True)
                res.setdefault((rec["group"], rec["logn"]), {}).setdefault(label, []).append(rec["ms_median"])
    for (name, logn), v in res.items():
        print(json.dumps({"ab_summary": name, "logn": logn, "ms_by_variant": v,
                          "fastest": min(v, key=lambda k: min(v[k]))}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--cases", default="")
    ap.add_argument("--ab", action="store_true")
    ap.add_argument("--ab-cases", default="")
    ap.add_argument("--no-card", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if not args.no_card:
        print(json.dumps(card()), flush=True)
    time_cases(_cases(args.cases, DEFAULT), args.reps, args.warmup)
    if args.ab:
        ab(_cases(args.ab_cases, AB_DEFAULT), args.reps, args.warmup)


if __name__ == "__main__":
    main()
