"""Where the time of a device-resident MultiExp goes between the scatter (K1c) and the bucket accumulation (K2): for each
configuration, the call time, the stage times, and the timeline of profiling level 2 -- CUDA events around every
k_scatter_window launch, on the call's stream and on the context's auxiliary stream, around both k_accumulate parts, and the
wait of part 2 for the auxiliary stream.  One JSON line per configuration (medians over the timed calls), then a table.
The card's name, power limit and SM clock are read in the same run.

  python tools/time_msm_timeline.py [--curve bn254_g1] [--logn 24] [--steps 7] [--configs default,split15,plain,rank]

A configuration sets the engine's knobs for its own context: `default` (none), `splitS` (GMSM_SPLIT_W=S: S windows scattered
on the call's stream before the accumulate, the rest underneath part 1; S >= W scatters everything first, one part),
`plain` / `rank` (GMSM_K1_MODE), combined with `+` (e.g. `split4+rank`).  Inputs are bench.py's: bases [1 + i]·B, seeded
uniform scalars.  Every configuration must give the same MultiExp result; `result` shows it."""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench as B  # noqa: E402  (the headline's input generators)

KNOBS = ("GMSM_SPLIT_W", "GMSM_K1_MODE")


def card():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    vals = [s.strip() for s in r.stdout.splitlines()[0].split(",")] if r.returncode == 0 and r.stdout else ["unknown"] * 4
    return dict(zip(("name", "power_limit", "max_sm_clock", "sm_clock_idle"), vals))


def knobs_of(cfg):
    env = {}
    for part in cfg.split("+"):
        if part == "default":
            continue
        if part.startswith("split"):
            env["GMSM_SPLIT_W"] = part[5:]
        elif part in ("plain", "rank"):
            env["GMSM_K1_MODE"] = part
        else:
            raise SystemExit("unknown configuration %r" % cfg)
    return env


def summarise(tl, stages):
    passes, parts = tl["passes"], tl["parts"]
    main = [(s, e) for k, s, e in passes if k == "main"]
    aux = [(s, e) for k, s, e in passes if k == "aux"]
    out = {
        "scatter_ms_per_pass": [round(e - s, 4) for _, s, e in passes],
        "scatter_main_ms": round(sum(e - s for s, e in main), 4),
        "aux_span_ms": round(max(e for _, e in aux) - min(s for s, _ in aux), 4) if aux else 0.0,
        "aux_end_ms": round(max(e for _, e in aux), 4) if aux else None,
        "part_ms": [round(e - s, 4) for s, e in parts],
        "accumulate_pure_ms": round(sum(e - s for s, e in parts), 4),
        "stage_accumulate_ms": round(stages[3], 4),
        "stages_ms": dict(zip(B.STAGE_NAMES, [round(x, 4) for x in stages])),
    }
    if len(parts) == 2:
        out["part1_start_ms"] = round(parts[0][0], 4)
        out["part2_wait_ms"] = round(parts[1][0] - parts[0][1], 4)
        # scatter time of the auxiliary stream that ran while part 1 ran (the launches' own ends; CUDA events only bound them)
        p1s, p1e = parts[0]
        out["aux_under_part1_ms"] = round(sum(max(0.0, min(e, p1e) - max(s, p1s)) for s, e in aux), 4)
    return out


def median_dict(ds):
    out = {}
    for k in ds[0]:
        v = [d[k] for d in ds]
        if isinstance(v[0], list):
            out[k] = [round(statistics.median(x), 4) for x in zip(*v)]
        elif isinstance(v[0], dict):
            out[k] = median_dict(v)
        elif v[0] is None:
            out[k] = None
        else:
            out[k] = round(statistics.median(v), 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--curve", default="bn254_g1")
    ap.add_argument("--logn", type=int, default=24)
    ap.add_argument("--steps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--configs", default="default,split15,plain,rank")
    ap.add_argument("--label", default="", help="name of this build in the output")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch

    import gnark_crypto_b200 as pkg

    g, n = a.curve, 1 << a.logn
    info = card()
    h_scalars = B.synth_scalars(n, B.CURVE_BITS[g], 0x5EED0000 + 2, B.fr_mod(g))
    lines = []
    for cfg in a.configs.split(","):
        env = knobs_of(cfg)
        for k in KNOBS:
            os.environ.pop(k, None)
        os.environ.update(env)
        eng = pkg.Engine(g, n)
        d_b = eng.generate_multiples(B._generator_limbs(g), B.BASE_MULT, 1)
        base = d_b.cpu().numpy().view(np.uint64).copy()
        d_points = eng.generate_multiples(base, 1, n)
        d_scalars = eng.to_device(h_scalars)
        torch.cuda.synchronize()
        # call time at profiling level 1 (what bench.py times), back to back
        eng.set_profiling(1)
        for _ in range(a.warmup):
            eng.msm(d_points, d_scalars, n)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.steps):
            out = eng.msm(d_points, d_scalars, n)
        e1.record()
        torch.cuda.synchronize()
        call_ms = e0.elapsed_time(e1) / a.steps
        res = hashlib.sha256(out.cpu().numpy().tobytes()).hexdigest()[:16]
        # the timeline, one call at a time
        eng.set_profiling(2)
        eng.msm(d_points, d_scalars, n)
        torch.cuda.synchronize()
        per = []
        for _ in range(a.steps):
            eng.msm(d_points, d_scalars, n)
            torch.cuda.synchronize()
            per.append(summarise(eng.last_timeline_ms(), eng.last_stage_ms()))
        line = {"build": a.label, "config": cfg, "knobs": env, "curve": g, "logn": a.logn, "c": eng.c, "windows": eng.nwin,
                "call_ms": round(call_ms, 4), "result": res, "launches": eng.last_launches, "steps": a.steps}
        line.update(median_dict(per))
        line["card"] = info
        print(json.dumps(line), flush=True)
        lines.append(line)
        eng.close()
        del d_points, d_scalars, eng
        torch.cuda.empty_cache()
    for k in KNOBS:
        os.environ.pop(k, None)
    print("\n%-14s %-16s %8s %9s %8s %8s %8s %8s %8s" % ("build", "config", "call", "scat/pass", "acc", "part1", "wait", "part2",
                                                          "aux_span"))
    for ln in lines:
        pm = ln["part_ms"] + [0.0] * (2 - len(ln["part_ms"]))
        print("%-14s %-16s %8.2f %9.3f %8.2f %8.2f %8.2f %8.2f %8.2f" % (
            ln["build"], ln["config"], ln["call_ms"], statistics.median(ln["scatter_ms_per_pass"]), ln["accumulate_pure_ms"],
            pm[0], ln.get("part2_wait_ms", 0.0), pm[1], ln["aux_span_ms"]))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "a") as f:
            for ln in lines:
                f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
