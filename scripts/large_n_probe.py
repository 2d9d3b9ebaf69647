"""Times the solve of problems above 32768 correspondences (the large clique route) and the route's own cost.

Prints one JSON line per case with the card name and power limit read in the same run: the median per-stage device
milliseconds (prep, graph, clique, rot+trans; CUDA events around each stage) of --reps timed calls after one warm-up
call.  Cases: ball model, 99 % outliers, fixed scale, n in {32769, 40000, 49152, 65536} for B = 1 and B = 4
(tzr_solve_batch_dev), and n = 5000 with debug flag 524288 (large route) against the default route.  Writes nothing.

    python scripts/large_n_probe.py [--reps 5]
"""
import argparse
import importlib
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
capi = importlib.import_module("teaser-plusplus_b200.capi")
synth = importlib.import_module("teaser-plusplus_b200.synth")
LARGE = 524288


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    name, pl = out[0].split(", ")
    return name, pl


def run(ctx, torch, n, B, reps, flags=0):
    prs = [synth.make_problem(n, 0.99 if n > 5000 else 0.95, 100 + b, "ball", sigma=0.01,
                              noise_bound=synth.NOISE_BOUND_SIGMA_001) for b in range(B)]
    p = capi.default_params(noise_bound=prs[0]["noise_bound"], estimate_scaling=0)
    src = torch.tensor(np.stack([q["src"] for q in prs]), device="cuda")
    dst = torch.tensor(np.stack([q["dst"] for q in prs]), device="cuda")
    sols = torch.zeros((B, capi.SOLUTION_DTYPE.itemsize), dtype=torch.uint8, device="cuda")
    ctx.set_flags(flags)
    stages = []
    for r in range(reps + 1):
        ctx.solve_batch_dev(p, B, n, src.data_ptr(), dst.data_ptr(), sols.data_ptr())
        ctx.synchronize()
        if r:
            stages.append(ctx.last_stage_ms())
    ctx.set_flags(0)
    recs = np.frombuffer(sols.cpu().numpy().tobytes(), dtype=capi.SOLUTION_DTYPE)
    med = {k: float(np.median([s[k] for s in stages])) for k in stages[0]}
    return med, recs, ctx.clique_route(B)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import torch
    name, pl = card()
    ctx = capi.Context(0, max_n=65536)
    for n in (32769, 40000, 49152, 65536):
        for B in (1, 4):
            med, recs, route = run(ctx, torch, n, B, a.reps)
            print(json.dumps(dict(card=name, power_limit=pl, n=n, B=B, route="large", stage_ms=med,
                                  clique_route=route.tolist(), proven=recs["clique_proven_optimal"].tolist(),
                                  clique_size=recs["clique_size"].tolist())), flush=True)
    for flags, route_name in ((0, "small"), (LARGE, "large")):
        med, recs, route = run(ctx, torch, 5000, 1, a.reps, flags)
        print(json.dumps(dict(card=name, power_limit=pl, n=5000, B=1, route=route_name, stage_ms=med,
                              clique_route=route.tolist(), proven=recs["clique_proven_optimal"].tolist(),
                              clique_size=recs["clique_size"].tolist())), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
