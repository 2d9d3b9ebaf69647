"""Time three ways to solve and certify a batch of C2-geometry problems (n = 1000, rotation_cost_threshold low enough
that every problem's certifier iterates), B = 16 and 64 by default.  One JSON line per (B, workflow) with the card name
and power limit read in the same run, the median wall time of --reps runs (after one warm-up run) and the problems
certified optimal.  Workflows:
  a  B tzr_solve calls (each returns its masks), host-built TIMs, tzr_certify_batch
  b  tzr_solve_batch, tzr_last_inliers per problem, host-built TIMs, tzr_certify_batch
  c  tzr_solve_batch, tzr_certify_last_solve
"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
capi = importlib.import_module("teaser-plusplus_b200.capi")
synth = importlib.import_module("teaser-plusplus_b200.synth")


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    name, pl = out[0].split(", ")
    return name, pl


def chain(src, dst, clique, scale):
    c = np.asarray(clique)
    leaf = np.roll(c, -1)
    return (src[leaf] - src[c]).T, ((dst[leaf] - dst[c]) * (1.0 / scale)).T


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bs", type=int, nargs="+", default=[16, 64])
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    name, pl = card()
    ctx = capi.Context(0)
    for B in a.bs:
        probs = [synth.config_problem("C2", b, n=1000) for b in range(B)]
        srcs, dsts = [p["src"] for p in probs], [p["dst"] for p in probs]
        nb = probs[0]["noise_bound"]
        prm = capi.default_params(noise_bound=nb, estimate_scaling=0, rotation_cost_threshold=1e-12)
        cert = dict(noise_bound=2 * nb, cbar2=1.0)

        def host_certify(sols, masks):
            R, S, D = [], [], []
            for b in range(B):
                s, d = chain(srcs[b], dsts[b], masks[b][2], sols[b]["scale"])
                R.append(sols[b]["R"])
                S.append(s)
                D.append(d)
            return ctx.certify_batch(R, S, D, [m[0] for m in masks], **cert)

        def wf_a():
            ones = [ctx.solve(srcs[b], dsts[b], prm) for b in range(B)]
            return host_certify([dict(scale=o["scale"], R=o["R"]) for o in ones],
                                [(o["rot_inliers"], o["trans_inliers"], o["clique"]) for o in ones])

        def wf_b():
            sols, cliques = ctx.solve_batch(srcs, dsts, prm)
            masks = [ctx.last_inliers(b) + (cliques[b],) for b in range(B)]
            return host_certify([dict(scale=s["scale"], R=capi.rotation_from_solution_record(s)) for s in sols], masks)

        def wf_c():
            ctx.solve_batch(srcs, dsts, prm)
            return ctx.certify_last(**cert)

        for label, fn in (("a", wf_a), ("b", wf_b), ("c", wf_c)):
            fn()
            ts, res = [], None
            for _ in range(a.reps):
                t0 = time.perf_counter()
                res = fn()
                ts.append((time.perf_counter() - t0) * 1e3)
            print(json.dumps(dict(card=name, power_limit=pl, workload="C2", n=1000, B=B, workflow=label,
                                  median_ms=round(float(np.median(ts)), 1), reps=a.reps,
                                  optimal=int(sum(r["is_optimal"] for r in res)),
                                  iterations=int(sum(len(r["suboptimality_traj"]) for r in res)))), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
