"""Times tzr_certify_batch against a loop of tzr_certify (its B = 1 case) on the same inputs.

Inputs: m chain TIMs of a noisy registration problem (unit-cube points, uniform noise inside the noise bound, 10 %
outliers, the true rotation as the estimate; the TIM noise bound is twice the point noise bound), m in {50, 100, 250},
B in {1, 8, 16, 64}.  Every call runs exactly --iters DRS iterations (sub_optimality = -1, so no problem stops early): the
numbers are per-iteration throughput at a fixed amount of work.  For each (m, B) it prints one JSON line with the median
wall time (host clock around the synchronous call) of --reps timed calls after one warm-up call of each: the loop of
single calls, the batch on its default eigen route and the batch with debug flag 2097152 (one cusolverDnDsyevd per
problem).  Cases whose loop takes longer than --budget seconds per call are timed once (reps = 1 in the line).

Uneven convergence, the normal case, gets two more lines timed the same way at the default sub_optimality: the five
reference fixtures in one batch (9, 11, 15, 20 and 1000 iterations; large/case_2 scaled to the common noise bound, which
leaves its gap trajectory unchanged), and m = 250 with one problem held at a wrong rotation (it runs to the cap of 50
iterations) beside 15 that converge on iteration 1.  The card name and power limit are read in the same run.

    python scripts/certify_batch_probe.py [--iters 10] [--reps 3] [--budget 20]
"""
import argparse
import importlib
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
capi = importlib.import_module("teaser-plusplus_b200.capi")
synth = importlib.import_module("teaser-plusplus_b200.synth")
LOOP_EIG = 2097152


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                          "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    return out[0]


def chain_tims(m, seed, nb=0.01):
    rng = np.random.default_rng(seed)
    R = synth.random_rotation(rng)
    p = rng.uniform(-1, 1, size=(m, 3))
    q = p @ R.T + rng.uniform(-nb, nb, size=(m, 3)) / np.sqrt(3)
    out = rng.random(m) < 0.1
    q[out] = rng.uniform(-1, 1, size=(out.sum(), 3))
    nxt = (np.arange(m) + 1) % m
    src, dst = (p[nxt] - p).T, (q[nxt] - q).T
    theta = np.where(out | out[nxt], -1.0, 1.0)
    return R, src, dst, theta


def fixtures():
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import certifier_fixtures as cf
    cases = cf.cases("small") + cf.cases("large")
    nb = cases[0]["params"]["noise_bound"]
    probs = []
    for c in cases:
        s = nb / c["params"]["noise_bound"]
        probs.append((c["R_est"], s * c["v1"], s * c["v2"], c["theta_est"]))
    return probs, dict(noise_bound=nb, cbar2=1.0, max_iterations=1000)


def one_slow(m, B, seed=5):
    probs = []
    for b in range(B):
        rng = np.random.default_rng(seed * 100 + b)
        R = synth.random_rotation(rng)
        src = rng.uniform(-1, 1, size=(3, m))
        dst = R @ src
        th = np.ones(m)
        k0 = int(0.9 * m)
        dst[:, k0:] = rng.uniform(-1, 1, size=(3, m - k0)) * 5 + 5
        th[k0:] = -1
        probs.append((synth.random_rotation(rng) if b == 0 else R, src, dst, th))
    return probs, dict(noise_bound=0.01, cbar2=1.0, max_iterations=50)


def timed(fn, reps):
    fn()  # warm-up
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--budget", type=float, default=20.0)
    ap.add_argument("--ms", default="50,100,250")
    ap.add_argument("--bs", default="1,8,16,64")
    a = ap.parse_args()
    ctx = capi.Context(0)
    kw = dict(noise_bound=0.02, cbar2=1.0, max_iterations=a.iters, sub_optimality=-1.0)
    gpu = card()
    for name, (probs, kwm) in (("fixtures", fixtures()), ("one_slow_m250_B16", one_slow(250, 16))):
        cols = [[p[k] for p in probs] for k in range(4)]
        loop = lambda: [ctx.certify(*p, **kwm) for p in probs]

        def batch(flags):
            ctx.set_flags(flags)
            try:
                return ctx.certify_batch(*cols, **kwm)
            finally:
                ctx.set_flags(0)

        ref, got = loop(), batch(0)
        row = dict(gpu=gpu, case=name, B=len(probs), n=[4 * p[3].size + 4 for p in probs],
                   iterations=[len(r["suboptimality_traj"]) for r in got], reps=a.reps,
                   loop_ms=timed(loop, a.reps), batch_ms=timed(lambda: batch(0), a.reps),
                   batch_loop_eig_ms=timed(lambda: batch(LOOP_EIG), a.reps),
                   same_lengths=all(len(r["suboptimality_traj"]) == len(g["suboptimality_traj"])
                                    for r, g in zip(ref, got)))
        row["speedup"] = row["loop_ms"] / row["batch_ms"]
        print(json.dumps(row), flush=True)
    for m in [int(x) for x in a.ms.split(",")]:
        for B in [int(x) for x in a.bs.split(",")]:
            probs = [chain_tims(m, 1000 * m + b) for b in range(B)]
            cols = [[p[k] for p in probs] for k in range(4)]

            def loop():
                return [ctx.certify(*p, **kw) for p in probs]

            def batch(flags):
                ctx.set_flags(flags)
                try:
                    return ctx.certify_batch(*cols, **kw)
                finally:
                    ctx.set_flags(0)

            t0 = time.perf_counter()
            ref = loop()
            once = time.perf_counter() - t0
            reps = a.reps if once < a.budget else 1
            got = batch(0)
            err = max(float(np.abs(r["suboptimality_traj"] - g["suboptimality_traj"]).max()) for r, g in zip(ref, got))
            row = dict(gpu=gpu, m=m, n=4 * m + 4, B=B, iters=a.iters, reps=reps,
                       loop_ms=timed(loop, reps), batch_ms=timed(lambda: batch(0), reps),
                       batch_loop_eig_ms=timed(lambda: batch(LOOP_EIG), reps), max_traj_diff=err)
            row["speedup"] = row["loop_ms"] / row["batch_ms"]
            row["speedup_loop_eig"] = row["loop_ms"] / row["batch_loop_eig_ms"]
            print(json.dumps(row), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
