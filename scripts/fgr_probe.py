"""Timings of Fast Global Registration on the device (DESIGN.md §3.20), with the card's name and power limit from the
same run.  Host wall time of the synchronous calls, median of --reps after one warm-up call.

  (a) 64 problems of about 3000 matched correspondences: tzr_fgr_batch, and tzr_solve_batch on the same rows as
      context (a different problem: TEASER++'s certifiable robust solve, not a claim about either);
  (b) one problem of 100 000 correspondences (past the robust solve's 65536 cap): one CTA runs all 64 iterations;
  (c) tzr_register_cloud_pairs_fgr against the chain of public calls it replaces (tzr_compute_fpfh_batch,
      tzr_match_correspondences_batch, tzr_fgr_batch) on 64 pairs of 5000-point clouds.

Usage: python scripts/fgr_probe.py [--reps 5]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
capi = importlib.import_module("teaser-plusplus_b200.capi")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def median_ms(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def problem(rng, K, n):
    x = rng.uniform(-1, 1, (n, 3))
    R = np.linalg.qr(rng.normal(size=(3, 3)))[0]
    R *= np.sign(np.linalg.det(R))
    y = x @ R.T + rng.uniform(-1, 1, 3) + rng.normal(scale=1e-3, size=x.shape)
    i = rng.integers(0, n, K)
    j = np.where(rng.random(K) < 0.5, i, rng.integers(0, n, K))
    return x.astype(np.float32), y.astype(np.float32), np.stack([i, j], 1).astype(np.int32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    ctx = capi.Context(0)
    rng = np.random.default_rng(0)
    out = dict(card=card())
    # (a)
    probs = [problem(rng, 3000, 3000) for _ in range(64)]
    X, Y, K = [p[0] for p in probs], [p[1] for p in probs], [p[2] for p in probs]
    out["a_fgr_batch_64x3000_ms"] = median_ms(lambda: ctx.fgr_batch(X, Y, K), a.reps)
    src = [np.ascontiguousarray(x[k[:, 0]], dtype=np.float64) for x, k in zip(X, K)]
    dst = [np.ascontiguousarray(y[k[:, 1]], dtype=np.float64) for y, k in zip(Y, K)]
    prm = capi.default_params(noise_bound=0.01, rotation_cost_threshold=1e-12)
    out["a_solve_batch_64x3000_ms"] = median_ms(lambda: ctx.solve_batch(src, dst, prm), a.reps)
    # (b)
    x, y, k = problem(rng, 100000, 100000)
    out["b_fgr_1x100000_ms"] = median_ms(lambda: ctx.fgr_batch([x], [y], [k]), a.reps)
    out["b_fgr_1x100000_1iter_ms"] = median_ms(lambda: ctx.fgr_batch([x], [y], [k],
                                                                     fgr=capi.fgr_params(iteration_number=1)), a.reps)
    # (c)
    from test_gpu_register_pairs import EXAMPLE, RF, RN, sequence
    clouds, pairs = sequence([5000] * 65, seed=1)
    seeds = list(range(len(pairs)))

    def chain():
        feats = ctx.compute_fpfh_batch(clouds, RN, RF)
        m = ctx.match_correspondences_batch([clouds[p[0]] for p in pairs], [clouds[p[1]] for p in pairs],
                                            [feats[p[0]] for p in pairs], [feats[p[1]] for p in pairs], *EXAMPLE,
                                            tuple_seeds=seeds)
        ctx.fgr_batch([clouds[p[0]] for p in pairs], [clouds[p[1]] for p in pairs], m)

    out["c_register_cloud_pairs_fgr_64x5000_ms"] = median_ms(
        lambda: ctx.register_cloud_pairs_fgr(clouds, pairs, RN, RF, *EXAMPLE, tuple_seeds=seeds), a.reps)
    out["c_three_call_chain_64x5000_ms"] = median_ms(chain, a.reps)
    print(json.dumps(out, indent=1))
    ctx.close()


if __name__ == "__main__":
    main()
