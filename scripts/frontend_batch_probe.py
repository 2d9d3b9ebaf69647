"""Front-end throughput for many cloud pairs: FPFH of both clouds plus correspondence matching, as a loop of single
calls (compute_fpfh x 2 + match_correspondences per pair) and as the batch calls (compute_fpfh_batch over all 2B
clouds + match_correspondences_batch over the B pairs).  Both must produce identical outputs.

The clouds are wavy surface patches (tests/test_gpu_fpfh.py) with per-point noise; the target of every pair is a
rigidly moved (small rotation, 5 cm shift), permuted copy that shares 2/3 of the source's points (the rest are new
samples of the surface), like synth.matcher_problem's partial overlap.  Matching uses the example's flags
(examples/teaser_cpp_fpfh: absolute scale off, cross check on, no tuple test).

usage: python scripts/frontend_batch_probe.py [--reps 3] [--out results.json]
Prints one JSON line per (n, B) and the card's name and power limit; --out also writes the rows to a JSON file.  A context without the batch calls (an older
build) is timed on the single-call loop only."""
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

RADII = {1000: (0.1, 0.15), 5000: (0.05, 0.075)}


def surface(rng, n):
    uv = rng.uniform(-1, 1, size=(n, 2))
    pts = np.stack([uv[:, 0], uv[:, 1], 0.3 * np.sin(3 * uv[:, 0]) * np.cos(2 * uv[:, 1])], axis=1)
    return pts + rng.normal(scale=0.003, size=pts.shape) + np.array([0.5, -0.2, 2.0])


def make_pair(n, seed):
    rng = np.random.default_rng(seed)
    src = surface(rng, n)
    keep = n - n // 3
    dst = np.concatenate([src[:keep], surface(rng, n - keep)])[rng.permutation(n)]
    a = rng.normal(size=3)
    a *= 0.05 / np.linalg.norm(a)                        # ~3 degree rotation
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    R = np.eye(3) + np.sin(0.05) * K / 0.05 + (1 - np.cos(0.05)) * (K @ K) / 0.05 ** 2
    dst = dst @ R.T + np.array([0.05, 0.0, 0.0])
    return src.astype(np.float32), dst.astype(np.float32)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
        return name, power
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})", "unknown"


def timed(fn, reps):
    fn()  # warm-up of this shape
    ts = []
    out = None
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)), float(min(ts)), float(max(ts)), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sizes", default="1000,5000")
    ap.add_argument("--batches", default="1,16,256")
    ap.add_argument("--out", default=None, help="JSON file for the rows (default: stdout only)")
    a = ap.parse_args()
    ctx = capi.Context(0)
    has_batch = hasattr(ctx, "compute_fpfh_batch")
    name, power = card()
    print(json.dumps(dict(card=name, power_limit=power, batch_calls=has_batch)), flush=True)
    flags = (False, True, False, 0.95)
    rows = []
    for n in [int(x) for x in a.sizes.split(",")]:
        rn, rf = RADII[n]
        for B in [int(x) for x in a.batches.split(",")]:
            pairs = [make_pair(n, 1000 * n + b) for b in range(B)]
            seeds = list(range(B))

            def singles():
                out = []
                for (s, d), seed in zip(pairs, seeds):
                    fs = ctx.compute_fpfh(s, rn, rf)
                    fd = ctx.compute_fpfh(d, rn, rf)
                    out.append((fs, fd, ctx.match_correspondences(s, d, fs, fd, *flags, tuple_seed=seed)))
                return out

            def batch():
                f = ctx.compute_fpfh_batch([p[0] for p in pairs] + [p[1] for p in pairs], rn, rf)
                fs, fd = f[:B], f[B:]
                m = ctx.match_correspondences_batch([p[0] for p in pairs], [p[1] for p in pairs], fs, fd, *flags,
                                                    tuple_seeds=seeds)
                return list(zip(fs, fd, m))

            med_s, min_s, max_s, out_s = timed(singles, a.reps)
            row = dict(n=n, B=B, reps=a.reps, single_loop_ms=1e3 * med_s, single_loop_ms_range=[1e3 * min_s, 1e3 * max_s],
                       single_per_pair_ms=1e3 * med_s / B, mean_pairs=float(np.mean([len(o[2]) for o in out_s])))
            if has_batch:
                med_b, min_b, max_b, out_b = timed(batch, a.reps)
                same = all(np.array_equal(x[0], y[0], equal_nan=True) and np.array_equal(x[1], y[1], equal_nan=True)
                           and np.array_equal(x[2], y[2]) for x, y in zip(out_s, out_b))
                # stage split of the batch: descriptors alone, matching alone (inputs precomputed)
                fl = [p[0] for p in pairs] + [p[1] for p in pairs]
                med_f = timed(lambda: ctx.compute_fpfh_batch(fl, rn, rf), a.reps)[0]
                fs, fd = [o[0] for o in out_b], [o[1] for o in out_b]
                med_m = timed(lambda: ctx.match_correspondences_batch([p[0] for p in pairs], [p[1] for p in pairs],
                                                                      fs, fd, *flags, tuple_seeds=seeds), a.reps)[0]
                row.update(batch_ms=1e3 * med_b, batch_ms_range=[1e3 * min_b, 1e3 * max_b],
                           batch_per_pair_ms=1e3 * med_b / B, batch_fpfh_ms=1e3 * med_f, batch_match_ms=1e3 * med_m,
                           speedup=med_s / med_b, identical=bool(same))
                assert same, f"batch and single calls differ at n={n} B={B}"
            row.update(card=name, power_limit=power)
            rows.append(row)
            print(json.dumps(row), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(rows, fh, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
