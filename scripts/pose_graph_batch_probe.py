"""Measure tzr_pose_graph_optimize_batch (the batched GNC-TLS pose graph) against a loop of tzr_pose_graph_optimize on
make_fragments-shaped graphs (tests/line_process_fragments.py), for K in {32, 64, 100, 128} and G in {1, 8, 64, 256},
with the iterations each run.  Prints one JSON line per measurement and, with --out PATH, writes them all as one JSON
document with the card's name and power limit read in the same run.  Times are medians of several calls after a warm-up
call; every batched graph's decisions are compared with the single entry's."""
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
from line_process_fragments import fragment  # noqa: E402

R = 0.05


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [x.strip() for x in q.split(",")]
        return name, limit
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})", "unknown"


def graphs(B, K):
    out = []
    for b in range(B):
        gt, e, T, L, u = fragment(1000 * K + b, K, n_wrong=2 if K >= 30 else 0)
        out.append(dict(K=K, edges=e, transforms=T, information=L, uncertain=u))
    return out


def median_ms(f, reps):
    f()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        f()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def loop(ctx, gs):
    return [ctx.optimize_pose_graph(g["K"], g["edges"], g["transforms"], g["information"], R, uncertain=g["uncertain"])
            for g in gs]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", help="write the JSON document here")
    ap.add_argument("--K", type=int, nargs="+", default=[32, 64, 100, 128], help="node counts")
    ap.add_argument("--B", type=int, nargs="+", default=[1, 8, 64, 256], help="batch sizes")
    args = ap.parse_args()
    ctx = capi.Context(0)
    name, limit = card()
    rows = []
    for K in args.K:
        for B in args.B:
            gs = graphs(B, K)
            l0 = ctx.kernel_launches()
            res = ctx.optimize_pose_graph_batch(gs, R)
            launches = ctx.kernel_launches() - l0
            l0 = ctx.kernel_launches()
            sng = loop(ctx, gs)
            launches_loop = ctx.kernel_launches() - l0
            same = sum(r["iterations"] == s["iterations"] and r["inner_iterations"] == s["inner_iterations"] and
                       np.array_equal(r["mask"], s["mask"]) for r, s in zip(res, sng))
            inner = [r["inner_iterations"] for r in res]
            tb = median_ms(lambda: ctx.optimize_pose_graph_batch(gs, R), 5 if B <= 64 else 3)
            tl = median_ms(lambda: loop(ctx, gs), 5 if B <= 8 else 2)
            n = 6 * (K - 1)
            rows.append(dict(K=K, B=B, batch_ms=tb, loop_ms=tl, speedup=tl / tb, launches_batch=launches,
                             launches_loop=launches_loop, decisions_equal=f"{same}/{B}",
                             gnc_iterations_mean=float(np.mean([r["iterations"] for r in res])),
                             inner_mean=float(np.mean(inner)), inner_max=int(max(inner)),
                             factor_mflop=n ** 3 / 3 / 1e6,
                             batch_ms_per_inner_B1=(tb / float(np.mean(inner))) if B == 1 else None))
            print(json.dumps(rows[-1]), flush=True)
    doc = dict(card=name, power_limit=limit, rows=rows)
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(doc, fh, indent=1)
    print(json.dumps(dict(card=name, power_limit=limit)))
    ctx.close()


if __name__ == "__main__":
    main()
