"""Many scan sequences in one multiway call: tzr_register_cloud_pairs_multiway(_line_process)_batch against a loop of
register_multiway, for both optimisers, in the same run.

Sequences are scripts/multiway_probe.py's (32 scans of 2000 points, odometry pairs and a loop closure every 8 scans);
--distinct of them are generated and cycled, so that S = 256 does not spend minutes on the host.  For each S reports:
the batch's and the loop's time (median of --reps calls after a warm-up call); the pose-graph share of each (the
batched pose-graph entry on the batch's graphs, and the sum of the single entry over them, timed the same way); the
map step's device time (from one separately profiled call with map_voxel_size: the summed durations of the kernels
from map_transform_kernel's start on, which are the map's transform and voxel pipeline, the call's last device work);
whether every sequence's decisions matched the loop's; and the card's name and power limit, read in the same run.
JSON lines on stdout; --out PATH writes one document.

usage: python scripts/multiway_batch_probe.py [--sizes 1,8,64,256] [--scans 32] [--n 2000] [--reps 2] [--out rows.json]"""
import argparse
import importlib
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
capi = importlib.import_module("teaser-plusplus_b200.capi")
mp = importlib.import_module("multiway_probe")

VOX = 0.02
LP_KEYS = ("iterations", "trials", "stop_reason", "pruned", "mu")


def decisions(d, optimizer):
    if optimizer == "line_process":
        return tuple(str(d[k]) for k in LP_KEYS) + (d["kept"].tobytes(), d["status"])
    return d["iterations"], d["inner_iterations"], d["mask"].tobytes(), d["status"]


def map_kernel_ms(fn):
    """Device time of the map step of one call of fn: the kernels that start at or after map_transform_kernel"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as fh:
            ev = [e for e in json.load(fh)["traceEvents"] if e.get("cat") == "kernel"]
    start = min(e["ts"] for e in ev if "map_transform_kernel" in e["name"])
    return sum(e["dur"] for e in ev if e["ts"] >= start) / 1e3


def graphs_of(res, pairs):
    """The pose graphs the call built: each sequence's refined pairs, their transforms and information matrices"""
    out = []
    for r, pr in zip(res, pairs):
        icp, d = r[6], r[7]
        refined = [p for p in range(len(pr)) if icp[p]["transform"]["scale"] > 0]
        out.append(dict(K=len(d["poses"]), edges=[pr[p] for p in refined], information=d["information"][refined],
                        transforms=[dict(scale=1.0, rotation=icp[p]["transform"]["rotation"],
                                         translation=icp[p]["transform"]["translation"]) for p in refined],
                        uncertain=[0 if pr[p][1] == pr[p][0] + 1 else 1 for p in refined]))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,8,64,256")
    ap.add_argument("--scans", type=int, default=32)
    ap.add_argument("--n", type=int, default=2000)
    ap.add_argument("--distinct", type=int, default=8)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    card = mp.card()
    print("card:", card, flush=True)
    pool = [mp.sequence(a.n, a.scans, 7 + 100 * k)[0] for k in range(a.distinct)]
    pr = [(k, k + 1) for k in range(a.scans - 1)] + [(k, k - 2) for k in range(2, a.scans, 8)]
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=0, rotation_cost_threshold=1e-12)
    ctx = capi.Context(0)
    rows = []
    for S in [int(x) for x in a.sizes.split(",")]:
        seqs, pairs = [pool[k % a.distinct] for k in range(S)], [pr] * S
        for optimizer in ("gnc_tls", "line_process"):
            kw = dict(optimizer=optimizer, **mp.FLAGS)
            t_batch, got = mp.median_time(lambda: ctx.register_multiway_batch(seqs, pairs, prm, mp.R_CORR, **kw),
                                          a.reps)
            map_ms = map_kernel_ms(lambda: ctx.register_multiway_batch(seqs, pairs, prm, mp.R_CORR,
                                                                       map_voxel_size=VOX, **kw))
            t_loop, loop = mp.median_time(lambda: [ctx.register_multiway(s, p, prm, mp.R_CORR, **kw)
                                                   for s, p in zip(seqs, pairs)], a.reps)
            gr = graphs_of(got, pairs)
            if optimizer == "line_process":
                t_pg_batch, _ = mp.median_time(lambda: ctx.global_optimization_batch(gr, mp.R_CORR), a.reps)
                t_pg_loop, _ = mp.median_time(lambda: [ctx.global_optimization(g["K"], g["edges"], g["transforms"],
                                                                               g["information"], mp.R_CORR,
                                                                               uncertain=g["uncertain"]) for g in gr],
                                              a.reps)
            else:
                t_pg_batch, _ = mp.median_time(lambda: ctx.optimize_pose_graph_batch(gr, mp.R_CORR), a.reps)
                t_pg_loop, _ = mp.median_time(lambda: [ctx.optimize_pose_graph(g["K"], g["edges"], g["transforms"],
                                                                               g["information"], mp.R_CORR,
                                                                               uncertain=g["uncertain"]) for g in gr],
                                              a.reps)
            row = dict(S=S, scans=a.scans, n=a.n, optimizer=optimizer, batch_ms=1e3 * t_batch, loop_ms=1e3 * t_loop,
                       speedup=t_loop / t_batch, pose_graph_batch_ms=1e3 * t_pg_batch,
                       pose_graph_loop_ms=1e3 * t_pg_loop, map_kernel_ms=map_ms,
                       solved=sum(r[7]["status"] == 0 for r in got),
                       decisions_match=all(decisions(x[7], optimizer) == decisions(y[7], optimizer)
                                           for x, y in zip(got, loop)),
                       pairs_match=all(x[6].tobytes() == y[6].tobytes() for x, y in zip(got, loop)), card=card)
            rows.append(row)
            print(json.dumps(row), flush=True)
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(dict(card=card, rows=rows), fh)
    ctx.close()


if __name__ == "__main__":
    main()
