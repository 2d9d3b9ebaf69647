"""Open3D's line process against the GNC-TLS pose graph, and the line process at the K = 1024 cap.

1. The 32-scan sequence of scripts/multiway_probe.py (odometry, closures two scans apart every 8 scans, and wrong
   closures between scans 16 apart) through tzr_register_cloud_pairs_multiway (GNC-TLS) and
   tzr_register_cloud_pairs_multiway_line_process: each call's median time, the largest pose error against the truth,
   and which closures each optimiser rejects (mask 0 / not kept).
2. The cap graph of tests/test_gpu_line_process.py::test_cap_1024_against_the_restatement (K = 1024, a chain with
   closures and two wrong ones): the call's median wall time, trials run and enqueued per pass, and the time of one
   enqueued trial (run or idle): the wall time less that of a call whose passes both stop at their start
   (min_right_term = 1e30, one idle trial per pass), over the remaining enqueued trials.
3. The numpy restatement's CPU time on that graph (--restatement, once).

The card's name and power limit are read in the same run.  usage: python scripts/line_process_probe.py [--reps 3]
[--restatement] [--out rows.json]"""
import argparse
import importlib
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
capi = importlib.import_module("teaser-plusplus_b200.capi")
mwp = importlib.import_module("multiway_probe")
ref = importlib.import_module("pose_graph_reference")
lpref = importlib.import_module("line_process_reference")
graphs = importlib.import_module("line_process_graphs")

R_CORR = 0.05


def cap_graph():
    extra = [(k + 37, k) for k in range(0, 980, 61)]
    return graphs.graph(47, 1024, extra, wrong=[(500, 3), (900, 450)], noise=0.002, points=(60, 120))


def enqueued(trials, cap=2000):
    """Trials a pass enqueues: chunks of 1, 2, 4, then 8 until one ends at or past its last trial."""
    end, chunk = 0, 1
    while True:
        end += min(chunk, cap - end)
        chunk = min(2 * chunk, 8)
        if end >= max(1, trials) or end >= cap:
            return end


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--scans", type=int, default=32)
    ap.add_argument("--n", type=int, default=2000)
    ap.add_argument("--restatement", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    card = mwp.card()
    print("card:", card, flush=True)
    ctx = capi.Context(0)
    rows = []
    # 1. the scan sequence under both optimisers
    clouds, gt = mwp.sequence(a.n, a.scans, 7)
    pairs = [(k, k + 1) for k in range(a.scans - 1)] + [(k, k - 2) for k in range(2, a.scans, 8)]
    wrong = []
    for k in range(16, a.scans, 7):
        wrong.append(len(pairs))
        pairs.append((k, k - 16))
    unc = [0 if d == s + 1 else 1 for s, d in pairs]
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=0, rotation_cost_threshold=1e-12)
    err = lambda P: float(max(np.linalg.norm(P[k][:3, 3] - gt[k][:3, 3]) for k in range(a.scans)))
    for opt in ("gnc_tls", "line_process"):
        t, got = mwp.median_time(lambda: ctx.register_multiway(clouds, pairs, prm, R_CORR, uncertain=unc,
                                                               optimizer=opt, **mwp.FLAGS), a.reps)
        mw, icp = got[7], got[6]
        keep = mw["mask"] if opt == "gnc_tls" else mw["kept"]
        edges = [p for p in range(len(pairs)) if icp[p]["transform"]["scale"] > 0]
        row = dict(part="sequence", optimizer=opt, scans=a.scans, n=a.n, pairs=len(pairs), edges=len(edges),
                   call_ms=1e3 * t, max_pose_err=err(mw["poses"]), wrong_closures=wrong,
                   not_refined=[p for p in range(len(pairs)) if p not in edges],
                   rejected=[p for p in edges if unc[p] and not keep[p]],
                   kept_closures=[p for p in edges if unc[p] and keep[p]], status=mw["status"])
        if opt == "line_process":
            row.update(trials=mw["trials"], iterations=mw["iterations"], stop_reason=mw["stop_reason"],
                       pruned=mw["pruned"])
        else:
            row.update(gnc_iterations=mw["iterations"], inner_iterations=mw["inner_iterations"])
        rows.append(row)
        print(json.dumps(row), flush=True)
    # 2. the cap graph
    gt_c, edges, T, L, unc_c = cap_graph()
    t, got = mwp.median_time(lambda: ctx.global_optimization(1024, edges, T, L, R_CORR, uncertain=unc_c), a.reps)
    trials = sum(got["trials"])
    enq = sum(enqueued(x) for x in got["trials"])
    # a call whose passes both stop at their start enqueues one trial per pass, which runs idle: the rest of the wall
    # time over the rest of the enqueued trials is what one trial costs at this size
    t_idle, idle = mwp.median_time(lambda: ctx.global_optimization(1024, edges, T, L, R_CORR, uncertain=unc_c,
                                                                   min_right_term=1e30), a.reps)
    assert idle["trials"] == [0, 0]
    row = dict(part="cap", K=1024, E=len(edges), wall_ms=1e3 * t, trials=got["trials"], iterations=got["iterations"],
               stop_reason=got["stop_reason"], pruned=got["pruned"], trials_enqueued=enq,
               start_stop_call_ms=1e3 * t_idle,
               ms_per_enqueued_trial=1e3 * (t - t_idle) / max(enq - 2, 1))
    if a.restatement:
        t0 = time.perf_counter()
        want = lpref.optimize(1024, edges, T, L, R_CORR, unc_c)
        row.update(restatement_s=time.perf_counter() - t0,
                   restatement_max_pose_diff=float(np.abs(want["poses"] - got["poses"]).max()))
    rows.append(row)
    print(json.dumps(row), flush=True)
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(dict(card=card, rows=rows), fh)
    ctx.close()


if __name__ == "__main__":
    main()
