"""Multiway registration of a scan sequence: tzr_register_cloud_pairs_multiway against the chain of public calls
(register_cloud_pairs_icp point-to-plane -> information_matrix_batch -> optimize_pose_graph), in the same run.

The scans are the wavy-surface sequence of scripts/register_pairs_probe.py (every scan a moved copy of the one before,
2/3 of its points kept).  Edges: odometry (k, k + 1), loop closures (k, k - 2) every 8 scans, and a few deliberately
wrong closures between scans 16 apart, which barely overlap: a record there is made of coincidental matches, and the
pose graph has to reject it.  Reports the chained call's
time against the chain, the information-matrix and pose-graph times on their own, the pose error against ground truth
for odometry composition and for the optimised graph, which wrong closures were rejected, and the card's name and power
limit, read in the same run, and every pair's error against the truth (the source scan's centroid moved by the refined
transform against the true one).  Each time is the median of --reps calls after a warm-up call.

usage: python scripts/multiway_probe.py [--scans 32] [--n 2000] [--reps 3] [--out rows.json]"""
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
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
capi = importlib.import_module("teaser-plusplus_b200.capi")
rpp = importlib.import_module("register_pairs_probe")
ref = importlib.import_module("pose_graph_reference")

R_CORR = 0.05
FLAGS = dict(normal_search_radius=0.1, fpfh_search_radius=0.15, use_absolute_scale=False, use_crosscheck=True,
             use_tuple_test=False)


def sequence(n, scans, seed):
    """The sequence topology of register_pairs_probe.clouds_of, step for step, with each step's motion kept: scan k + 1
    is scan k with 2/3 of its points kept, moved by (R_k, (0.05, 0, 0)).  Returns the clouds and the ground-truth poses
    T_k (scan k into the frame of scan 0)."""
    clouds = [rpp.fbp.make_pair(n, seed)[0]]
    poses = [np.eye(4)]
    for k in range(scans - 1):
        rng = np.random.default_rng(seed + 1 + k)
        src = clouds[-1].astype(np.float64)
        keep = n - n // 3
        dst = np.concatenate([src[:keep], rpp.fbp.surface(rng, n - keep)])[rng.permutation(n)]
        a = rng.normal(size=3)
        a *= 0.05 / np.linalg.norm(a)
        K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
        R = np.eye(3) + np.sin(0.05) * K / 0.05 + (1 - np.cos(0.05)) * (K @ K) / 0.05 ** 2
        clouds.append((dst @ R.T + np.array([0.05, 0.0, 0.0])).astype(np.float32))
        step = np.eye(4)
        step[:3, :3], step[:3, 3] = R, [0.05, 0.0, 0.0]
        poses.append(poses[-1] @ ref.inv(step))
    return clouds, poses


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"unknown ({e})"


def median_time(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=32)
    ap.add_argument("--n", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    print("card:", card(), flush=True)
    clouds, gt = sequence(a.n, a.scans, 7)
    assert all(np.array_equal(x, y) for x, y in zip(clouds, rpp.clouds_of(a.n, a.scans - 1, "sequence", 7)[0]))
    # loop closures every 8 scans, between scans two apart ((2/3)^2 of their points shared)
    pairs = [(k, k + 1) for k in range(a.scans - 1)] + [(k, k - 2) for k in range(2, a.scans, 8)]
    # wrong closures: scans 16 apart barely overlap ((2/3)^16 of their points), so a valid record there is made of
    # coincidental matches
    wrong = []
    for k in range(16, a.scans, 7):
        wrong.append(len(pairs))
        pairs.append((k, k - 16))
    unc = [0 if d == s + 1 else 1 for s, d in pairs]
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=0, rotation_cost_threshold=1e-12)
    ctx = capi.Context(0)
    t_one, got = median_time(lambda: ctx.register_multiway(clouds, pairs, prm, R_CORR, uncertain=unc, **FLAGS),
                             a.reps)
    mw = got[7]

    def chain():
        res = ctx.register_cloud_pairs_icp(clouds, pairs, prm, R_CORR, method="point_to_plane", **FLAGS)
        icp = res[6]
        refined = [p for p in range(len(pairs)) if icp[p]["transform"]["scale"] > 0]
        trs = [dict(scale=float(icp[p]["transform"]["scale"]), rotation=icp[p]["transform"]["rotation"],
                    translation=icp[p]["transform"]["translation"]) for p in refined]
        L, _n = ctx.information_matrix_batch([clouds[pairs[p][0]] for p in refined],
                                             [clouds[pairs[p][1]] for p in refined], trs, R_CORR)
        pg = ctx.optimize_pose_graph(len(clouds), [pairs[p] for p in refined], trs, L, R_CORR,
                                     uncertain=[unc[p] for p in refined])
        return refined, trs, L, pg

    t_chain, (refined, trs, L, pg) = median_time(chain, a.reps)
    same = mw["poses"].tobytes() == pg["poses"].tobytes()
    t_info, _ = median_time(lambda: ctx.information_matrix_batch([clouds[pairs[p][0]] for p in refined],
                                                                 [clouds[pairs[p][1]] for p in refined], trs, R_CORR),
                            a.reps)
    t_pg, _ = median_time(lambda: ctx.optimize_pose_graph(len(clouds), [pairs[p] for p in refined], trs, L, R_CORR,
                                                          uncertain=[unc[p] for p in refined]), a.reps)
    # odometry composition: the refined odometry transforms chained from scan 0
    icp = got[6]
    odo = [np.eye(4)]
    for k in range(a.scans - 1):
        tr = icp[k]["transform"]
        T = np.eye(4)
        T[:3, :3] = np.asarray(tr["rotation"]).reshape(3, 3).T
        T[:3, 3] = tr["translation"]
        odo.append(odo[-1] @ ref.inv(T))
    err = lambda P: float(max(np.linalg.norm(P[k][:3, 3] - gt[k][:3, 3]) for k in range(a.scans)))
    # each refined pair's transform against the truth T_d^-1 T_s (translation error of the source scan's centroid)
    sols = got[0]
    pair_err = []
    for p, (s_, d_) in enumerate(pairs):
        tr = icp[p]["transform"]
        T = np.eye(4)
        T[:3, :3] = np.asarray(tr["rotation"]).reshape(3, 3).T
        T[:3, 3] = tr["translation"]
        c = np.append(clouds[s_].astype(np.float64).mean(axis=0), 1.0)
        truth = ref.inv(gt[d_]) @ gt[s_]
        pair_err.append(float(np.linalg.norm((T @ c - truth @ c)[:3])) if tr["scale"] > 0 else None)
    row = dict(scans=a.scans, n=a.n, pairs=len(pairs), edges=len(refined), one_call_ms=1e3 * t_one,
               chain_ms=1e3 * t_chain, information_ms=1e3 * t_info, pose_graph_ms=1e3 * t_pg,
               outputs_identical=bool(same), odometry_max_err=err(odo), optimised_max_err=err(mw["poses"]),
               wrong_closures=wrong, wrong_rejected=[bool(not mw["mask"][p]) for p in wrong],
               correct_closures_kept=bool(all(mw["mask"][p] for p in range(len(pairs))
                                              if unc[p] and p not in wrong and icp[p]["transform"]["scale"] > 0)),
               gnc_iterations=mw["iterations"], inner_iterations=mw["inner_iterations"], status=mw["status"],
               pair_valid=[int(x) for x in sols["valid"]], pair_err=pair_err,
               weights=[float(x) for x in mw["weights"]])
    print(json.dumps(row), flush=True)
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(dict(card=card(), rows=[row]), fh)
    ctx.close()


if __name__ == "__main__":
    main()
