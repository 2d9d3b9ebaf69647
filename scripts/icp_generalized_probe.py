"""Generalized ICP against point-to-plane and point-to-point ICP on identical inputs (DESIGN.md §3.14), on the card
this runs on.

  python scripts/icp_generalized_probe.py [--reps 5]

The workloads and columns are scripts/icp_plane_probe.py's: the three methods run alternately, one call each per
repetition, after one warm-up call each, and every time is the median over the repetitions on the host clock.  Rows:
256 pairs of 5000-point scans from perturbed seeds (ms per call, median and largest iteration count, share converged,
median final rmse, median rotation and translation error against ground truth); one pair of 200 000-point scans; the
three chained entries (register_cloud_pairs_icp) on 128 pairs.  Prints the card's name and power limit first.
"""
import argparse
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import icp_plane_probe as base  # noqa: E402

capi, R_CORR, RN = base.capi, base.R_CORR, base.RN


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--epsilon", type=float, default=1e-3)
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    print(f"card: {q.stdout.strip()}")
    ctx = capi.Context(0)
    rng = np.random.default_rng(0)
    pairs = [base.scan_pair(rng, 5000, 5000) for _ in range(256)]
    S, D, I = [p[0] for p in pairs], [p[1] for p in pairs], [p[2] for p in pairs]
    truth = [(p[3], p[4]) for p in pairs]
    NS, ND = ctx.estimate_normals_batch(S, RN), ctx.estimate_normals_batch(D, RN)
    rows = alternate3(a.reps,
                      lambda: ctx.icp_generalized_batch(S, D, NS, ND, R_CORR, I, epsilon=a.epsilon),
                      lambda: ctx.icp_point_to_plane_batch(S, D, ND, R_CORR, I),
                      lambda: ctx.icp_batch(S, D, R_CORR, I))
    print(f"256 pairs 5000x5000, r = {R_CORR}, max_iteration 30, epsilon {a.epsilon}:")
    for name, (ms, (res, _)) in rows:
        print(base.summary(name, ms, res, truth))
    src, dst, init, R, t = base.scan_pair(rng, 200000, 200000)
    sn, dn = ctx.estimate_normals(src, 0.03), ctx.estimate_normals(dst, 0.03)
    rows = alternate3(max(1, a.reps // 2),
                      lambda: ctx.icp_generalized_batch([src], [dst], [sn], [dn], R_CORR, [init], epsilon=a.epsilon),
                      lambda: ctx.icp_point_to_plane_batch([src], [dst], [dn], R_CORR, [init]),
                      lambda: ctx.icp_batch([src], [dst], R_CORR, [init]))
    print("one pair 200000x200000 (normals at radius 0.03):")
    for name, (ms, (res, _)) in rows:
        print(base.summary(name, ms, res, [(R, t)]))
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=0, rotation_cost_threshold=1e-12)
    flags = dict(normal_search_radius=0.1, fpfh_search_radius=0.15, use_absolute_scale=False, use_crosscheck=True,
                 use_tuple_test=False)
    P = 128
    clouds = S[:P] + D[:P]
    cp = [(k, P + k) for k in range(P)]
    rows = alternate3(max(1, a.reps // 2),
                      lambda: ctx.register_cloud_pairs_icp(clouds, cp, prm, R_CORR, method="generalized",
                                                           epsilon=a.epsilon, **flags),
                      lambda: ctx.register_cloud_pairs_icp(clouds, cp, prm, R_CORR, method="point_to_plane", **flags),
                      lambda: ctx.register_cloud_pairs_icp(clouds, cp, prm, R_CORR, **flags))
    out = rows[0][1][1]
    ok = [k for k in range(P) if out[1][k] == 0 and out[0][k]["valid"]]
    print(f"register_cloud_pairs_icp, {P} pairs 5000x5000, radii 0.1 / 0.15 ({len(ok)} refined):")
    for name, (ms, res) in rows:
        print(base.summary(name, ms, res[6][ok], [truth[k] for k in ok]))
    ctx.close()


def alternate3(reps, gicp, plane, p2p):
    """base.alternate over the three methods, labelled."""
    return list(zip(("generalized", "point-to-plane", "point-to-point"), base.alternate([gicp, plane, p2p], reps)))


if __name__ == "__main__":
    main()
