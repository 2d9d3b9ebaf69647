"""Robust kernels against L2 for point-to-plane and generalized ICP on identical inputs (DESIGN.md §3.15), on the card
this runs on.

  python scripts/icp_robust_probe.py [--reps 5]

The workloads and columns are scripts/icp_plane_probe.py's: the compared calls run alternately, one call each per
repetition, after one warm-up call each, and every time is the median over the repetitions on the host clock.  Rows:
256 pairs of 5000-point scans from perturbed seeds, per method, L2 against Tukey; the same with exactly 4 iterations
for every problem (both convergence criteria 0), so that the calls differ only in their system pass (robust generalized
ICP adds a 3 x 3 Jacobi SVD per correspondence); one pair of 200 000-point scans; the chained entry
(register_cloud_pairs_icp) on 128 pairs, L2 against Tukey per method; the clutter fixture of
tests/icp_robust_reference.py (distance to the truth, L2 against Tukey).  Prints the card's name and power limit first.
"""
import argparse
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import icp_plane_probe as base  # noqa: E402

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import icp_robust_reference as rref  # noqa: E402

capi, R_CORR, RN = base.capi, base.R_CORR, base.RN
K_PLANE, K_GICP = 0.03, 0.6  # Tukey's k: a distance for point-to-plane, a whitened residual for generalized ICP


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
    eps = a.epsilon
    rows = labelled(("plane L2", "plane Tukey", "generalized L2", "generalized Tukey"), a.reps, [
        lambda: ctx.icp_point_to_plane_batch(S, D, ND, R_CORR, I),
        lambda: ctx.icp_point_to_plane_batch(S, D, ND, R_CORR, I, kernel=("tukey", K_PLANE)),
        lambda: ctx.icp_generalized_batch(S, D, NS, ND, R_CORR, I, epsilon=eps),
        lambda: ctx.icp_generalized_batch(S, D, NS, ND, R_CORR, I, epsilon=eps, kernel=("tukey", K_GICP))])
    print(f"256 pairs 5000x5000, r = {R_CORR}, max_iteration 30, epsilon {eps}, Tukey k {K_PLANE} / {K_GICP}:")
    for name, (ms, (res, _)) in rows:
        print(base.summary(name, ms, res, truth))
    fixed = dict(max_iteration=4, relative_fitness=0.0, relative_rmse=0.0)
    rows = labelled(("plane L2", "plane Tukey", "generalized L2", "generalized Tukey"), a.reps, [
        lambda: ctx.icp_point_to_plane_batch(S, D, ND, R_CORR, I, **fixed),
        lambda: ctx.icp_point_to_plane_batch(S, D, ND, R_CORR, I, kernel=("tukey", K_PLANE), **fixed),
        lambda: ctx.icp_generalized_batch(S, D, NS, ND, R_CORR, I, epsilon=eps, **fixed),
        lambda: ctx.icp_generalized_batch(S, D, NS, ND, R_CORR, I, epsilon=eps, kernel=("tukey", K_GICP), **fixed)])
    print("the same, exactly 4 iterations per problem (4 system passes per call):")
    for name, (ms, (res, _)) in rows:
        print(base.summary(name, ms, res, truth))
    src, dst, init, R, t = base.scan_pair(rng, 200000, 200000)
    sn, dn = ctx.estimate_normals(src, 0.03), ctx.estimate_normals(dst, 0.03)
    rows = labelled(("plane L2", "plane Tukey", "generalized L2", "generalized Tukey"), max(1, a.reps // 2), [
        lambda: ctx.icp_point_to_plane_batch([src], [dst], [dn], R_CORR, [init]),
        lambda: ctx.icp_point_to_plane_batch([src], [dst], [dn], R_CORR, [init], kernel=("tukey", K_PLANE)),
        lambda: ctx.icp_generalized_batch([src], [dst], [sn], [dn], R_CORR, [init], epsilon=eps),
        lambda: ctx.icp_generalized_batch([src], [dst], [sn], [dn], R_CORR, [init], epsilon=eps,
                                          kernel=("tukey", K_GICP))])
    print("one pair 200000x200000 (normals at radius 0.03):")
    for name, (ms, (res, _)) in rows:
        print(base.summary(name, ms, res, [(R, t)]))
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=0, rotation_cost_threshold=1e-12)
    flags = dict(normal_search_radius=0.1, fpfh_search_radius=0.15, use_absolute_scale=False, use_crosscheck=True,
                 use_tuple_test=False)
    P = 128
    clouds = S[:P] + D[:P]
    cp = [(k, P + k) for k in range(P)]
    chain = lambda method, kern: lambda: ctx.register_cloud_pairs_icp(  # noqa: E731
        clouds, cp, prm, R_CORR, method=method, epsilon=eps, kernel=kern, **flags)
    rows = labelled(("plane L2", "plane Tukey", "generalized L2", "generalized Tukey"), max(1, a.reps // 2), [
        chain("point_to_plane", None), chain("point_to_plane", ("tukey", K_PLANE)), chain("generalized", None),
        chain("generalized", ("tukey", K_GICP))])
    out = rows[0][1][1]
    ok = [k for k in range(P) if out[1][k] == 0 and out[0][k]["valid"]]
    print(f"register_cloud_pairs_icp, {P} pairs 5000x5000, radii 0.1 / 0.15 ({len(ok)} refined):")
    for name, (ms, res) in rows:
        print(base.summary(name, ms, res[6][ok], [truth[k] for k in ok]))
    f = rref.clutter_pair(0)
    seed = dict(scale=1.0, rotation=f["R0"], translation=f["t0"])
    err = lambda r: rref.pose_error(r["R"], r["t"], f["R"], f["t"])  # noqa: E731
    for method, k in (("point-to-plane", f["k_plane"]), ("generalized", f["k_gicp"])):
        out = []
        for kern in (None, ("tukey", k)):
            if method == "point-to-plane":
                r, _ = ctx.icp_point_to_plane(f["src"], f["dst"], f["dst_normals"], f["r"], init=seed, kernel=kern)
            else:
                r, _ = ctx.icp_generalized(f["src"], f["dst"], f["src_normals"], f["dst_normals"], f["r"], init=seed,
                                           kernel=kern)
            out.append((err(r), r["iterations"]))
        print(f"clutter fixture, {method}: seed {err(dict(R=f['R0'], t=f['t0'])):.3e}, L2 {out[0][0]:.3e} "
              f"({out[0][1]} it), Tukey k {k} {out[1][0]:.3e} ({out[1][1]} it)")
    ctx.close()


def labelled(names, reps, fns):
    """base.alternate over the calls, labelled."""
    return list(zip(names, base.alternate(fns, reps)))


if __name__ == "__main__":
    main()
