"""Point-to-point against point-to-plane ICP on identical inputs (DESIGN.md §3.13), on the card this runs on.

  python scripts/icp_plane_probe.py [--reps 5]

The two methods run alternately, one call each per repetition, after one warm-up call each; every time is the median
over the repetitions, on the host clock.  Rows: 256 pairs of 5000-point scans from perturbed seeds (ms per call,
median and largest iteration count, share converged, median final rmse, median rotation and translation error against
ground truth); one pair of 200 000-point scans; estimate_normals_batch against compute_fpfh_batch on the 256 targets;
both chained entries (register_cloud_pairs_icp) on 128 pairs.  Prints the card's name and power limit first.
"""
import argparse
import importlib
import os
import subprocess
import sys
import time

import numpy as np
from scipy.spatial.transform import Rotation

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
capi = importlib.import_module("teaser-plusplus_b200.capi")
R_CORR = 0.05
RN = 0.15        # normal radius of the targets (about 25 neighbours at 5000 points)
CENTRE = np.array([0.5, -0.2, 2.0])


def scan_pair(rng, ns, nd):
    """Two scans of one wavy surface (2/3 shared points, noise 0.003), the target moved by a ground-truth (R, t), and a
    seed a few degrees and a few r away from it."""
    def surface(n):
        uv = rng.uniform(-1, 1, size=(n, 2))
        p = np.stack([uv[:, 0], uv[:, 1], 0.3 * np.sin(3 * uv[:, 0]) * np.cos(2 * uv[:, 1])], axis=1)
        return p + rng.normal(scale=0.003, size=p.shape) + CENTRE
    src = surface(ns)
    keep = min(ns, nd - nd // 3)
    pts = np.concatenate([src[:keep], surface(nd - keep)])[rng.permutation(nd)]
    R = Rotation.from_rotvec(rng.normal(size=3) * 0.03).as_matrix()
    t = CENTRE - R @ CENTRE + rng.normal(size=3) * 0.02
    dst = pts @ R.T + t
    dR = Rotation.from_rotvec(rng.normal(size=3) * 0.03).as_matrix()
    m = R @ CENTRE + t
    init = dict(scale=1.0, rotation=dR @ R, translation=dR @ (t - m) + m + rng.normal(size=3) * 0.05)
    return src.astype(np.float32), dst.astype(np.float32), init, R, t


def errors(res, truth):
    """Median rotation error (degrees) and translation error at the scans' centre over the problems."""
    rot, tr = [], []
    for r, (R, t) in zip(res, truth):
        d = capi.icp_result_dict(r)
        rot.append(np.degrees(Rotation.from_matrix(d["R"] @ R.T).magnitude()))
        tr.append(np.linalg.norm((d["R"] @ CENTRE + d["t"]) - (R @ CENTRE + t)))
    return float(np.median(rot)), float(np.median(tr))


def alternate(fns, reps):
    """One warm-up call of each, then reps rounds calling each once in turn: (median ms, last output) per function."""
    outs = [fn() for fn in fns]
    ts = [[] for _ in fns]
    for _ in range(reps):
        for k, fn in enumerate(fns):
            t0 = time.perf_counter()
            outs[k] = fn()
            ts[k].append((time.perf_counter() - t0) * 1e3)
    return [(float(np.median(t)), o) for t, o in zip(ts, outs)]


def summary(name, ms, res, truth, launches=None):
    it = res["iterations"]
    rot, tr = errors(res, truth)
    extra = f"  launches/call {launches}" if launches is not None else ""
    return (f"  {name:15s} {ms:9.2f} ms  iterations median {np.median(it):4.1f} max {int(it.max()):3d}  converged "
            f"{res['converged'].mean():6.1%}  rmse median {np.median(res['inlier_rmse']):.5f}  error median "
            f"{rot:.4f} deg {tr:.2e}{extra}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    print(f"card: {q.stdout.strip()}")
    ctx = capi.Context(0)
    rng = np.random.default_rng(0)
    pairs = [scan_pair(rng, 5000, 5000) for _ in range(256)]
    S, D, I = [p[0] for p in pairs], [p[1] for p in pairs], [p[2] for p in pairs]
    truth = [(p[3], p[4]) for p in pairs]
    N = ctx.estimate_normals_batch(D, RN)
    (ms_p, (res_p, _)), (ms_l, (res_l, _)) = alternate(
        [lambda: ctx.icp_batch(S, D, R_CORR, I), lambda: ctx.icp_point_to_plane_batch(S, D, N, R_CORR, I)], a.reps)
    print("256 pairs 5000x5000, r = 0.05, max_iteration 30:")
    print(summary("point-to-point", ms_p, res_p, truth))
    print(summary("point-to-plane", ms_l, res_l, truth))
    src, dst, init, R, t = scan_pair(rng, 200000, 200000)
    nrm = ctx.estimate_normals(dst, 0.03)
    (ms_p, (res_p, _)), (ms_l, (res_l, _)) = alternate(
        [lambda: ctx.icp_batch([src], [dst], R_CORR, [init]),
         lambda: ctx.icp_point_to_plane_batch([src], [dst], [nrm], R_CORR, [init])], max(1, a.reps // 2))
    print("one pair 200000x200000 (normals at radius 0.03):")
    print(summary("point-to-point", ms_p, res_p, [(R, t)]))
    print(summary("point-to-plane", ms_l, res_l, [(R, t)]))
    (ms_n, _), (ms_f, _) = alternate([lambda: ctx.estimate_normals_batch(D, RN),
                                      lambda: ctx.compute_fpfh_batch(D, RN, 2 * RN)], a.reps)
    print(f"normals of the 256 targets (radius {RN}): estimate_normals_batch {ms_n:9.2f} ms  compute_fpfh_batch "
          f"(fpfh radius {2 * RN}) {ms_f:9.2f} ms")
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=0, rotation_cost_threshold=1e-12)
    flags = dict(normal_search_radius=0.1, fpfh_search_radius=0.15, use_absolute_scale=False, use_crosscheck=True,
                 use_tuple_test=False)
    P = 128
    clouds = S[:P] + D[:P]
    cp = [(k, P + k) for k in range(P)]
    l0 = ctx.kernel_launches()
    (ms_p, out_p), (ms_l, out_l) = alternate(
        [lambda: ctx.register_cloud_pairs_icp(clouds, cp, prm, R_CORR, **flags),
         lambda: ctx.register_cloud_pairs_icp(clouds, cp, prm, R_CORR, method="point_to_plane", **flags)],
        max(1, a.reps // 2))
    launches = (ctx.kernel_launches() - l0) // (2 * (max(1, a.reps // 2) + 1))
    ok = [k for k in range(P) if out_p[1][k] == 0 and out_p[0][k]["valid"]]
    print(f"register_cloud_pairs_icp, {P} pairs 5000x5000, radii 0.1 / 0.15 ({len(ok)} refined), launches per call "
          f"(mean of both) {launches}:")
    print(summary("point-to-point", ms_p, out_p[6][ok], [truth[k] for k in ok]))
    print(summary("point-to-plane", ms_l, out_l[6][ok], [truth[k] for k in ok]))
    ctx.close()


if __name__ == "__main__":
    main()
