"""Timing of tzr_icp_batch (DESIGN.md §3.11): medians after warm-up, on the card this runs on.

  python scripts/icp_probe.py [--reps 5] [--host-pairs 4]

Rows: icp_batch at B = 1, 16 and 256 pairs of 5000-point scans against B single calls and against the numpy/cKDTree
loop on the host's cores (timed on --host-pairs pairs and scaled to B); one dense pair of 200 000 points a side; both
nearest-neighbour routes across target sizes (where the route switch comes from).  Prints the card's name and power
limit first, then one line per row: ms per call, iterations, launches per call.
"""
import argparse
import importlib
import os
import subprocess
import sys
import time

import numpy as np
from scipy.spatial import cKDTree
from scipy.spatial.transform import Rotation

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
capi = importlib.import_module("teaser-plusplus_b200.capi")
R_CORR = 0.05


def scan_pair(rng, ns, nd):
    def surface(n):
        uv = rng.uniform(-1, 1, size=(n, 2))
        p = np.stack([uv[:, 0], uv[:, 1], 0.3 * np.sin(3 * uv[:, 0]) * np.cos(2 * uv[:, 1])], axis=1)
        return p + rng.normal(scale=0.003, size=p.shape) + [0.5, -0.2, 2.0]
    src = surface(ns)
    keep = min(ns, nd - nd // 3)
    pts = np.concatenate([src[:keep], surface(nd - keep)])[rng.permutation(nd)]
    R = Rotation.from_rotvec(rng.normal(size=3) * 0.03).as_matrix()
    t = rng.normal(size=3) * 0.02
    dst = pts @ R.T + t
    dR = Rotation.from_rotvec(rng.normal(size=3) * 0.03).as_matrix()
    init = dict(scale=1.0, rotation=dR @ R, translation=t + rng.normal(size=3) * 0.05)
    return src.astype(np.float32), dst.astype(np.float32), init


def host_icp(src, dst, init, max_iteration=30):
    """Open3D-style point-to-point ICP on the host: cKDTree nearest neighbour on every core, numpy Kabsch."""
    tree = cKDTree(dst.astype(np.float64))
    x = src.astype(np.float64)
    R, t = np.asarray(init["rotation"]), np.asarray(init["translation"])
    prev = None
    it = 0
    for it in range(max_iteration + 1):
        p = x @ R.T + t
        d, j = tree.query(p, k=1, distance_upper_bound=R_CORR, workers=-1)
        m = np.isfinite(d)
        cur = (m.mean(), np.sqrt((d[m] ** 2).mean()) if m.any() else 0.0)
        if prev is not None and abs(cur[0] - prev[0]) < 1e-6 and abs(cur[1] - prev[1]) < 1e-6:
            break
        prev = cur
        if it == max_iteration:
            break
        P, Q = p[m], dst[j[m]].astype(np.float64)
        mp, mq = P.mean(0), Q.mean(0)
        U, _, Vt = np.linalg.svd((P - mp).T @ (Q - mq))
        V = Vt.T
        if np.linalg.det(U) * np.linalg.det(V) < 0:
            V[:, 2] *= -1
        Ru = V @ U.T
        R, t = Ru @ R, Ru @ t + mq - Ru @ mp
    return it


def timed(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts)), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-pairs", type=int, default=4)
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    print(f"card: {q.stdout.strip()}")
    ctx = capi.Context(0)
    rng = np.random.default_rng(0)
    pairs = [scan_pair(rng, 5000, 5000) for _ in range(256)]
    for B in (1, 16, 256):
        S, D, I = [p[0] for p in pairs[:B]], [p[1] for p in pairs[:B]], [p[2] for p in pairs[:B]]
        l0 = ctx.kernel_launches()
        ms, (res, _) = timed(lambda: ctx.icp_batch(S, D, R_CORR, I), a.reps)
        launches = (ctx.kernel_launches() - l0) // (a.reps + 1)
        ms1, _ = timed(lambda: [ctx.icp_batch([s], [d], R_CORR, [i]) for s, d, i in zip(S, D, I)], max(1, a.reps // 2))
        k = min(B, a.host_pairs)
        t0 = time.perf_counter()
        for s, d, i in zip(S[:k], D[:k], I[:k]):
            host_icp(s, d, i)
        host = (time.perf_counter() - t0) * 1e3 / k * B
        it = res["iterations"]
        print(f"icp_batch B={B:3d} 5000x5000: {ms:9.2f} ms  ({ms / B:.3f} ms/pair)  B single calls {ms1:9.2f} ms  "
              f"host cKDTree {host:9.1f} ms  iterations median {int(np.median(it))} max {int(it.max())}  "
              f"launches/call {launches}")
    src, dst, init = scan_pair(rng, 200000, 200000)
    ms, (res, _) = timed(lambda: ctx.icp_batch([src], [dst], R_CORR, [init]), max(1, a.reps // 2))
    t0 = time.perf_counter()
    host_icp(src, dst, init)
    host = (time.perf_counter() - t0) * 1e3
    print(f"dense pair 200000x200000: {ms:9.2f} ms  host cKDTree {host:9.1f} ms  iterations {int(res[0]['iterations'])}")
    for nd in (256, 512, 1024, 2048, 4096, 8192):
        S, D, I = zip(*[scan_pair(rng, nd, nd) for _ in range(64)])
        row = []
        for name, flag in (("brute", capi.FLAG_ICP_BRUTE_FORCE), ("grid", capi.FLAG_ICP_GRID)):
            ctx.set_flags(flag)
            ms, (res, _) = timed(lambda: ctx.icp_batch(list(S), list(D), R_CORR, list(I), max_iteration=10,
                                                        relative_fitness=0, relative_rmse=0), a.reps)
            row.append(f"{name} {ms:8.2f} ms")
        ctx.set_flags(0)
        print(f"route B=64 n={nd:5d} 10 iterations: " + "  ".join(row))
    # the chained entry against register_cloud_pairs followed by icp_batch over the valid solved pairs
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=0, rotation_cost_threshold=1e-12)
    flags = dict(normal_search_radius=0.1, fpfh_search_radius=0.15, use_absolute_scale=False, use_crosscheck=True,
                 use_tuple_test=False)
    for P in (16, 256):
        clouds = [p[0] for p in pairs[:P]] + [p[1] for p in pairs[:P]]
        cp = [(k, P + k) for k in range(P)]

        def chain():
            s = ctx.register_cloud_pairs(clouds, cp, prm, **flags)
            ok = [k for k in range(P) if s[1][k] == 0 and s[0][k]["valid"]]
            seeds = [dict(scale=s[0][k]["scale"], rotation=s[0][k]["rotation"], translation=s[0][k]["translation"])
                     for k in ok]
            return ctx.icp_batch([clouds[k] for k in ok], [clouds[P + k] for k in ok], R_CORR, seeds)

        ms_chain, _ = timed(chain, a.reps)
        l0 = ctx.kernel_launches()
        ms_one, out = timed(lambda: ctx.register_cloud_pairs_icp(clouds, cp, prm, R_CORR, **flags), a.reps)
        launches = (ctx.kernel_launches() - l0) // (a.reps + 1)
        it = out[6]["iterations"]
        print(f"register_cloud_pairs_icp P={P:3d} 5000x5000: {ms_one:9.2f} ms  register_cloud_pairs + icp_batch "
              f"{ms_chain:9.2f} ms  iterations median {int(np.median(it))}  launches/call {launches}")
    ctx.close()


if __name__ == "__main__":
    main()
