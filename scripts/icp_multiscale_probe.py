"""Multi-scale ICP in one call against the chain of public calls (DESIGN.md §3.19), on the card this runs on.

  python scripts/icp_multiscale_probe.py [--reps 5]

Prints the card's name and power limit, then two rows, each the median over the repetitions on the host clock after
one warm-up call of each variant, the variants called in turn, and each call's records compared with the chain's bit for
bit (the probe stops if they differ):
  (a) Open3D's coloured-ICP tutorial schedule (voxel 0.04 / 0.02 / 0.01, 50 / 30 / 14 iterations, normals at 2 voxel,
      correspondences at 1.5 voxel) on icp_colored_probe's 400 000-point coloured pair: tzr_icp_multiscale_batch
      against voxel_downsample_colors_batch, estimate_normals_batch and icp_colored_batch scale by scale;
  (b) the reconstruction system's point-to-plane schedule (voxel v, v/2, v/4 with v = 0.04, distance 1.4 voxel, normals
      at 2 voxel, 50 / 30 / 14 iterations) on 64 pairs of 100 000-point scans: one call against voxel_downsample_batch,
      estimate_normals_batch and icp_point_to_plane_batch scale by scale.
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import icp_colored_probe as cp  # noqa: E402

base, capi = cp.base, cp.capi


def chain(ctx, method, scales, clouds, pairs, inits, colors=None):
    """The public calls scale by scale: (P, S) records."""
    P, S = len(pairs), len(scales)
    rec = np.zeros((P, S), dtype=capi.ICP_RESULT_DTYPE)
    poses = list(inits)
    for s, sc in enumerate(scales):
        if colors is not None:
            pts, cols = ctx.voxel_downsample_batch(clouds, sc.voxel_size, colors=colors)
        else:
            pts, cols = ctx.voxel_downsample_batch(clouds, sc.voxel_size), None
        nrm = ctx.estimate_normals_batch(pts, sc.normal_search_radius)
        kw = dict(max_iteration=sc.max_iteration, relative_fitness=sc.relative_fitness, relative_rmse=sc.relative_rmse)
        src, dst = [pts[a] for a, _ in pairs], [pts[b] for _, b in pairs]
        dn = [nrm[b] for _, b in pairs]
        if method == "colored":
            res, _ = ctx.icp_colored_batch(src, dst, dn, [cols[a] for a, _ in pairs], [cols[b] for _, b in pairs],
                                           sc.max_correspondence_distance, poses, **kw)
        else:
            res, _ = ctx.icp_point_to_plane_batch(src, dst, dn, sc.max_correspondence_distance, poses, **kw)
        rec[:, s] = res
        poses = [r["transform"] for r in res]
    return rec


def compare(name, ctx, reps, method, scales, clouds, pairs, inits, colors=None):
    one = lambda: ctx.icp_multiscale(clouds, pairs, scales, inits, method=method, colors=colors)[0]  # noqa: E731
    ref = lambda: chain(ctx, method, scales, clouds, pairs, inits, colors)  # noqa: E731
    fns = [one, ref]
    outs = [fn() for fn in fns]
    ts = [[] for _ in fns]
    for _ in range(reps):
        for k, fn in enumerate(fns):
            ctx.synchronize()
            t0 = time.perf_counter()
            outs[k] = fn()
            ts[k].append((time.perf_counter() - t0) * 1e3)
        if outs[0].tobytes() != outs[1].tobytes():
            sys.exit(f"{name}: the call's records differ from the chain's")
    l0 = ctx.kernel_launches()
    one()
    l1 = ctx.kernel_launches()
    ref()
    l2 = ctx.kernel_launches()
    ms = [float(np.median(t)) for t in ts]
    last = outs[0][:, -1]
    print(f"{name}: one call {ms[0]:.1f} ms ({l1 - l0} launches), chain {ms[1]:.1f} ms ({l2 - l1} launches), "
          f"ratio {ms[1] / ms[0]:.2f}; records bit-identical; last scale: median fitness "
          f"{float(np.median(last['fitness'])):.3f}, median iterations {float(np.median(last['iterations'])):.0f}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    print(f"card: {q.stdout.strip()}")
    ctx = capi.Context(0)
    rng = np.random.default_rng(0)
    cp.coloured_pair(rng, 200000, 200000)  # icp_colored_probe's draws before its 400 000-point pair
    [cp.coloured_pair(rng, 5000, 5000) for _ in range(256)]
    src, dst, sc, dc, init, _, _ = cp.coloured_pair(rng, 400000, 400000)
    tut = [capi.icp_scale(dict(voxel_size=v, max_correspondence_distance=1.5 * v, max_iteration=it))
           for v, it in ((0.04, 50), (0.02, 30), (0.01, 14))]
    compare("(a) tutorial schedule, 1 coloured pair 400000x400000", ctx, a.reps, "colored", tut, [src, dst], [(0, 1)],
            [init], [sc, dc])
    clouds, pairs, inits = [], [], []
    for k in range(64):
        s, d, i, _, _ = base.scan_pair(rng, 100000, 100000)
        clouds += [s, d]
        pairs.append((2 * k, 2 * k + 1))
        inits.append(i)
    v = 0.04
    rec = [capi.icp_scale(dict(voxel_size=x, max_correspondence_distance=1.4 * x, max_iteration=it))
           for x, it in ((v, 50), (v / 2, 30), (v / 4, 14))]
    compare("(b) reconstruction schedule, point-to-plane, 64 pairs 100000x100000", ctx, a.reps, "point_to_plane", rec,
            clouds, pairs, inits)
    ctx.close()


if __name__ == "__main__":
    main()
