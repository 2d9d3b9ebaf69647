"""Coloured ICP on the card this runs on (DESIGN.md §3.17).

  python scripts/icp_colored_probe.py [--reps 5]

Rows, every time the median over the repetitions on the host clock after one warm-up call: one pair of 200 000-point
coloured scans; 256 pairs of 5000-point coloured scans, coloured ICP against point-to-plane on the same pairs
(alternating); and Open3D's tutorial schedule (voxel 0.04 / 0.02 / 0.01, 50 / 30 / 14 iterations, radius 2 voxel for the
normals and 1.5 voxel for the correspondences) on a synthetic coloured scan pair of 400 000 points: voxel downsampling
with colours, normals and coloured ICP at each scale, each stage's median time over the repetitions (after a warm-up
run) and the error against the truth.  Prints the card's name and power limit first.
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import icp_plane_probe as base  # noqa: E402

capi, R_CORR, RN, CENTRE = base.capi, base.R_CORR, base.RN, base.CENTRE


def texture(p):
    """A smooth colour field over the surface's (x, y) in [0, 1]."""
    x, y = p[:, 0] - CENTRE[0], p[:, 1] - CENTRE[1]
    a = 0.5 + 0.4 * np.sin(9.0 * x) * np.cos(7.0 * y)
    b = 0.5 + 0.4 * np.cos(5.0 * x + 3.0 * y)
    return np.stack([a, b, 0.5 * (a + b)], axis=1).astype(np.float32)


def coloured_pair(rng, ns, nd):
    src, dst, init, R, t = base.scan_pair(rng, ns, nd)
    back = (dst.astype(np.float64) - t) @ R  # the target's points in the source frame: one texture on both
    return src, dst, texture(src.astype(np.float64)), texture(back), init, R, t


def timed(fn, reps):
    out = fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts)), out


def voxel_colours(ctx, pts, cols, v):
    """Voxel means of the points and their colours in one device call (tzr_voxel_downsample_colors)."""
    t0 = time.perf_counter()
    out, c = ctx.voxel_downsample(pts, v, colors=cols)
    return out, c, (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    print(f"card: {q.stdout.strip()}")
    ctx = capi.Context(0)
    rng = np.random.default_rng(0)

    src, dst, sc, dc, init, R, t = coloured_pair(rng, 200000, 200000)
    dn = ctx.estimate_normals(dst, 0.03)
    ms_g, _ = timed(lambda: ctx.estimate_color_gradients(dst, dn, dc, 2 * 0.02), a.reps)
    ms, (res, _) = timed(lambda: ctx.icp_colored_batch([src], [dst], [dn], [sc], [dc], 0.02, [init]), a.reps)
    print(f"one pair 200000x200000, r = 0.02, normals r 0.03: gradients alone {ms_g:.2f} ms")
    print(base.summary("coloured", ms, res, [(R, t)]))

    pairs = [coloured_pair(rng, 5000, 5000) for _ in range(256)]
    S, D, SC, DC, I = ([p[k] for p in pairs] for k in range(5))
    truth = [(p[5], p[6]) for p in pairs]
    ND = ctx.estimate_normals_batch(D, RN)
    rows = base.alternate([lambda: ctx.icp_point_to_plane_batch(S, D, ND, R_CORR, I),
                           lambda: ctx.icp_colored_batch(S, D, ND, SC, DC, R_CORR, I)], a.reps)
    print(f"256 pairs 5000x5000, r = {R_CORR}, max_iteration 30, lambda 0.968:")
    for name, (ms, (res, _)) in zip(("point-to-plane", "coloured"), rows):
        print(base.summary(name, ms, res, truth))

    src, dst, sc, dc, init, R, t = coloured_pair(rng, 400000, 400000)
    print("tutorial schedule on 400000x400000 (voxel with colours, normals r = 2 v, coloured ICP r = 1.5 v), "
          f"median of {a.reps} runs after a warm-up run:")
    sched = [(0.04, 50), (0.02, 30), (0.01, 14)]

    def schedule():
        T = dict(scale=1.0, rotation=np.asarray(init["rotation"]), translation=np.asarray(init["translation"]))
        rows = []
        for v, iters in sched:
            s_d, s_c, s_vox = voxel_colours(ctx, src, sc, v)
            d_d, d_c, d_vox = voxel_colours(ctx, dst, dc, v)
            t1 = time.perf_counter()
            nrm = ctx.estimate_normals(d_d, 2 * v)
            t2 = time.perf_counter()
            res, _ = ctx.icp_colored(s_d, d_d, nrm, s_c, d_c, 1.5 * v, init=T, max_iteration=iters)
            t3 = time.perf_counter()
            T = dict(scale=1.0, rotation=res["R"], translation=res["t"])
            rot = np.degrees(np.arccos(np.clip((np.trace(res["R"] @ R.T) - 1) / 2, -1, 1)))
            tr = np.linalg.norm((res["R"] @ CENTRE + res["t"]) - (R @ CENTRE + t))
            rows.append((len(s_d), len(d_d), s_vox + d_vox, (t2 - t1) * 1e3, (t3 - t2) * 1e3, res["iterations"],
                         res["fitness"], rot, tr))
        return rows

    schedule()
    runs = [schedule() for _ in range(a.reps)]
    for k, (v, _) in enumerate(sched):
        r = [run[k] for run in runs]
        med = lambda j: float(np.median([x[j] for x in r]))  # noqa: E731
        ns, nd, _, _, _, it, fit, rot, tr = r[-1]
        print(f"  voxel {v}: {ns} / {nd} points; voxel with colours {med(2):.2f} ms, normals {med(3):.2f} ms, "
              f"coloured ICP {med(4):.2f} ms ({it} iterations, fitness {fit:.3f}); error {rot:.4f} deg {tr:.2e}")
    tot = [sum(x[2] + x[3] + x[4] for x in run) for run in runs]
    print(f"  schedule total (stages summed) median {float(np.median(tot)):.1f} ms")
    ctx.close()


if __name__ == "__main__":
    main()
