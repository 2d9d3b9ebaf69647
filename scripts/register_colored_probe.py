"""Coloured ICP inside the chained calls on the card this runs on (DESIGN.md §3.18).

  python scripts/register_colored_probe.py [--reps 3] [--pairs 256] [--n 5000] [--scans 32]

Rows, every time the median over --reps calls after one warm-up call, the variants alternating:
  - --pairs pairs of --n-point coloured scans (icp_colored_probe's coloured_pair: one texture on both scans of a pair):
    the chained coloured call (register_cloud_pairs_icp(method="colored")) against the chained point-to-plane call and
    against the public chain it stands for (register_cloud_pairs, estimate_normals_batch, icp_colored_batch), with the
    median error of the refined pairs against the truth;
  - multiway_probe's scan sequence (--scans scans of 2000 points, loop closures and wrong closures), coloured from one
    texture in the frame of scan 0: coloured multiway (register_multiway(colors=...)) against point-to-plane multiway,
    with the largest pose error against the truth.
Prints the card's name and power limit first."""
import argparse
import importlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
icp_colored_probe = importlib.import_module("icp_colored_probe")
multiway_probe = importlib.import_module("multiway_probe")
base = icp_colored_probe.base
capi = base.capi

R_CORR = 0.05
FLAGS = multiway_probe.FLAGS


def pair_errors(icp, truth):
    """Rotation (degrees) and translation errors of the refined records against the truth (R, t)."""
    rot, tr = [], []
    for rec, (R, t) in zip(icp, truth):
        if rec["transform"]["scale"] <= 0:
            continue
        Rg = np.asarray(rec["transform"]["rotation"]).reshape(3, 3).T
        c = np.clip((np.trace(Rg.T @ R) - 1) / 2, -1, 1)
        rot.append(np.degrees(np.arccos(c)))
        tr.append(np.linalg.norm(np.asarray(rec["transform"]["translation"]) - t))
    return len(rot), float(np.median(rot)), float(np.median(tr))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--pairs", type=int, default=256)
    ap.add_argument("--n", type=int, default=5000)
    ap.add_argument("--scans", type=int, default=32)
    a = ap.parse_args()
    print("card:", multiway_probe.card(), flush=True)
    ctx = capi.Context(0)
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=0, rotation_cost_threshold=1e-12)

    rng = np.random.default_rng(0)
    clouds, cols, truth = [], [], []
    for _ in range(a.pairs):
        src, dst, sc, dc, _init, R, t = icp_colored_probe.coloured_pair(rng, a.n, a.n)
        clouds += [src.astype(np.float32), dst.astype(np.float32)]
        cols += [sc, dc]
        truth.append((R, t))
    pairs = [(2 * p, 2 * p + 1) for p in range(a.pairs)]

    def public_chain():
        sols = ctx.register_cloud_pairs(clouds, pairs, prm, **FLAGS)[0]
        ok = [p for p in range(a.pairs) if sols[p]["valid"]]
        normals = ctx.estimate_normals_batch([clouds[2 * p + 1] for p in ok], FLAGS["normal_search_radius"])
        seeds = [dict(scale=sols[p]["scale"], rotation=sols[p]["rotation"], translation=sols[p]["translation"])
                 for p in ok]
        return ctx.icp_colored_batch([clouds[2 * p] for p in ok], [clouds[2 * p + 1] for p in ok], normals,
                                     [cols[2 * p] for p in ok], [cols[2 * p + 1] for p in ok], R_CORR, seeds)[0]

    rows = base.alternate([
        lambda: ctx.register_cloud_pairs_icp(clouds, pairs, prm, R_CORR, method="colored", colors=cols, **FLAGS),
        lambda: ctx.register_cloud_pairs_icp(clouds, pairs, prm, R_CORR, method="point_to_plane", **FLAGS),
        public_chain], a.reps)
    print(f"{a.pairs} pairs of {a.n}-point coloured scans, r = {R_CORR}, max_iteration 30, lambda 0.968:")
    for name, (ms, out) in zip(["chained coloured", "chained point-to-plane"], rows[:2]):
        k, rot, tr = pair_errors(out[6], truth)
        print(f"  {name:24s} {ms:9.1f} ms  refined {k}  error median {rot:.4f} deg {tr:.2e}")
    print(f"  {'public chain (coloured)':24s} {rows[2][0]:9.1f} ms")

    seq, gt = multiway_probe.sequence(2000, a.scans, 7)
    # one texture in the frame of scan 0: the point of scan k at p sits at gt[k] p there
    scols = [icp_colored_probe.texture(c.astype(np.float64) @ g[:3, :3].T + g[:3, 3]) for c, g in zip(seq, gt)]
    spairs = [(k, k + 1) for k in range(a.scans - 1)] + [(k, k - 2) for k in range(2, a.scans, 8)]
    spairs += [(k, k - 16) for k in range(16, a.scans, 7)]
    unc = [0 if d == s + 1 else 1 for s, d in spairs]
    mrows = base.alternate([
        lambda: ctx.register_multiway(seq, spairs, prm, R_CORR, uncertain=unc, colors=scols, **FLAGS),
        lambda: ctx.register_multiway(seq, spairs, prm, R_CORR, uncertain=unc, **FLAGS)], a.reps)
    print(f"multiway: {a.scans} scans of 2000 points, {len(spairs)} pairs, r = {R_CORR}:")
    for name, (ms, out) in zip(["coloured multiway", "point-to-plane multiway"], mrows):
        mw = out[7]
        err = max(np.linalg.norm(mw["poses"][k][:3, 3] - gt[k][:3, 3]) for k in range(a.scans))
        print(f"  {name:24s} {ms:9.1f} ms  pose graph status {mw['status']}  largest pose error {err:.2e}")
    ctx.close()


if __name__ == "__main__":
    main()
