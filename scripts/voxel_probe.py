"""Voxel-grid downsampling on the device (tzr_voxel_downsample(_batch), DESIGN.md §3.12): medians after warm-up, on the
host clock around synchronous calls.

Rows: one 300k-point scan at v = 0.05; batches of B = 16 and 256 scans of 50k-300k points; host baselines for each row
(the numpy reference and an np.unique downsampler, timed on a few clouds and scaled to the row's points); the cost of
composing voxel_downsample_batch with register_cloud_pairs_icp (each call's time and the bytes of the downsampled
clouds' re-upload); a voxel-size sweep over one scan (the per-voxel sequential sum's cost as points per voxel grow).

usage: python scripts/voxel_probe.py [--reps 5]
"""
import argparse
import importlib
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
capi = importlib.import_module("teaser-plusplus_b200.capi")
import voxel_reference as ref  # noqa: E402


def surface(rng, n, offset=(0.5, -0.2, 2.0)):
    uv = rng.uniform(-1, 1, size=(n, 2))
    z = 0.3 * np.sin(3 * uv[:, 0]) * np.cos(2 * uv[:, 1]) + 0.25 * np.exp(-((uv[:, 0] - 0.3) ** 2 + (uv[:, 1] + 0.4) ** 2) / 0.05)
    pts = np.stack([uv[:, 0], uv[:, 1], z], axis=1)
    return (pts + rng.normal(scale=0.003, size=pts.shape) + np.asarray(offset)).astype(np.float32)


def unique_downsample(pts, v):
    """A typical host downsampler: np.unique over the voxel triples, then per-voxel means (bincount)."""
    p = pts.astype(np.float64)
    p = p[np.isfinite(p).all(axis=1)]
    vmin = p.min(axis=0) - v * 0.5
    ijk = np.floor((p - vmin) / v).astype(np.int64)
    _, inv, cnt = np.unique(ijk, axis=0, return_inverse=True, return_counts=True)
    inv = inv.ravel()
    return (np.stack([np.bincount(inv, weights=p[:, k]) for k in range(3)], axis=1) / cnt[:, None]).astype(np.float32)


def median_ms(fn, reps, warmup=2):
    for _ in range(warmup):
        fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(t)


def host_ms_per_point(clouds, v):
    """Median host time per point of the numpy reference and the np.unique downsampler over a few clouds."""
    r, u = [], []
    for c in clouds:
        t0 = time.perf_counter()
        ref.downsample(c, v)
        r.append((time.perf_counter() - t0) * 1e3 / len(c))
        t0 = time.perf_counter()
        unique_downsample(c, v)
        u.append((time.perf_counter() - t0) * 1e3 / len(c))
    return statistics.median(r), statistics.median(u)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    print("card:", q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown")
    ctx = capi.Context(0)
    rng = np.random.default_rng(0)
    v = 0.05
    pool = [surface(rng, n) for n in np.linspace(50000, 300000, 16).astype(int)]
    host_few = pool[::5]
    ref_pp, uniq_pp = host_ms_per_point(host_few, v)

    one = surface(rng, 300000)
    out = ctx.voxel_downsample(one, v)
    assert out.tobytes() == ref.downsample(one, v)[0].tobytes()
    ms = median_ms(lambda: ctx.voxel_downsample(one, v), args.reps)
    print(f"single 300000 pts v={v}: {ms:.2f} ms on the device ({len(out)} voxels); host reference "
          f"{ref_pp * 300000:.1f} ms, np.unique {uniq_pp * 300000:.1f} ms")

    for B in (16, 256):
        clouds = [pool[k % len(pool)] for k in range(B)]
        npts = sum(len(c) for c in clouds)
        outs = ctx.voxel_downsample_batch(clouds, v)
        for k in range(0, B, max(1, B // 4)):
            assert outs[k].tobytes() == ctx.voxel_downsample(clouds[k], v).tobytes()
        ms = median_ms(lambda: ctx.voxel_downsample_batch(clouds, v), args.reps)
        print(f"batch B={B} ({npts} pts, {sum(len(o) for o in outs)} voxels): {ms:.2f} ms on the device; host reference "
              f"{ref_pp * npts / 1e3:.2f} s, np.unique {uniq_pp * npts / 1e3:.2f} s (scaled from {len(host_few)} clouds)")

    # composing the two calls: raw scans -> downsampled clouds (read back) -> register_cloud_pairs_icp (uploaded again)
    for P in (16, 128):
        raw = [pool[k % len(pool)] for k in range(2 * P)]
        down = ctx.voxel_downsample_batch(raw, v)
        pairs = [(2 * p, 2 * p + 1) for p in range(P)]
        prm = capi.default_params(noise_bound=v, estimate_scaling=0, rotation_cost_threshold=1e-12)
        kw = dict(normal_search_radius=2 * v, fpfh_search_radius=5 * v, use_absolute_scale=False, use_crosscheck=True,
                  use_tuple_test=False)
        t_down = median_ms(lambda: ctx.voxel_downsample_batch(raw, v), args.reps, warmup=1)
        t_reg = median_ms(lambda: ctx.register_cloud_pairs_icp(down, pairs, prm, v, **kw), args.reps, warmup=1)
        up = sum(d.nbytes for d in down)
        print(f"compose P={P} pairs ({sum(len(r) for r in raw)} raw pts -> {sum(len(d) for d in down)}): "
              f"voxel_downsample_batch {t_down:.2f} ms + register_cloud_pairs_icp {t_reg:.2f} ms; "
              f"re-upload of the downsampled clouds {up} bytes ({up / 1e6:.2f} MB)")

    # voxel-size sweep on one scan: points per voxel grow, each voxel's sum is one thread's sequential loop
    for vs in (0.005, 0.02, 0.05, 0.2, 1.0, 10.0):
        o, tr = ctx.voxel_downsample(one, vs, return_trace=True)
        per = np.bincount(tr[tr >= 0])
        ms = median_ms(lambda: ctx.voxel_downsample(one, vs), args.reps)
        print(f"sweep v={vs}: {len(o)} voxels, mean {per.mean():.1f} / max {per.max()} points per voxel: {ms:.2f} ms")
    ctx.close()


if __name__ == "__main__":
    main()
