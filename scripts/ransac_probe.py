"""Correspondence RANSAC on the device (tzr_ransac_batch, DESIGN.md §3.21): timings, run on an H100.

(a) one tutorial-sized pair: 5000 matched rows, 100 000 iterations, confidence 0.999, edge length 0.9 and distance
    1.5 voxel: the time, the hypotheses drawn and passed, and the score kernel's FP64 rate from the shapes;
(b) 64 such problems in one ransac_batch call against 64 single calls;
(c) register_cloud_pairs_ransac on 64 pairs against the three public calls;
(d) for context, fgr_batch and the robust solve on the same rows.
The card and its power limit are read in the same run.  Usage: python scripts/ransac_probe.py
"""
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
capi = importlib.import_module("teaser-plusplus_b200.capi")

VOXEL = 0.05


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def problem(K, seed, outlier_rate=0.7):
    rng = np.random.default_rng(seed)
    x = rng.uniform(-1, 1, (K, 3)).astype(np.float32)
    a = 0.6
    R = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
    y = (x @ R.T + np.array([0.3, -0.1, 0.2]) + rng.normal(scale=0.005, size=x.shape)).astype(np.float32)
    j = np.arange(K)
    bad = rng.random(K) < outlier_rate
    j[bad] = rng.integers(0, K, int(bad.sum()))
    return x, y, np.stack([np.arange(K), j], axis=1).astype(np.int32)


def timed(f, reps=5):
    f()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = f()
        ts.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(ts)), out


def kernel_times(f):
    """Device time per RANSAC kernel (summed over its launches) of one call of f, after a warm-up call."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    f()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        f()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for k in ("ransac_prep_kernel", "ransac_hyp_kernel", "ransac_score_kernel", "ransac_select_kernel",
                  "ransac_seed_kernel"):
            if k in e.key:
                t = getattr(e, "device_time_total", None)
                if t is None:
                    t = e.cuda_time_total
                out.setdefault(k, dict(ms=0.0, launches=0))
                out[k]["ms"] += t / 1e3
                out[k]["launches"] += e.count
    return out


def main():
    ctx = capi.Context(0)
    out = {"card": card()}
    p = capi.ransac_params(1.5 * VOXEL, check_edge_length=1, edge_length_similarity=0.9, check_distance=1,
                           distance_threshold=1.5 * VOXEL)
    x, y, c = problem(5000, 1)
    ms, (res, info, _) = timed(lambda: ctx.ransac_batch([x], [y], [c], p, seeds=[1]))
    drawn, passed = int(info[0]["drawn"]), int(info[0]["passed"])
    out["a_one_pair"] = dict(ms=ms, drawn=drawn, passed=passed, fitness=float(res[0]["fitness"]))
    p_full = capi.ransac_params(1.5 * VOXEL, check_edge_length=1, check_distance=1, distance_threshold=1.5 * VOXEL,
                                confidence=1.0)
    ms_full, (_, info_f, _) = timed(lambda: ctx.ransac_batch([x], [y], [c], p_full, seeds=[1]), reps=3)
    out["a_all_100000"] = dict(ms=ms_full, drawn=int(info_f[0]["drawn"]), passed=int(info_f[0]["passed"]),
                               score_fp64_gflops_whole_call=int(info_f[0]["passed"]) * 5000 * 27 / (ms_full * 1e-3) / 1e9)
    # the score kernel's own device time (CUPTI through torch.profiler), and its rate from the shapes
    out["a_kernels"] = kernel_times(lambda: ctx.ransac_batch([x], [y], [c], p_full, seeds=[1]))
    sk = out["a_kernels"].get("ransac_score_kernel")
    if sk:
        out["a_all_100000"]["score_kernel_ms"] = sk["ms"]
        out["a_all_100000"]["score_fp64_gflops_kernel"] = int(info_f[0]["passed"]) * 5000 * 27 / (sk["ms"] * 1e-3) / 1e9
    probs = [problem(5000, s) for s in range(64)]
    ms_b, _ = timed(lambda: ctx.ransac_batch([q[0] for q in probs], [q[1] for q in probs], [q[2] for q in probs], p,
                                             seeds=list(range(64))), reps=3)
    ms_s, _ = timed(lambda: [ctx.ransac_batch([q[0]], [q[1]], [q[2]], p, seeds=[s]) for s, q in enumerate(probs)],
                    reps=3)
    out["b_64_problems"] = dict(batch_ms=ms_b, single_calls_ms=ms_s)
    from test_gpu_register_pairs import EXAMPLE, RF, RN, sequence
    clouds, pairs = sequence([5000] * 65, seed=5)
    pairs = pairs[:64]
    pc = capi.ransac_params(0.02, check_edge_length=1)
    ms_c, _ = timed(lambda: ctx.register_cloud_pairs_ransac(clouds, pairs, pc, RN, RF, *EXAMPLE), reps=3)

    def three():  # compute_fpfh_batch, match_correspondences_batch, ransac_batch on the pairs with rows
        feats = ctx.compute_fpfh_batch(clouds, RN, RF)
        m = ctx.match_correspondences_batch([clouds[a] for a, _ in pairs], [clouds[b] for _, b in pairs],
                                            [feats[a] for a, _ in pairs], [feats[b] for _, b in pairs], *EXAMPLE,
                                            tuple_seeds=[0] * len(pairs))
        reg = [q for q in range(len(pairs)) if len(m[q])]
        return ctx.ransac_batch([clouds[pairs[q][0]] for q in reg], [clouds[pairs[q][1]] for q in reg],
                                [m[q] for q in reg], pc)
    ms_3, _ = timed(three, reps=3)
    out["c_64_pairs"] = dict(chained_ms=ms_c, three_calls_ms=ms_3)
    fg = capi.fgr_params(maximum_correspondence_distance=1.5 * VOXEL)
    ms_f, _ = timed(lambda: ctx.fgr_batch([q[0] for q in probs], [q[1] for q in probs], [q[2] for q in probs], fgr=fg),
                    reps=3)
    src = [q[0][q[2][:, 0]].astype(np.float64) for q in probs[:8]]
    dst = [q[1][q[2][:, 1]].astype(np.float64) for q in probs[:8]]
    ms_t, _ = timed(lambda: [ctx.solve(s, d, capi.default_params(noise_bound=0.01, estimate_scaling=0))
                             for s, d in zip(src, dst)], reps=1)
    out["d_context"] = dict(fgr_64_ms=ms_f, robust_solve_8_single_ms=ms_t)
    print(json.dumps(out, indent=1))
    ctx.close()


if __name__ == "__main__":
    main()
