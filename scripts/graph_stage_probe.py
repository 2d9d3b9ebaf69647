"""Time the graph stage (graph_strip2_kernel + tc_patch_kernel) alone at the benchmark's batch shapes.

For each config, one batch of the benchmark's synthetic problems is built once, solved `--warmup` times, then `--steps`
times with the library's per-stage CUDA events on; the graph stage's mean time per call is printed as one JSON line, with
the card's name and power limit.  `--flags` sets the library's debug / A-B flags (as TZR_FLAGS does for bench.py).
Writes nothing unless `--out` names a file (the JSON lines are appended to it).

    python scripts/graph_stage_probe.py --configs C2,C4,C5 --steps 10 --warmup 2
"""
import argparse
import importlib
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# name: (n, batch) as bench.py runs them on one GPU
SHAPES = {"C2": (5000, 1024), "C2cube": (5000, 256), "C3": (10000, 32), "C4": (2000, 4096), "C5": (8000, 256)}


def card():
    import torch
    info = {"device": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit_and_max_sm_clock"] = q
    except (OSError, subprocess.SubprocessError):
        info["power_limit_and_max_sm_clock"] = None
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="C2,C4,C5")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--flags", type=int, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    capi = importlib.import_module("teaser-plusplus_b200.capi")
    synth = importlib.import_module("teaser-plusplus_b200.synth")
    hw = card()
    for cfg in args.configs.split(","):
        n, B = SHAPES[cfg]
        src = np.empty((B, n, 3))
        dst = np.empty((B, n, 3))
        nb = None
        for b in range(B):
            pr = synth.config_problem(cfg, b)
            src[b], dst[b], nb = pr["src"], pr["dst"], pr["noise_bound"]
        src_d = torch.from_numpy(src).cuda()
        dst_d = torch.from_numpy(dst).cuda()
        sol_d = torch.zeros(B * capi.SOLUTION_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
        params = capi.default_params(noise_bound=nb, cbar2=1.0, estimate_scaling=0, rotation_estimation_algorithm=0,
                                     rotation_gnc_factor=1.4, rotation_max_iterations=100, rotation_cost_threshold=1e-12,
                                     rotation_tim_graph=0, inlier_selection_mode=0)
        ctx = capi.Context(0)
        ctx.set_flags(args.flags)
        stream = torch.cuda.Stream()
        ctx.set_stream(stream.cuda_stream)

        def step():
            ctx.solve_batch_dev(params, B, n, src_d.data_ptr(), dst_d.data_ptr(), sol_d.data_ptr())

        for _ in range(args.warmup):
            step()
        ctx.synchronize()
        ctx.stage_log(True)
        for _ in range(args.steps):
            step()
        ctx.synchronize()
        stage, calls = ctx.stage_log_read()
        ctx.stage_log(False)
        ctx.close()
        line = {"config": cfg, "n": n, "batch": B, "flags": args.flags, "steps": calls,
                "graph_ms_per_call": stage["graph"] / max(calls, 1),
                "stage_ms_per_call": {k: v / max(calls, 1) for k, v in stage.items()}, **hw}
        print(json.dumps(line), flush=True)
        if args.out:
            with open(args.out, "a") as fh:
                fh.write(json.dumps(line) + "\n")
        del src_d, dst_d, sol_d
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
