"""Break the graph stage down by kernel at the benchmark's batch shapes, for two flag settings alternated in one process.

For each config, one batch of the benchmark's synthetic problems is built once.  Then, `--rounds` times and for each of
`--flags` in turn, the batch is solved `--warmup` times and then `--steps` times under torch.profiler (CUDA activities).
Each kernel's and memset's device time per step is printed as one JSON line per (config, round, flags), next to the
graph stage's own CUDA-event time from a separate unprofiled pass of the same steps, and with the card's name and power
limit.  Writes nothing unless `--out` names a file (the JSON lines are appended to it).

    python scripts/graph_kernel_probe.py --configs C2,C4,C5 --flags 0,134217728 --rounds 3
"""
import argparse
import collections
import importlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
probe = importlib.import_module("graph_stage_probe")


def kernel_name(name):
    """'void tzr::graph_strip2_kernel<false, 6, true, true>(tzr::Batch)' -> 'graph_strip2_kernel<false, 6, true, true>'."""
    name = name.replace("void ", "").split("(")[0]
    return name.replace("tzr::", "")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="C2,C4,C5")
    ap.add_argument("--flags", default="0,134217728")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    capi = importlib.import_module("teaser-plusplus_b200.capi")
    synth = importlib.import_module("teaser-plusplus_b200.synth")
    hw = probe.card()
    flags_list = [int(f) for f in args.flags.split(",")]
    for cfg in args.configs.split(","):
        n, B = probe.SHAPES[cfg]
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
        stream = torch.cuda.Stream()
        ctx.set_stream(stream.cuda_stream)

        def step():
            ctx.solve_batch_dev(params, B, n, src_d.data_ptr(), dst_d.data_ptr(), sol_d.data_ptr())

        for rnd in range(args.rounds):
            for flags in flags_list:
                ctx.set_flags(flags)
                for _ in range(args.warmup):
                    step()
                ctx.synchronize()
                ctx.stage_log(True)  # graph stage by the library's own events, profiler off
                for _ in range(args.steps):
                    step()
                ctx.synchronize()
                stage, calls = ctx.stage_log_read()
                ctx.stage_log(False)
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(args.steps):
                        step()
                    ctx.synchronize()
                per = collections.defaultdict(float)
                for e in prof.events():
                    if e.device_type.name == "CUDA":  # device activity: kernels, memsets, copies
                        per[kernel_name(e.name)] += e.time_range.elapsed_us() / 1000.0 / args.steps
                graph_kernels = {k: v for k, v in per.items()
                                 if k.startswith(("graph_strip", "tc_patch", "Memset", "Memcpy", "graph_tc", "edge_count",
                                                  "degree_kernel", "prep_kernel"))}
                line = {"config": cfg, "n": n, "batch": B, "round": rnd, "flags": flags, "steps": args.steps,
                        "graph_stage_ms_per_step": stage["graph"] / max(calls, 1),
                        "prep_stage_ms_per_step": stage["prep"] / max(calls, 1),
                        "kernels_ms_per_step": dict(sorted(graph_kernels.items(), key=lambda kv: -kv[1])),
                        "all_device_ms_per_step": sum(per.values()), **hw}
                print(json.dumps(line), flush=True)
                if args.out:
                    with open(args.out, "a") as fh:
                        fh.write(json.dumps(line) + "\n")
        ctx.set_flags(0)
        ctx.close()
        del src_d, dst_d, sol_d
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
