"""Split the solve's step time by kernel: every kernel of a tzr_solve_batch_dev step, plus the idle gaps between them.

For each config, one batch of the benchmark's synthetic problems is built and solved `--warmup` times; then `--steps`
back-to-back solves run under torch.profiler with CUDA activities (a run of their own: the end-to-end numbers come from
bench.py with the profiler off).  The device timeline of those steps is read from the profiler's trace, and one table
per config is printed: per kernel name its launches and ms per step, the device-idle gaps between consecutive device
activities (ms per step), and the span from the first activity to the last.  One JSON line per config follows the
table, with the card's name, power limit and SM clocks read in the same run.  There is no CPU fallback: without a GPU
the script fails.

    python scripts/step_kernel_probe.py --configs C2,C4,C3 --steps 10 --warmup 3 [--out DIR]
"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import tempfile
from collections import defaultdict

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# name: (n, batch) as bench.py runs them on one GPU
SHAPES = {"C2": (5000, 1024), "C2cube": (5000, 256), "C3": (10000, 32), "C4": (2000, 4096), "C5": (8000, 256)}
DEVICE_CATS = ("kernel", "gpu_memset", "gpu_memcpy")


def card():
    import torch
    info = {"device": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit_sm_clock_max_sm_clock"] = q
    except (OSError, subprocess.SubprocessError):
        info["power_limit_sm_clock_max_sm_clock"] = None
    return info


def device_timeline(trace_path):
    """(name, start_us, dur_us) of every kernel, memset and copy in a chrome trace, in start order."""
    with open(trace_path) as fh:
        tr = json.load(fh)
    ev = [(e["name"], float(e["ts"]), float(e["dur"])) for e in tr.get("traceEvents", [])
          if e.get("ph") == "X" and e.get("cat") in DEVICE_CATS]
    ev.sort(key=lambda e: e[1])
    return ev


def short(name):
    """Kernel name without its namespace, template arguments and parameter list."""
    base = name.replace("(anonymous namespace)::", "").split("(")[0]
    if "<" in base:
        base = base[:base.index("<")]
    base = base.split("::")[-1].strip()
    return base.replace("void ", "") or name


def summarise(ev, steps):
    per = defaultdict(lambda: [0, 0.0])
    gaps = 0.0
    end = None
    for name, ts, dur in ev:
        p = per[short(name)]
        p[0] += 1
        p[1] += dur
        if end is not None and ts > end:
            gaps += ts - end
        end = ts + dur if end is None else max(end, ts + dur)
    span = (end - ev[0][1]) if ev else 0.0
    rows = sorted(((k, v[0] / steps, v[1] / steps / 1000.0) for k, v in per.items()), key=lambda r: -r[2])
    return rows, gaps / steps / 1000.0, span / steps / 1000.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="C2,C4,C3")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--flags", type=int, default=0)
    ap.add_argument("--out", default=None, help="directory for the traces and the JSON lines (default: a temporary one)")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    if not torch.cuda.is_available():
        raise SystemExit("step_kernel_probe.py: no CUDA device — this probe has no CPU fallback")
    capi = importlib.import_module("teaser-plusplus_b200.capi")
    synth = importlib.import_module("teaser-plusplus_b200.synth")
    out = args.out or tempfile.mkdtemp(prefix="step_kernel_probe_")
    os.makedirs(out, exist_ok=True)
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
        clq_d = torch.zeros((B, n), dtype=torch.int32, device="cuda")
        params = capi.default_params(noise_bound=nb, cbar2=1.0, estimate_scaling=0, rotation_estimation_algorithm=0,
                                     rotation_gnc_factor=1.4, rotation_max_iterations=100, rotation_cost_threshold=1e-12,
                                     rotation_tim_graph=0, inlier_selection_mode=0)
        ctx = capi.Context(0)
        ctx.set_flags(args.flags)
        stream = torch.cuda.Stream()
        ctx.set_stream(stream.cuda_stream)

        def step():
            ctx.solve_batch_dev(params, B, n, src_d.data_ptr(), dst_d.data_ptr(), sol_d.data_ptr(), clq_d.data_ptr())

        for _ in range(args.warmup):
            step()
        ctx.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                step()
            ctx.synchronize()
        trace = os.path.join(out, f"step_{cfg}.pt.trace.json")
        prof.export_chrome_trace(trace)
        ctx.close()
        rows, gap_ms, span_ms = summarise(device_timeline(trace), args.steps)
        busy = sum(r[2] for r in rows)
        print(f"== {cfg}: n={n} batch={B}, {args.steps} steps; {hw['device']}, "
              f"power limit / SM clock / max SM clock: {hw['power_limit_sm_clock_max_sm_clock']}")
        print(f"{'kernel':<34}{'launches/step':>14}{'ms/step':>10}")
        for name, cnt, ms in rows:
            print(f"{name:<34}{cnt:>14.1f}{ms:>10.3f}")
        print(f"{'(device busy)':<34}{'':>14}{busy:>10.3f}")
        print(f"{'(gaps between activities)':<34}{'':>14}{gap_ms:>10.3f}")
        print(f"{'(span first..last activity)':<34}{'':>14}{span_ms:>10.3f}", flush=True)
        line = {"config": cfg, "n": n, "batch": B, "steps": args.steps, "flags": args.flags,
                "kernels": [{"name": r[0], "launches_per_step": r[1], "ms_per_step": r[2]} for r in rows],
                "busy_ms_per_step": busy, "gap_ms_per_step": gap_ms, "span_ms_per_step": span_ms, **hw}
        print(json.dumps(line), flush=True)
        with open(os.path.join(out, "step_kernel_probe.jsonl"), "a") as fh:
            fh.write(json.dumps(line) + "\n")
        del src_d, dst_d, sol_d, clq_d
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
