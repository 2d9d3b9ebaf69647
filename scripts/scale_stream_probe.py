"""Times the unknown-scale stage's regenerating route at n in {5000, 16384, 33000, 46340, 65536}.

The stage's time is the difference between the median wall time of a device-resident solve (tzr_solve_batch_dev,
synchronised) with estimate_scaling = 1 and the same solve with the scale fixed, over --reps timed calls after one
warm-up call each.  Prints one JSON line per n with the card name and power limit read in the same run, the chunk count
(tzr_ctx_last_scale_chunks), the passes over all TIMs that chunk count implies (12 boundary-selection histograms and one
counting pass per 32 chunks per sweep when there is more than one chunk, one generating pass per chunk per sweep), the
device memory the stage added to a fresh context (torch.cuda.mem_get_info) and the estimate.  Writes nothing.

    python scripts/scale_stream_probe.py [--reps 3] [--sizes 5000,65536]
"""
import argparse
import importlib
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
capi = importlib.import_module("teaser-plusplus_b200.capi")
synth = importlib.import_module("teaser-plusplus_b200.synth")


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    name, pl = out[0].split(", ")
    return name, pl


def passes(chunks):
    if chunks <= 1:
        return 2
    windows = -(-chunks // 32)
    return 12 + (windows if chunks <= 32 else 2 * windows) + 2 * chunks


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sizes", default="5000,16384,33000,46340,65536")
    a = ap.parse_args()
    import torch
    name, pl = card()
    s = 1.7
    for n in [int(v) for v in a.sizes.split(",")]:
        pr = synth.make_problem(n, 0.80, 300 + n, "ball", sigma=0.01, noise_bound=synth.NOISE_BOUND_SIGMA_001)
        src = torch.tensor(pr["src"][None], device="cuda")
        dst = torch.tensor((pr["dst"] * s)[None], device="cuda")
        sols = torch.zeros((1, capi.SOLUTION_DTYPE.itemsize), dtype=torch.uint8, device="cuda")
        ctx = capi.Context(0, max_n=65536)
        times, mem = {}, {}
        try:
            for est in (0, 1):
                p = capi.default_params(noise_bound=pr["noise_bound"] * s, estimate_scaling=est)
                torch.cuda.synchronize()
                free0, _ = torch.cuda.mem_get_info()
                ts = []
                for r in range(a.reps + 1):
                    t0 = time.perf_counter()
                    ctx.solve_batch_dev(p, 1, n, src.data_ptr(), dst.data_ptr(), sols.data_ptr())
                    ctx.synchronize()
                    ts.append(time.perf_counter() - t0)
                    if r == 0:
                        mem[est] = free0 - torch.cuda.mem_get_info()[0]
                times[est] = statistics.median(ts[1:]) * 1e3
            chunks = ctx.last_scale_chunks()
        finally:
            ctx.close()
        rec = np.frombuffer(sols.cpu().numpy().tobytes(), dtype=capi.SOLUTION_DTYPE)[0]
        print(json.dumps(dict(card=name, power_limit=pl, n=n, tims=n * (n - 1) // 2, chunks=chunks,
                              passes=passes(chunks), scale_stage_ms=round(times[1] - times[0], 2),
                              solve_ms=round(times[1], 2), fixed_scale_solve_ms=round(times[0], 2),
                              stage_bytes=int(mem[1]), scale=float(rec["scale"]), valid=bool(rec["valid"]))),
              flush=True)


if __name__ == "__main__":
    main()
