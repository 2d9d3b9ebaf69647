"""Times ragged batches of the solve: size classes against the one-call-per-size behaviour they replace.

Workload: C2 geometry (95 % outliers, fixed scale) and a C2scale-like unknown-scale variant (80 % outliers, target
scaled by 1.5), n drawn uniformly from [500, 5000] with all sizes distinct, for each B of --bs (unknown scale: the
first B only).  Per workload and variant, one JSON line with the card name and power limit read in the same run: the
median wall time of --reps calls that end in a synchronisation (after one warm-up call), the kernel launches of one
call (tzr_ctx_kernel_launches), the device memory in use after it, and for the host variants the problems whose record
differs from the first tzr_solve_batch call's.  Variants:
  per_size        one tzr_solve_batch call per distinct n (what a ragged batch cost before size classes)
  host_r1.41      tzr_solve_batch, size classes at r = sqrt(2) (the default)
  host_r2         tzr_solve_batch, r = 2 (TZR_RAGGED_RATIO)
  host_one_class  tzr_solve_batch under debug flag 16777216 (one padded class)
  dev_r1.41       tzr_solve_batch_ragged_dev on flat device tensors
  uniform_floor   tzr_solve_batch on B problems of one size with the same sum of n^2
Writes nothing.

    python scripts/ragged_batch_probe.py [--bs 64 256 1024] [--reps 3]
"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
capi = importlib.import_module("teaser-plusplus_b200.capi")
synth = importlib.import_module("teaser-plusplus_b200.synth")
ONE_CLASS = 16777216


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    name, pl = out[0].split(", ")
    return name, pl


def workload(B, unknown_scale):
    sizes = np.random.default_rng(B).choice(np.arange(500, 5001), size=B, replace=False)
    probs = []
    for b, n in enumerate(sizes):
        pr = synth.config_problem("C2scale" if unknown_scale else "C2", b, n=int(n))
        probs.append((pr["src"], 1.5 * pr["dst"] if unknown_scale else pr["dst"]))
    return probs


def differing(sols, ref):
    """Problems whose record differs from the first call's, with the fields that differ and the reference's proof code
    (2 = maximum size proven after the first search pass's deadline: which maximum clique is found depends on timing)."""
    out = []
    for b in range(len(ref)):
        if sols[b:b + 1].tobytes() != ref[b:b + 1].tobytes():
            fields = [f for f in ref.dtype.names if sols[b][f].tobytes() != ref[b][f].tobytes()]
            out.append(dict(b=b, fields=fields, proven=int(ref[b]["clique_proven_optimal"])))
    return out


def timed(ctx, fn, reps):
    fn()
    ts, launches = [], 0
    for _ in range(reps):
        l0 = ctx.kernel_launches()
        t0 = time.perf_counter()
        fn()
        ctx.synchronize()
        ts.append(time.perf_counter() - t0)
        launches = ctx.kernel_launches() - l0
    return float(np.median(ts)) * 1e3, launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bs", type=int, nargs="+", default=[64, 256, 1024])
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    import torch
    name, pl = card()
    ctx = capi.Context(0)
    for unknown_scale in (False, True):
        for B in (a.bs[:1] if unknown_scale else a.bs):
            probs = workload(B, unknown_scale)
            prm = capi.default_params(noise_bound=synth.NOISE_BOUND_SIGMA_001, estimate_scaling=int(unknown_scale))
            srcs, dsts = [p[0] for p in probs], [p[1] for p in probs]
            ns = np.array([len(s) for s in srcs], dtype=np.int32)
            ref, _ = ctx.solve_batch(srcs, dsts, prm)

            def per_size():
                for b in range(B):
                    ctx.solve_batch(srcs[b:b + 1], dsts[b:b + 1], prm)

            diffs = []

            def host(ratio, flags=0):
                def f():
                    os.environ["TZR_RAGGED_RATIO"] = str(ratio)
                    ctx.set_flags(flags)
                    sols, _ = ctx.solve_batch(srcs, dsts, prm)
                    ctx.set_flags(0)
                    os.environ.pop("TZR_RAGGED_RATIO")
                    diffs[:] = differing(sols, ref)
                return f

            src_t = torch.from_numpy(np.concatenate(srcs)).cuda()
            dst_t = torch.from_numpy(np.concatenate(dsts)).cuda()
            sol_t = torch.zeros(B * capi.SOLUTION_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
            clq_t = torch.zeros(int(ns.sum()), dtype=torch.int32, device="cuda")

            def dev():
                ctx.solve_batch_ragged_dev(prm, ns, src_t.data_ptr(), dst_t.data_ptr(), sol_t.data_ptr(),
                                           clq_t.data_ptr())

            nu = int(round(np.sqrt(np.mean(ns.astype(np.float64) ** 2))))
            uni = [synth.config_problem("C2scale" if unknown_scale else "C2", b, n=nu) for b in range(B)]
            us = np.ascontiguousarray(np.stack([u["src"] for u in uni]))
            ud = np.ascontiguousarray(np.stack([1.5 * u["dst"] if unknown_scale else u["dst"] for u in uni]))

            def floor():
                ctx.solve_batch_array(us, ud, prm)

            for variant, fn in (("per_size", per_size), ("host_r1.41", host(2 ** 0.5)), ("host_r2", host(2.0)),
                                ("host_one_class", host(2 ** 0.5, ONE_CLASS)), ("dev_r1.41", dev),
                                ("uniform_floor", floor)):
                diffs.clear()
                ms, launches = timed(ctx, fn, a.reps)
                free, total = torch.cuda.mem_get_info()
                print(json.dumps(dict(card=name, power_limit=pl, workload="C2scale-like" if unknown_scale else "C2",
                                      B=B, n_min=int(ns.min()), n_max=int(ns.max()), variant=variant,
                                      median_ms=round(ms, 2), launches=int(launches),
                                      device_bytes_in_use=int(total - free), reps=a.reps,
                                      differs_from_first_call=diffs[:8])), flush=True)
            del src_t, dst_t, sol_t, clq_t
    ctx.close()


if __name__ == "__main__":
    main()
