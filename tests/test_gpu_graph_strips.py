"""GPU tests of graph_strip2_kernel's two strip lengths (`pytest -m gpu`).  launch_graph takes 6-block strips when every
CTA slot (6 per SM) has at least 512 blocks of 128 x 128 pairs to sweep and 4-block strips otherwise; single problems (the
other graph tests) only ever see the short ones.  Here a batch large enough for the long strips is built from a few
distinct problems, and the bitset, degrees and edge count of copies at both ends and in the middle of the batch are held
against the oracle, at sizes on both sides of a 128-block and of whole 6-block strips (n = 769: 7 blocks, n = 1000: 8), under the production
template, the verifying one (flag 2: zero disagreements) and a 64-entry re-check queue (flag 16384: in-place re-checks under
the column ring and the split-phase mirror barrier)."""
import importlib

import numpy as np
import pytest
import torch

import oracle_lib as orc
from test_gpu_graph_boundary import ctx  # noqa: F401 (fixture)

capi = importlib.import_module("teaser-plusplus_b200.capi")
synth = importlib.import_module("teaser-plusplus_b200.synth")

pytestmark = pytest.mark.gpu

DISTINCT = 3


def long_strip_batch(n):
    """smallest batch (a multiple of DISTINCT) that launch_graph sweeps in 6-block strips"""
    nt = (n + 127) // 128
    slots = torch.cuda.get_device_properties(0).multi_processor_count * 6
    per_problem = nt * (nt + 1) // 2
    B = -(-512 * slots // per_problem) + 1
    return -(-B // DISTINCT) * DISTINCT


@pytest.mark.parametrize("n", [769, 1000])
@pytest.mark.parametrize("flags", [0, 2 | 4, 16384])
def test_long_strips_match_oracle(ctx, n, flags):
    B = long_strip_batch(n)
    prs = [synth.config_problem("C2", 40 + k, n=n) for k in range(DISTINCT)]
    nb = prs[0]["noise_bound"]
    src = np.ascontiguousarray(np.stack([prs[b % DISTINCT]["src"] for b in range(B)]))
    dst = np.ascontiguousarray(np.stack([prs[b % DISTINCT]["dst"] for b in range(B)]))
    p = capi.default_params(noise_bound=nb, cbar2=1.0, estimate_scaling=0, rotation_cost_threshold=1e-12)
    # device-resident inputs: one launch of the graph kernel for the whole batch (host batches are fed in smaller chunks)
    src_d, dst_d = torch.from_numpy(src).cuda(), torch.from_numpy(dst).cuda()
    sol_d = torch.zeros(B * capi.SOLUTION_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    ctx.set_flags(flags)
    try:
        ctx.solve_batch_dev(p, B, n, src_d.data_ptr(), dst_d.data_ptr(), sol_d.data_ptr())
        ctx.synchronize()
        cnt = ctx.debug_counters()
    finally:
        ctx.set_flags(0)
    sols = np.frombuffer(sol_d.cpu().numpy().tobytes(), dtype=capi.SOLUTION_DTYPE)
    if flags & 2:
        assert cnt["filter_mismatches"] == 0
    want = [orc.build_graph_bits(pr["src"], pr["dst"], nb) for pr in prs]
    for b in [0, 1, 2, B // 2, B - 3, B - 2, B - 1]:
        obits, odeg, oe = want[b % DISTINCT]
        bits, deg = ctx.last_graph(b, n)
        assert np.array_equal(bits, obits), f"n={n} flags {flags} problem {b}: bitset differs"
        assert np.array_equal(deg, odeg), f"n={n} flags {flags} problem {b}: degrees differ"
        assert int(sols[b]["n_edges"]) == oe, f"n={n} flags {flags} problem {b}: edge count"
    ne = np.array([int(s["n_edges"]) for s in sols])
    assert np.array_equal(ne, np.array([want[b % DISTINCT][2] for b in range(B)])), "edge counts differ across the batch"
