"""GPU tests of graph_strip2_kernel's Gram-test schedule (`pytest -m gpu`) at the edges of its layout: the row sweep bounded
by the rows below n (rounded up to 4), column groups wholly past n left out of the sweep, and the mirror half of every
off-diagonal block gathered through a CTA-shared slice behind a barrier that every warp reaches, also the warps of the last
row block that have no rows.  The oracle's FP64 bitset, degrees and edge count are the checker, under the production
template (flag 0, fused degrees), the verifying template (flag 2: zero disagreements), the separate degree pass (flag 256)
and a 64-entry re-check queue (flag 16384)."""
import importlib

import numpy as np
import pytest

import oracle_lib as orc
from test_gpu_graph_boundary import N, NB, _mixed_batch, assert_graph, build, ctx, use_gram  # noqa: F401 (fixture)

capi = importlib.import_module("teaser-plusplus_b200.capi")
synth = importlib.import_module("teaser-plusplus_b200.synth")

pytestmark = pytest.mark.gpu

# 128-blocks, 32-row warps, 1-3 rows in the last block (129-131, 385-387), last warps without rows (161: warps 2 and 3 of
# the last block; 1331: warps 2 and 3), 1, 2 or 3 column groups in the last block (424, 454, 4999-5001)
SIZES = [1, 2, 3, 5, 31, 32, 33, 127, 128, 129, 130, 131, 161, 255, 256, 257, 385, 386, 387, 424, 454, 4999, 5000, 5001]
FLAGS = [0, 2 | 4, 256, 16384]


@pytest.mark.parametrize("n", SIZES)
def test_gram_schedule_matches_oracle(ctx, n):
    pr = synth.config_problem("C2", 11, n=n)
    src, dst, nb = pr["src"], pr["dst"], pr["noise_bound"]
    want = orc.build_graph_bits(src, dst, nb)
    if n >= 4999:
        assert use_gram(src, dst, nb)
    degs = {}
    for flags in FLAGS:
        got = build(ctx, src, dst, nb, flags)
        if flags & 2:
            assert got[3]["filter_mismatches"] == 0
            assert got[3]["gram_problems"] == use_gram(src, dst, nb)
        assert_graph(got, want, f"n={n} flags {flags}")
        degs[flags] = got[1]
    assert np.array_equal(degs[0], degs[256]), "fused degrees differ from the degree pass"


@pytest.mark.parametrize("n", [129, 387, 1000])
def test_many_undecided_pairs_across_mirror_blocks(ctx, n):
    """A guard-edge problem (~2 % of the pairs undecided): queued pairs and in-place re-checks (flag 16384) land in the
    mirror words that leave through the shared slice."""
    band = importlib.import_module("gram_band_check")
    src, dst, nb = band.guard_edge(1.02, 0.6, n=n, seed=n + 1)
    want = orc.build_graph_bits(src, dst, nb)
    for flags in FLAGS:
        got = build(ctx, src, dst, nb, flags)
        if flags & 2:
            assert got[3]["filter_mismatches"] == 0
        assert_graph(got, want, f"guard-edge n={n} flags {flags}")


@pytest.mark.parametrize("flags", [0, 256, 16384])
def test_mixed_batch_with_rowless_warps(ctx, flags):
    """Gram, interval and exact-path problems in one launch at n = 1331 (the last 128-block has 51 rows: warps 2 and 3 own
    none and still reach the block barriers)."""
    B = 16
    src, dst, gram = _mixed_batch(B, seed0=100)
    p = capi.default_params(noise_bound=NB, cbar2=1.0, estimate_scaling=0, rotation_cost_threshold=1e-12)
    ctx.set_flags(flags | 4)
    try:
        sols, _ = ctx.solve_batch_array(src, dst, p)
        cnt = ctx.debug_counters()
    finally:
        ctx.set_flags(0)
    assert cnt["gram_problems"] == gram
    for b in range(B):
        obits, odeg, oe = orc.build_graph_bits(src[b], dst[b], NB)
        bits, deg = ctx.last_graph(b, N)
        assert np.array_equal(bits, obits), f"problem {b}: bitset differs"
        assert np.array_equal(deg, odeg), f"problem {b}: degrees differ"
        assert int(sols[b]["n_edges"]) == oe, f"problem {b}: edge count"
