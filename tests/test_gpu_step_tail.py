"""The solve's work around the graph sweep at every batch shape (run on an H100: `pytest -m gpu`).

prep_kernel runs one cluster of CTAs per problem (boxes reduced across the cluster, constants on CTA 0); the small
route's heuristic and peel kernels switch to smaller CTAs once a batch fills the GPU with them; rot_trans_kernel is
built for eight CTAs per SM for large batches.  None of that may change a result:
  * a batch of 1, 63, 64, 65 or 1024 problems gives every problem the solution record (byte for byte, stage_ms aside)
    and clique that tzr_solve gives it alone; so does a ragged batch, in its own size classes and in one class;
  * a batch that mixes problems the uniqueness shortcut settles with problems that need the exact search gives each
    the clique it gets alone;
  * the filter constants prep_kernel writes equal the CPU copies of their formulas bit for bit;
  * a batch that mixes Gram-test, interval-test and exact-path problems builds each one's graph exactly (the
    oracle's bits, and no decided pair that disagrees with FP64 under debug flag 2), with debug counter 15 equal to
    the number of problems the CPU copy of the guard sends to the Gram test.
"""
import importlib
import os
import sys

import numpy as np
import pytest

import oracle_lib as orc

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))
import gram_band_check as band  # noqa: E402
import slope_band_check as slope  # noqa: E402
from test_gpu_graph_boundary import _guard_fixtures  # noqa: E402

capi = importlib.import_module("teaser-plusplus_b200.capi")
synth = importlib.import_module("teaser-plusplus_b200.synth")

pytestmark = pytest.mark.gpu

ONE_CLASS = 16777216
VERIFY = 2
COUNTERS = 4
STAGE_OFF = capi.SOLUTION_DTYPE.fields["stage_ms"][1]


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.set_flags(0)
    c.close()


def params(nb, **kw):
    d = dict(noise_bound=nb, cbar2=1.0, estimate_scaling=0, rotation_cost_threshold=1e-12)
    d.update(kw)
    return capi.default_params(**d)


def assert_alone(ctx, srcs, dsts, prm, sols, cliques):
    """Every problem of a batch against tzr_solve on it alone."""
    for b, (s, d) in enumerate(zip(srcs, dsts)):
        one = ctx.solve(s, d, prm)
        assert sols[b:b + 1].tobytes()[:STAGE_OFF] == bytes(one["sol"])[:STAGE_OFF], b
        assert np.array_equal(np.asarray(cliques[b]), one["clique"]), b


def c2_batch(B, n, seed0=0):
    prs = [synth.config_problem("C2", seed0 + b, n=n) for b in range(B)]
    return (np.stack([p["src"] for p in prs]), np.stack([p["dst"] for p in prs]), prs[0]["noise_bound"])


@pytest.mark.parametrize("B,n", [(1, 600), (63, 600), (64, 600), (65, 600), (1, 5000), (65, 5000), (1024, 600)])
def test_batch_sizes_give_the_single_solve(ctx, B, n):
    src, dst, nb = c2_batch(B, n)
    prm = params(nb)
    sols, cliques = ctx.solve_batch_array(src, dst, prm)
    assert sols["valid"].all()
    assert_alone(ctx, list(src), list(dst), prm, sols, [cliques[b, :sols[b]["clique_size"]] for b in range(B)])


@pytest.mark.parametrize("flags", [0, ONE_CLASS])
def test_ragged_batch_gives_the_single_solve(ctx, flags):
    # 300 problems: in one class (flag) the batch takes the small-CTA heuristic and peel kernels
    sizes = [(400, 700, 1000, 129, 3)[b % 5] for b in range(300)]
    prs = [synth.config_problem("C2", 500 + b, n=n) for b, n in enumerate(sizes)]
    nb = prs[0]["noise_bound"]
    prm = params(nb)
    ctx.set_flags(flags)
    try:
        sols, cliques = ctx.solve_batch([p["src"] for p in prs], [p["dst"] for p in prs], prm)
    finally:
        ctx.set_flags(0)
    assert_alone(ctx, [p["src"] for p in prs], [p["dst"] for p in prs], prm, sols, cliques)


def test_shortcut_and_exact_search_in_one_batch(ctx):
    """C2 (ball outliers: the (L-1)-core is the clique, the shortcut settles it) interleaved with C2cube (in-cube
    outliers: the exact search runs), 300 problems so that the small-CTA kernels run."""
    n, B = 800, 300
    prs = [synth.config_problem("C2" if b % 2 else "C2cube", 900 + b, n=n) for b in range(B)]
    nb = prs[0]["noise_bound"]
    assert all(p["noise_bound"] == nb for p in prs)
    src = np.stack([p["src"] for p in prs])
    dst = np.stack([p["dst"] for p in prs])
    prm = params(nb)
    sols, cliques = ctx.solve_batch_array(src, dst, prm)
    assert sols["valid"].all()
    assert_alone(ctx, list(src), list(dst), prm, sols, [cliques[b, :sols[b]["clique_size"]] for b in range(B)])
    # the batch does mix both: exact-search nodes (debug counter 2) for some problems alone, none for the others
    nodes = []
    ctx.set_flags(COUNTERS)
    try:
        for b in range(B):
            ctx.solve(src[b], dst[b], prm)
            nodes.append(ctx.debug_counters()["clique_nodes"])
    finally:
        ctx.set_flags(0)
    searched = sum(1 for x in nodes if x > 0)
    assert 0 < searched < B, searched


def same_f32(a, b):
    a, b = np.float32(a), np.float32(b)
    return a.tobytes() == b.tobytes() or (np.isnan(a) and np.isnan(b))


def assert_consts(ctx, b, src, dst, nb, label):
    """prep_kernel's constants of problem b of the last solve, bit for bit against the CPU copies of its formulas."""
    got = ctx.last_filter_consts(b)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        g = band.consts(src, dst, 2 * nb)
        s = slope.consts(src, dst, 2 * nb)
    mn_s, mx_s, mn_d, mx_d = src.min(0), src.max(0), dst.min(0), dst.max(0)
    assert np.array_equal(got["cs"], 0.5 * (mn_s + mx_s)), label
    assert np.array_equal(got["cd"], 0.5 * (mn_d + mx_d)), label
    for k in ("mhi", "chi", "mlo", "clo"):
        assert same_f32(got[k], g[k]), (label, k, got[k], g[k])
    if got["use_fp64"]:
        assert not got["use_gram"], label
    else:
        assert got["use_gram"] == g["use_gram"], label
    if got["use_gram"]:
        for k in ("cu", "cv", "dl"):
            assert same_f32(got[k], s[k]), (label, k, got[k], s[k])
    else:
        assert got["cu"] == got["cv"] == got["dl"] == 0.0, label


def test_prep_constants_match_the_cpu_copies(ctx):
    """The constants prep_kernel writes (centres, both Gram forms, the guard) equal the CPU copies of its formulas bit
    for bit: on the guard's band fixtures (beta* and one ulp below, 8 beta = D_min and one ulp beyond, a lattice of
    exact ties), each solved alone, and on every problem of a batch mixing Gram-test and interval-test problems
    and problems with one coordinate at 2e8."""
    for label, src, dst, nb in _guard_fixtures():
        ctx.solve(src, dst, params(nb, inlier_selection_mode=1))  # the heuristic clique: the constants come first
        assert_consts(ctx, 0, src, dst, nb, label)
    n = 700
    src, dst, nb = c2_batch(12, n, seed0=60)
    src, dst = src.copy(), dst.copy()
    for b in range(1, 12, 3):
        dst[b, ::7] += 300.0
    for b in range(2, 12, 3):
        src[b, 5] = (2e8, 0.0, 0.0)
    ctx.solve_batch_array(src, dst, params(nb, inlier_selection_mode=1))
    paths = set()
    for b in range(12):
        assert_consts(ctx, b, src[b], dst[b], nb, f"batch/{b}")
        c = ctx.last_filter_consts(b)
        paths.add("fp64" if c["use_fp64"] else "gram" if c["use_gram"] else "interval")
    assert {"gram", "interval"} <= paths, paths


def test_mixed_filter_paths_in_one_batch(ctx):
    """Gram-test, interval-test (far outliers: the guard fails) and exact-path (a coordinate beyond 1e8) problems in
    one batch: each graph is the oracle's, no decided pair disagrees with FP64, counter 15 counts the Gram problems."""
    n = 700
    src, dst, nb = c2_batch(12, n, seed0=40)
    src, dst = src.copy(), dst.copy()
    for b in range(1, 12, 3):
        dst[b, ::7] += 300.0
    for b in range(2, 12, 3):
        src[b, 5] = (2e8, 0.0, 0.0)
    want_gram = 0
    with np.errstate(invalid="ignore", divide="ignore"):
        for b in range(12):
            want_gram += int(band.consts(src[b], dst[b], 2 * nb)["use_gram"])
    assert 0 < want_gram < 12
    prm = params(nb)
    for flags in (COUNTERS, VERIFY):
        ctx.set_flags(flags)
        try:
            ctx.solve_batch_array(src, dst, prm)
            cnt = ctx.debug_counters()
            graphs = [ctx.last_graph(b, n) for b in range(12)]
        finally:
            ctx.set_flags(0)
        if flags == COUNTERS:
            assert cnt["gram_problems"] == want_gram
        else:
            assert cnt["filter_mismatches"] == 0
        for b in range(12):
            obits, odeg, _ = orc.build_graph_bits(src[b], dst[b], nb)
            assert np.array_equal(graphs[b][0], obits), (flags, b)
            assert np.array_equal(graphs[b][1], odeg), (flags, b)
