"""GPU tests of the Gram test's single-slope form (the default since it replaced the two-slope form, which debug flag
134217728 keeps as a same-build A/B switch; DESIGN.md §3.1).  Every fixture of scripts/slope_band_check.py runs on the
device under both forms: the bitset, degrees and edge count against the oracle's FP64 graph, and the verifying template
(flag 2), which re-checks every decided pair in FP64, must count no mismatch.  Also: the queue-full path (flag 16384),
a mixed Gram / interval / exact-path batch, a ragged batch in one size class, and the tile edges n = 1 ... 1000."""
import importlib
import os
import sys

import numpy as np
import pytest

import oracle_lib as orc
from test_gpu_graph_boundary import (QUEUE_CAP, TILE_SIZES, _mixed_batch, _overflow_problems, _tile_problems, NB, N,
                                     assert_graph, build, use_gram)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
slope = importlib.import_module("slope_band_check")
capi = importlib.import_module("teaser-plusplus_b200.capi")
synth = importlib.import_module("teaser-plusplus_b200.synth")

pytestmark = pytest.mark.gpu

TWO_SLOPE = 134217728  # debug bit 27: the two-slope form
ONE_CLASS = 16777216   # debug bit 24: a ragged batch forms one size class
FORMS = [0, TWO_SLOPE]


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


FIXTURES = slope.fixtures(small=True)


@pytest.mark.parametrize("label", [f[0] for f in FIXTURES])
def test_both_forms_match_the_oracle_and_verify_clean(ctx, label):
    """Bitset against the oracle under both forms; flag 2 (every decided pair re-checked in FP64) counts 0 mismatches,
    and counter 15 counts the problem as a Gram problem under both forms exactly when the guard holds."""
    _, src, dst, nb = next(f for f in FIXTURES if f[0] == label)
    want = orc.build_graph_bits(src, dst, nb)
    gram = use_gram(src, dst, nb)
    for form in FORMS:
        assert_graph(build(ctx, src, dst, nb, form), want, f"{label} form {form}")
        got = build(ctx, src, dst, nb, form | 2 | 4)
        assert got[3]["filter_mismatches"] == 0, f"{label} form {form}"
        assert got[3]["gram_problems"] == gram, f"{label} form {form}"
        assert_graph(got, want, f"{label} form {form} flag 2")


@pytest.mark.parametrize("form", FORMS)
def test_full_queue_both_forms(ctx, form):
    """A 64-entry re-check queue (flag 16384): the pairs that do not fit are evaluated in place, under both forms."""
    for label, _, _, src, dst, nb in _overflow_problems():
        want = orc.build_graph_bits(src, dst, nb)
        got = build(ctx, src, dst, nb, form | 16384 | 4)
        assert got[3]["filter_rechecks"] > QUEUE_CAP, f"{label}: the queue never overflowed"
        assert_graph(got, want, f"{label} form {form}")
        got = build(ctx, src, dst, nb, form | 16384 | 2 | 4)
        assert got[3]["filter_mismatches"] == 0, label
        assert_graph(got, want, f"{label} form {form} flag 2")


@pytest.mark.parametrize("form", FORMS)
def test_mixed_batch_both_forms(ctx, form):
    """Gram, interval and exact-path problems, ties, duplicates and a guard-edge problem in one uniform batch."""
    src, dst, gram = _mixed_batch(16, seed0=100)
    p = capi.default_params(noise_bound=NB, cbar2=1.0, estimate_scaling=0, rotation_cost_threshold=1e-12)
    ctx.set_flags(form | 4)
    try:
        ctx.solve_batch_array(src, dst, p)
        cnt = ctx.debug_counters()
    finally:
        ctx.set_flags(0)
    assert cnt["gram_problems"] == gram
    for b in range(src.shape[0]):
        obits, odeg, _ = orc.build_graph_bits(src[b], dst[b], NB)
        bits, deg = ctx.last_graph(b, N)
        assert np.array_equal(bits, obits), f"problem {b}: bitset differs"
        assert np.array_equal(deg, odeg), f"problem {b}: degrees differ"


@pytest.mark.parametrize("form", FORMS)
def test_ragged_batch_mixed_paths(ctx, form):
    """A ragged batch in one padded size class (graph_strip2_ragged_kernel) that mixes Gram and interval problems of
    different sizes: every problem's graph equals the oracle's."""
    probs = []
    for k, n in enumerate([900, 130, 600, 33, 257]):
        pr = synth.make_problem(n, 0.9, 9100 + k, "ball")
        src, dst = pr["src"], pr["dst"].copy()
        if k % 2:  # outliers far away: the guard fails, the interval test builds the graph
            dst[::5] *= 500.0
        probs.append((src, dst))
    nb = 0.01
    p = capi.default_params(noise_bound=nb, cbar2=1.0, estimate_scaling=0, rotation_cost_threshold=1e-12)
    routes = [use_gram(s, d, nb) for s, d in probs]
    assert 0 < sum(routes) < len(routes)
    ctx.set_flags(form | ONE_CLASS)
    try:
        ctx.solve_batch([s for s, _ in probs], [d for _, d in probs], p)
        graphs = [ctx.last_graph(b, len(s)) for b, (s, _) in enumerate(probs)]
    finally:
        ctx.set_flags(0)
    for b, (s, d) in enumerate(probs):
        obits, odeg, _ = orc.build_graph_bits(s, d, nb)
        assert np.array_equal(graphs[b][0], obits), f"problem {b} (n={len(s)}): bitset differs"
        assert np.array_equal(graphs[b][1], odeg), f"problem {b} (n={len(s)}): degrees differ"


@pytest.mark.parametrize("n", TILE_SIZES)
def test_tile_edges_both_forms(ctx, n):
    """The production template at every tile edge under the two-slope switch (the default form runs in
    tests/test_gpu_graph_boundary.py), and the verifying template under the default form."""
    for label, src, dst, nb in _tile_problems(n):
        want = orc.build_graph_bits(src, dst, nb)
        assert_graph(build(ctx, src, dst, nb, TWO_SLOPE), want, f"{label} n={n} two-slope")
        got = build(ctx, src, dst, nb, 2 | 4)
        assert got[3]["filter_mismatches"] == 0
        assert_graph(got, want, f"{label} n={n} flag 2")


def test_the_switch_selects_the_form(ctx):
    """Bit 27 really runs the other form: at the guard edge the single-slope band leaves several times more pairs
    undecided than the two-slope band (11 % against 3 % on this fixture in scripts/slope_band_check.py), so the
    re-check counts tell the two kernels apart; both graphs equal the oracle's."""
    src, dst, nb = slope.gbc.guard_edge(1.02, 0.6, n=1000, seed=9)
    want = orc.build_graph_bits(src, dst, nb)
    single, two = build(ctx, src, dst, nb, 4), build(ctx, src, dst, nb, TWO_SLOPE | 4)
    assert single[3]["gram_problems"] == two[3]["gram_problems"] == 1
    assert single[3]["filter_rechecks"] > 2 * two[3]["filter_rechecks"] > 0
    assert_graph(single, want, "single-slope")
    assert_graph(two, want, "two-slope")
