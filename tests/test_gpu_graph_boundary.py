"""GPU tests of the default graph kernel where it can be wrong (`pytest -m gpu`): which pair test ran, the production
template (fused degrees, patched by tc_patch_kernel) at tile edges, exact FP64 ties on the threshold, a full re-check queue
and batches that mix the Gram, interval and exact paths in one launch.  The oracle's FP64 bitset is the checker; debug
counter 15 (`gram_problems`) says which problems graph_strip2_kernel built with the Gram test, and debug flag 16384 caps
the re-check queue at 64 entries so that its queue-full path runs.  The fixtures shared with tests/test_gram_band_cpu.py
come from scripts/gram_band_check.py, whose consts() is the CPU copy of prep_kernel's conditioning guard."""
import importlib
import os
import sys

import numpy as np
import pytest

import oracle_lib as orc
from test_gpu_parity import GRAPH_CASES

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
band = importlib.import_module("gram_band_check")
capi = importlib.import_module("teaser-plusplus_b200.capi")
synth = importlib.import_module("teaser-plusplus_b200.synth")

pytestmark = pytest.mark.gpu

QUEUE_CAP = 64  # entries of the re-check queue under debug flag 16384


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


def build(ctx, src, dst, nb, flags):
    """graph_build under `flags`; returns bits, degrees, edge count and the debug counters (flags 2 / 4)."""
    ctx.set_flags(flags)
    try:
        bits, deg, ne = ctx.graph_build(src, dst, 2 * nb)
        cnt = ctx.debug_counters() if flags & 6 else None
    finally:
        ctx.set_flags(0)
    return bits, deg, ne, cnt


def assert_graph(got, want, what=""):
    bits, deg, ne = got[:3]
    obits, odeg, oe = want
    assert np.array_equal(bits, obits), f"{what}: bitset differs from the oracle's"
    assert np.array_equal(deg, odeg), f"{what}: degrees differ from the oracle's"
    assert ne == oe, f"{what}: edge count {ne} != {oe}"


def use_gram(src, dst, nb):
    with np.errstate(invalid="ignore", divide="ignore"):  # n = 1: no extent, the guard fails on 0 / 0
        return int(band.consts(src, dst, 2 * nb)["use_gram"])


def far_outliers(n=400):
    """C1-like (test_tc_kernel_falls_back_when_ill_conditioned): outliers 300 extents away, noise bound 1e-5."""
    pr = synth.config_problem("C2", 4, n=n)
    dst = pr["dst"].copy()
    dst[::7] += 300.0
    return pr["src"], dst, 1e-5


def duplicate_heavy(n=700, nb=None, seed=8):
    """C2cube with many duplicated source / destination points (zero-length TIMs, s <= beta^2)."""
    pr = synth.make_problem(n, 0.95, 5000 * 1000 + seed, "incube", noise_bound=nb)
    src, dst = pr["src"].copy(), pr["dst"].copy()
    for k in range(0, n // 4, 3):
        src[k + 1] = src[k]
    for k in range(n // 4, n // 2, 3):
        dst[k + 1] = dst[k]
        src[k + 1] = src[k] + 1e-9
    return src, dst, pr["noise_bound"]


# ------------------------------------------------------------------ 1. routing and A/B identity
@pytest.mark.parametrize("cfg,n", GRAPH_CASES)
def test_routing_and_flag_ab_identity(ctx, cfg, n):
    """Every benchmark geometry takes the Gram test (counter 15 = 1), flag 512 takes it away, and flags 0 / 512 / 1 / 2048
    (Gram, interval, pure FP64, one-MUFU kernel) give the oracle's bitset."""
    pr = synth.config_problem(cfg, 3, n=n)
    src, dst, nb = pr["src"], pr["dst"], pr["noise_bound"]
    want = orc.build_graph_bits(src, dst, nb)
    assert use_gram(src, dst, nb)
    got = build(ctx, src, dst, nb, 4)
    assert got[3]["gram_problems"] == 1, "the problem did not take the Gram test"
    assert_graph(got, want, "flag 4")
    got = build(ctx, src, dst, nb, 512 | 4)
    assert got[3]["gram_problems"] == 0
    assert_graph(got, want, "flag 512")
    got = build(ctx, src, dst, nb, 2048 | 4)
    assert got[3]["gram_problems"] == 0  # graph_strip3_kernel has no Gram test
    assert_graph(got, want, "flag 2048")
    for flags in (0, 1):
        assert_graph(build(ctx, src, dst, nb, flags), want, f"flag {flags}")


def test_routing_ill_conditioned_problems_keep_the_interval_test(ctx):
    """C1 (bunny, outliers 5-10 extents away) and far outliers fail the guard: counter 15 = 0, bits exact."""
    pr = synth.bunny_problem(os.path.join(synth.GOLDEN_DIR, "bun_zipper_res3.ply"))
    for src, dst, nb in ((pr["src"], pr["dst"], pr["noise_bound"]), far_outliers()):
        assert not use_gram(src, dst, nb)
        got = build(ctx, src, dst, nb, 4)
        assert got[3]["gram_problems"] == 0
        assert_graph(got, orc.build_graph_bits(src, dst, nb), "ill-conditioned")


def _guard_fixtures():
    out = []
    src = band._cube(1200, 5)
    for rho in (0.3, 0.6, 1.0):
        b = band.guard_beta(src, rho)
        for beta in (b, np.nextafter(b, 0.0)):  # the first beta the guard admits, and one ulp below it
            out.append((f"beta*/{rho}" if beta == b else f"below/{rho}", src, band._stretched(src, beta, rho), 0.5 * beta))
    for beyond in (False, True):
        out.append((f"dmin{int(beyond)}",) + band.dmin_edge(beyond))
    out.append(("lattice",) + band.lattice(permute_seed=1))
    return out


def test_device_guard_matches_the_cpu_copy_at_its_edges(ctx):
    """At beta* and one ulp below it, and at 8 beta = D_min and one ulp beyond, counter 15 equals consts()["use_gram"]:
    the CPU copy of the guard that the band check relies on is the device's.  Bits exact either way."""
    routed = []
    for label, src, dst, nb in _guard_fixtures():
        got = build(ctx, src, dst, nb, 4)
        assert got[3]["gram_problems"] == use_gram(src, dst, nb), label
        routed.append(got[3]["gram_problems"])
        assert_graph(got, orc.build_graph_bits(src, dst, nb), label)
    assert routed == [1, 0, 1, 0, 1, 0, 1, 0, 1]


# ------------------------------------------------------------------ 2. production template at tile edges
TILE_SIZES = [1, 2, 31, 32, 33, 127, 128, 129, 255, 256, 257, 383, 385, 513, 1000]


def _tile_problems(n):
    pr = synth.config_problem("C2", 7, n=n)
    yield "C2", pr["src"], pr["dst"], pr["noise_bound"]
    if n >= 31:  # ~2 % of the pairs undecided: many queued pairs, in diagonal and off-diagonal 128-blocks
        yield "guard-edge", *band.guard_edge(1.02, 0.6, n=n, seed=n)


@pytest.mark.parametrize("n", TILE_SIZES)
def test_production_template_at_tile_edges(ctx, n):
    """graph_strip2_kernel<false, 8, true> (flag 0: fused degrees, adjusted by tc_patch_kernel) at every tile edge, then
    the interval test (flag 512) and the verifying template with the degree kernel (flag 2 | 4)."""
    for label, src, dst, nb in _tile_problems(n):
        want = orc.build_graph_bits(src, dst, nb)
        assert_graph(build(ctx, src, dst, nb, 0), want, f"{label} n={n} flag 0")
        assert_graph(build(ctx, src, dst, nb, 512), want, f"{label} n={n} flag 512")
        got = build(ctx, src, dst, nb, 2 | 4)
        assert got[3]["filter_mismatches"] == 0
        assert got[3]["gram_problems"] == use_gram(src, dst, nb)
        assert_graph(got, want, f"{label} n={n} flag 2|4")


# ------------------------------------------------------------------ 3. exact ties
LATTICES = [(0.0, 1.0, None, 3630), (1024.0, 1.0, None, 3630), (0.0, 1.0, 1, 3630), (1024.0, 1.0, 2, 3630),
            (0.0, 1.0 + 2.0 ** -50, 1, 363), (0.0, 1.0 - 2.0 ** -50, 1, 3630)]


@pytest.mark.parametrize("offset,scale,perm,edges", LATTICES)
def test_exact_ties_on_the_threshold(ctx, offset, scale, perm, edges):
    """Lattice neighbours with |d1 - d2| = beta exactly are edges (the predicate is <=).  Permuted, the ties fall inside
    and across the diagonal 128-blocks, where the patch kernel must flip the mirror bit only across blocks."""
    src, dst, nb = band.lattice(offset, scale, permute_seed=perm)
    want = orc.build_graph_bits(src, dst, nb)
    assert want[2] == edges
    got = build(ctx, src, dst, nb, 4)
    assert got[3]["gram_problems"] == 1
    assert got[3]["filter_rechecks"] >= 3630  # every tie was undecided and re-checked
    assert_graph(got, want, "Gram, flag 4")
    for flags in (0, 512, 2048, 2 | 4):
        got = build(ctx, src, dst, nb, flags)
        assert_graph(got, want, f"flag {flags}")
        if flags & 2:
            assert got[3]["filter_mismatches"] == 0


# ------------------------------------------------------------------ 4. queue overflow
def _overflow_problems():
    """(label, taken by the tensor-core kernel, overflows the queue under flag 2048 too, src, dst, noise bound).  The
    one-MUFU kernel's band is narrower on the duplicates problem: only a handful of its pairs are undecided there."""
    yield ("lattice", True, True) + band.lattice(permute_seed=3)
    yield ("duplicates", True, False) + duplicate_heavy()
    yield ("guard-edge", False, True) + band.guard_edge(1.02, 0.6, n=1000, seed=9)


@pytest.mark.parametrize("flags", [16384, 16384 | 2, 16384 | 2048, 16384 | 1024])
def test_full_queue_is_evaluated_in_place(ctx, flags):
    """A 64-entry queue: the first warp that does not fit leaves void entries, the rest evaluate in place, and
    tc_patch_kernel clamps its count.  Production template, verifying template, one-MUFU kernel and tensor-core kernel
    (which takes the lattice and the duplicates; the guard-edge problem's band is too wide for it)."""
    for label, tc_ok, v7_overflows, src, dst, nb in _overflow_problems():
        want = orc.build_graph_bits(src, dst, nb)
        got = build(ctx, src, dst, nb, flags | 4)
        if v7_overflows or not flags & 2048:
            assert got[3]["filter_rechecks"] > QUEUE_CAP, f"{label}: the queue never overflowed"
        if flags & 2:
            assert got[3]["filter_mismatches"] == 0
        if flags & 1024:
            assert got[3]["tc_problems"] == int(tc_ok), label
        assert_graph(got, want, f"{label} flags {flags}")
        assert_graph(build(ctx, src, dst, nb, flags), want, f"{label} flags {flags} without counters")


# ------------------------------------------------------------------ 5. mixed-path batches
NB = 2.0 ** -5  # one noise bound for the whole batch: beta = 2^-4 = the lattice spacing
N = 1331        # 11^3, the lattice's size


def _guard_edge_at(beta, n, seed, rho_unit=0.04, factor=1.02):
    """A unit-cube guard-edge fixture scaled by L so that its beta (factor * beta*) becomes `beta`; TIMs shorter than
    L * rho_unit are edges, so the graph stays sparse."""
    src = band._cube(n, seed)
    b_unit = factor * band.guard_beta(src, rho_unit)
    L = beta / b_unit
    src = src * L
    return src, (1.0 + b_unit / rho_unit) * src + band.GUARD_OFFSET


def _mixed_batch(B, seed0=0):
    """B problems of N points, noise bound NB; returns src, dst (B, N, 3) and the expected counter-15 value."""
    kinds = ["C2", "C4", "far", "fp64", "lattice", "dups", "guard", "C2"]
    S, D, gram = [], [], 0
    for b in range(B):
        kind, s = kinds[b % len(kinds)], seed0 + b
        if kind in ("C2", "C4"):
            pr = synth.make_problem(N, 0.95 if kind == "C2" else 0.9, 7000 + s, "ball", noise_bound=NB)
            src, dst = pr["src"], pr["dst"]
        elif kind == "far":  # interval test
            pr = synth.make_problem(N, 0.95, 7000 + s, "ball", noise_bound=NB)
            src, dst = pr["src"], pr["dst"].copy()
            dst[::7] += 300.0
        elif kind == "fp64":  # extent beyond 1e8: every pair takes the exact path
            pr = synth.make_problem(N, 0.95, 7000 + s, "ball", noise_bound=NB)
            src, dst = pr["src"], pr["dst"].copy()
            dst[5] = 3e8
        elif kind == "lattice":
            src, dst, _ = band.lattice(permute_seed=s)
        elif kind == "dups":
            src, dst, _ = duplicate_heavy(N, NB, seed=s)
        else:
            src, dst = _guard_edge_at(2 * NB, N, s)
        expect = {"C2": 1, "C4": 1, "far": 0, "fp64": 0, "lattice": 1, "dups": 1, "guard": 1}[kind]
        assert use_gram(src, dst, NB) == expect, kind
        gram += expect
        S.append(src)
        D.append(dst)
    return np.ascontiguousarray(np.stack(S)), np.ascontiguousarray(np.stack(D)), gram


@pytest.mark.parametrize("B,flags", [(8, 0), (64, 0), (64, 16384)])
def test_mixed_path_batch_every_problem_exact(ctx, B, flags):
    """One uniform batch with Gram, interval and exact-path problems, ties, duplicates and a guard-edge problem through
    solve_batch_array (B = 64: the chunked pipeline; flag 16384: the queue overflows across problems).  Every problem's
    retained bitset and degrees equal the oracle's; counter 15 counts exactly the Gram problems."""
    src, dst, gram = _mixed_batch(B)
    p = capi.default_params(noise_bound=NB, cbar2=1.0, estimate_scaling=0, rotation_cost_threshold=1e-12)
    ctx.set_flags(flags | 4)
    try:
        sols, _ = ctx.solve_batch_array(src, dst, p)
        cnt = ctx.debug_counters()
    finally:
        ctx.set_flags(0)
    assert cnt["gram_problems"] == gram
    if flags & 16384:
        assert cnt["filter_rechecks"] > QUEUE_CAP
    for b in range(B):
        obits, odeg, oe = orc.build_graph_bits(src[b], dst[b], NB)
        bits, deg = ctx.last_graph(b, N)
        assert np.array_equal(bits, obits), f"problem {b}: bitset differs"
        assert np.array_equal(deg, odeg), f"problem {b}: degrees differ"
        assert int(sols[b]["n_edges"]) == oe, f"problem {b}: edge count"


# ------------------------------------------------------------------ 6. unknown scale on the Gram path
def _scale_problems():
    pr = synth.make_problem(256, 0.5, 4243, "ball")
    yield "ball x1.7", pr["src"], pr["dst"] * 1.7, pr["noise_bound"] * 1.7
    src, dst, nb = band.guard_edge(1.2, 0.3, n=256, seed=11)
    dst = dst.copy()
    idx = np.arange(0, 256, 4)
    dst[idx] = dst[np.roll(idx, 1)]  # wrong correspondences inside the cloud: the bounding boxes do not move
    yield "guard-edge", src, dst, nb


def test_unknown_scale_gram_path_matches_oracle(ctx):
    """estimate_scaling = 1 at n <= 256 (scale bit-exact against the oracle): the float copies are pre-scaled, the exact
    re-check uses the division-based sequence; the retained bitset equals the oracle's, on the Gram path."""
    for label, src, dst, nb in _scale_problems():
        kw = dict(noise_bound=nb, cbar2=1.0, estimate_scaling=1, rotation_cost_threshold=1e-12)
        o = orc.solve(src, dst, orc.default_params(**kw), want_adj=True)
        assert band.consts(src * o["scale"], dst, 2 * nb)["use_gram"], label
        ctx.set_flags(4)
        try:
            g = ctx.solve(src, dst, capi.default_params(**kw))
            cnt = ctx.debug_counters()
        finally:
            ctx.set_flags(0)
        assert cnt["gram_problems"] == 1, label
        assert g["scale"] == o["scale"], label
        bits, deg = ctx.last_graph(0, len(src))
        assert np.array_equal(bits, o["adj_bits"]), label
        row_pop = np.unpackbits(bits.view(np.uint8), axis=1, bitorder="little").sum(1)
        assert np.array_equal(deg, row_pop), label
        assert g["n_edges"] == o["sol"].n_edges, label
