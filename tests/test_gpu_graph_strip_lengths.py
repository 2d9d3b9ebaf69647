"""GPU tests of graph_strip2_kernel at every strip length it can run (`pytest -m gpu`).  launch_graph picks 4 or 6 blocks
per strip from B, n and the SM count, so without help a test reaches only the length its batch and its card select, and
lengths 5, 7 and 8 never run: from 7 blocks on a ring slot of the column operands is filled a third time and its `full`
mbarrier phase returns to its starting parity.  Debug flag bits 28-31 force the length (capi.strip_flags) and
tzr_ctx_last_strip_blocks reports the length the last graph build ran, so every case here states the length it reached.

The checker is the oracle's FP64 bitset, degrees and edge count, at strip lengths 1 ... 8 and the automatic choice:
tile-edge sizes under the production, verifying, separate-degree and short-queue instances; exact-tie lattices,
guard-edge bands and a mixed Gram / interval / exact-path batch under both forms of the Gram test; the interval test and
the unknown-scale Gram path; ragged size classes whose problems end in the middle of a long strip or before whole strips;
the automatic switch from 4 to 6 blocks on both sides of its threshold; one problem above 16384 points; and one long-strip
batch run twice, whose bitsets must be byte-identical."""
import importlib

import numpy as np
import pytest
import torch

import oracle_lib as orc
from test_gpu_graph_boundary import LATTICES, NB, _mixed_batch, _scale_problems, assert_graph, far_outliers, use_gram
from test_gpu_graph_strip_schedule import FLAGS, SIZES

band = importlib.import_module("gram_band_check")
capi = importlib.import_module("teaser-plusplus_b200.capi")
synth = importlib.import_module("teaser-plusplus_b200.synth")

pytestmark = pytest.mark.gpu

LENGTHS = [0, 1, 2, 3, 4, 5, 6, 7, 8]  # 0: launch_graph's own choice
AUTO_SHORT, AUTO_LONG = 4, 6           # the two lengths the automatic choice takes
TWO_SLOPE = 134217728                  # the Gram test's two-slope form (bit 27)
ONE_CLASS = 16777216                   # a ragged batch forms one padded size class (bit 24)
STAGE_OFF = capi.SOLUTION_DTYPE.fields["stage_ms"][1]


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.set_flags(0)
    c.close()


def reached(L, auto=AUTO_SHORT):
    return L if L else auto


def build(ctx, src, dst, nb, flags, L):
    """graph_build with strips of L blocks (0: automatic); returns bits, degrees, edge count, counters (flags 2 / 4)."""
    ctx.set_flags(flags | capi.strip_flags(L))
    try:
        bits, deg, ne = ctx.graph_build(src, dst, 2 * nb)
        cnt = ctx.debug_counters() if flags & 6 else None
        got_L = ctx.last_strip_blocks()
    finally:
        ctx.set_flags(0)
    assert got_L == reached(L), f"flags {flags}: strips of {got_L} blocks, meant {reached(L)}"
    return bits, deg, ne, cnt


def solve_array(ctx, src, dst, flags, L, nb=NB):
    p = capi.default_params(noise_bound=nb, cbar2=1.0, estimate_scaling=0, rotation_cost_threshold=1e-12)
    ctx.set_flags(flags | capi.strip_flags(L))
    try:
        sols, cl = ctx.solve_batch_array(src, dst, p)
        cnt = ctx.debug_counters() if flags & 6 else None
        got_L = ctx.last_strip_blocks()
    finally:
        ctx.set_flags(0)
    assert got_L == reached(L), f"flags {flags}: strips of {got_L} blocks, meant {reached(L)}"
    graphs = [ctx.last_graph(b, src.shape[1]) for b in range(src.shape[0])]
    return sols, cl, graphs, cnt


# ------------------------------------------------------------------ 1. tile edges
@pytest.mark.parametrize("n", SIZES)
def test_tile_edges_at_every_strip_length(ctx, n):
    """test_gpu_graph_strip_schedule's sizes (1 ... 5001: rows and column groups cut off by n, warps without rows) at
    strip lengths 1 ... 8 and automatic, under flags 0, 2|4 (zero disagreements), 256 and 16384."""
    pr = synth.config_problem("C2", 11, n=n)
    src, dst, nb = pr["src"], pr["dst"], pr["noise_bound"]
    want = orc.build_graph_bits(src, dst, nb)
    for L in LENGTHS:
        for flags in FLAGS:
            got = build(ctx, src, dst, nb, flags, L)
            if flags & 2:
                assert got[3]["filter_mismatches"] == 0, f"n={n} L={L}"
                assert got[3]["gram_problems"] == use_gram(src, dst, nb), f"n={n} L={L}"
            assert_graph(got, want, f"n={n} L={L} flags {flags}")


# ------------------------------------------------------------------ 2. edge corpora, both Gram forms
@pytest.mark.parametrize("form", [0, TWO_SLOPE], ids=["single-slope", "two-slope"])
@pytest.mark.parametrize("offset,scale,perm,edges", LATTICES)
def test_exact_ties_at_every_strip_length(ctx, form, offset, scale, perm, edges):
    """11^3 lattices (n = 1331, 11 row blocks) whose neighbour pairs tie with beta exactly or sit an ulp off it: every
    tie is undecided, re-checked, and its mirror bit leaves through the split-phase barrier of a long strip."""
    src, dst, nb = band.lattice(offset, scale, permute_seed=perm)
    want = orc.build_graph_bits(src, dst, nb)
    assert want[2] == edges
    for L in LENGTHS:
        got = build(ctx, src, dst, nb, form | 4, L)
        assert got[3]["gram_problems"] == 1, f"L={L}"
        if not form:
            assert got[3]["filter_rechecks"] >= 3630, f"L={L}: the ties were not re-checked"
        assert_graph(got, want, f"lattice L={L} form {form}")
        got = build(ctx, src, dst, nb, form | 16384 | 2 | 4, L)  # queue full: ties evaluated in place
        assert got[3]["filter_mismatches"] == 0, f"L={L}"
        assert_graph(got, want, f"lattice L={L} form {form} short queue")


@pytest.mark.parametrize("form", [0, TWO_SLOPE], ids=["single-slope", "two-slope"])
@pytest.mark.parametrize("n", [387, 1000, 2049])
def test_guard_edge_bands_at_every_strip_length(ctx, form, n):
    """Guard-edge problems (~2 % of the pairs undecided) at 4, 8 and 17 row blocks: queued and in-place re-checks land
    in mirror words of every block of a strip, also the strip's last one, which leaves after the loop."""
    src, dst, nb = band.guard_edge(1.02, 0.6, n=n, seed=n + 1)
    want = orc.build_graph_bits(src, dst, nb)
    for L in LENGTHS:
        for flags in (0, 2 | 4, 16384):
            got = build(ctx, src, dst, nb, form | flags, L)
            if flags & 2:
                assert got[3]["filter_mismatches"] == 0
            assert_graph(got, want, f"guard-edge n={n} L={L} flags {form | flags}")


@pytest.fixture(scope="module")
def mixed():
    """16 problems of n = 1331 (11 row blocks): Gram, interval and exact-path problems, ties, duplicates, a guard edge"""
    src, dst, gram = _mixed_batch(16, seed0=200)
    return src, dst, gram, [orc.build_graph_bits(src[b], dst[b], NB) for b in range(src.shape[0])]


def assert_batch(sols, graphs, want, what):
    for b, ((bits, deg), (obits, odeg, oe)) in enumerate(zip(graphs, want)):
        assert np.array_equal(bits, obits), f"{what} problem {b}: bitset differs"
        assert np.array_equal(deg, odeg), f"{what} problem {b}: degrees differ"
        assert int(sols[b]["n_edges"]) == oe, f"{what} problem {b}: edge count"


@pytest.mark.parametrize("form", [0, TWO_SLOPE], ids=["single-slope", "two-slope"])
def test_mixed_path_batch_at_every_strip_length(ctx, mixed, form):
    """One uniform launch over Gram, interval and exact-path problems at every strip length: each problem's retained
    bitset and degrees equal the oracle's, and counter 15 counts exactly the Gram problems."""
    src, dst, gram, want = mixed
    for L in LENGTHS:
        for flags in (4, 16384 | 4):
            sols, _, graphs, cnt = solve_array(ctx, src, dst, form | flags, L)
            assert cnt["gram_problems"] == gram, f"L={L}"
            assert_batch(sols, graphs, want, f"mixed L={L} flags {form | flags}")


# ------------------------------------------------------------------ 3. interval test and unknown scale
def test_interval_test_at_every_strip_length(ctx):
    """The interval test, taken by a problem the guard refuses (outliers 300 extents away) and forced on a C2 problem
    (flag 512), at 10 and 11 row blocks."""
    src1, dst1, nb1 = far_outliers(n=1200)
    pr = synth.config_problem("C2", 21, n=1331)
    for label, src, dst, nb, flags in (("far outliers", src1, dst1, nb1, 0), ("C2 flag 512", pr["src"], pr["dst"],
                                                                               pr["noise_bound"], 512)):
        assert flags or not use_gram(src, dst, nb)
        want = orc.build_graph_bits(src, dst, nb)
        for L in LENGTHS:
            got = build(ctx, src, dst, nb, flags | 4, L)
            assert got[3]["gram_problems"] == 0, f"{label} L={L}: not the interval test"
            assert_graph(got, want, f"{label} L={L}")
            got = build(ctx, src, dst, nb, flags | 2 | 4, L)
            assert got[3]["filter_mismatches"] == 0
            assert_graph(got, want, f"{label} L={L} verify")


def test_unknown_scale_gram_path_at_every_strip_length(ctx):
    """estimate_scaling = 1: at n = 256 the retained bitset equals the oracle's (scale bit-exact there); at n = 1000
    (8 row blocks, where the scale comes from the large TLS path) every strip length gives the automatic choice's
    solution record, clique and bitset."""
    for label, src, dst, nb in _scale_problems():
        kw = dict(noise_bound=nb, cbar2=1.0, estimate_scaling=1, rotation_cost_threshold=1e-12)
        o = orc.solve(src, dst, orc.default_params(**kw), want_adj=True)
        for L in LENGTHS:
            ctx.set_flags(4 | capi.strip_flags(L))
            try:
                g = ctx.solve(src, dst, capi.default_params(**kw))
                cnt = ctx.debug_counters()
                assert ctx.last_strip_blocks() == reached(L)
            finally:
                ctx.set_flags(0)
            assert cnt["gram_problems"] == 1, f"{label} L={L}"
            assert g["scale"] == o["scale"], f"{label} L={L}"
            bits, deg = ctx.last_graph(0, len(src))
            assert np.array_equal(bits, o["adj_bits"]), f"{label} L={L}"
            assert g["n_edges"] == o["sol"].n_edges, f"{label} L={L}"
    pr = synth.make_problem(1000, 0.5, 4244, "ball")
    src, dst, nb = pr["src"], pr["dst"] * 1.7, pr["noise_bound"] * 1.7
    prm = capi.default_params(noise_bound=nb, cbar2=1.0, estimate_scaling=1, rotation_cost_threshold=1e-12)
    ref = None
    for L in LENGTHS:
        ctx.set_flags(4 | capi.strip_flags(L))
        try:
            g = ctx.solve(src, dst, prm)
            cnt = ctx.debug_counters()
            assert ctx.last_strip_blocks() == reached(L)
        finally:
            ctx.set_flags(0)
        assert cnt["gram_problems"] == 1, f"L={L}"
        bits, deg = ctx.last_graph(0, len(src))
        row_pop = np.unpackbits(bits.view(np.uint8), axis=1, bitorder="little").sum(1)
        assert np.array_equal(deg, row_pop), f"L={L}"
        got = (bytes(g["sol"])[:STAGE_OFF], g["clique"], bits)
        if ref is None:
            ref = got
            continue
        assert got[0] == ref[0], f"L={L}: solution record differs from the automatic choice's"
        assert np.array_equal(got[1], ref[1]) and np.array_equal(got[2], ref[2]), f"L={L}"


# ------------------------------------------------------------------ 4. ragged size classes
RAGGED = [2000, 700, 1, 1100, 129, 900, 1536, 385, 1665]  # padded to 2000: 16 row blocks


def test_ragged_sizes_cut_long_strips():
    """The sizes end in the middle of a strip of problem 0's row block 0 and before whole strips, at every forced length
    above 1 (from the strip order the device decodes)."""
    nt = (max(RAGGED) + 127) // 128
    for L in range(2, 9):
        I, J0 = capi.strip_schedule(nt, L)
        J1 = np.minimum(nt, J0 + L)
        clipped = past = False
        for n in RAGGED[1:]:
            ntb = (n + 127) // 128
            clipped |= bool(np.any((J0 < ntb) & (ntb < J1) & (J1 - J0 == L)))
            past |= bool(np.any((J0 >= ntb) & (I < ntb)))
        assert clipped and past, f"L={L}: clipped {clipped}, strips wholly past a problem {past}"


@pytest.fixture(scope="module")
def ragged_problems(ctx):
    """the problems, each one's single solve (flags 0) and the oracle's graph"""
    prm = capi.default_params(noise_bound=synth.NOISE_BOUND_SIGMA_001, cbar2=1.0, estimate_scaling=0,
                              rotation_cost_threshold=1e-12)
    out = []
    for i, n in enumerate(RAGGED):
        pr = synth.make_problem(n, 0.9 if n > 2 else 0.0, 7300 + i, "ball")
        one = ctx.solve(pr["src"], pr["dst"], prm)
        out.append((pr["src"], pr["dst"], one, orc.build_graph_bits(pr["src"], pr["dst"], synth.NOISE_BOUND_SIGMA_001)))
    return prm, out


@pytest.mark.parametrize("flags", [ONE_CLASS, ONE_CLASS | 2 | 4, ONE_CLASS | TWO_SLOPE],
                         ids=["production", "verify", "two-slope"])
def test_ragged_class_at_every_strip_length(ctx, ragged_problems, flags):
    """One padded size class (n = 1 ... 2000 in a 2000-point batch) through graph_strip2_ragged_kernel at every strip
    length: each problem equals its single solve (record bytes, clique) and its graph the oracle's."""
    prm, probs = ragged_problems
    for L in LENGTHS:
        ctx.set_flags(flags | capi.strip_flags(L))
        try:
            sols, cliques = ctx.solve_batch([p[0] for p in probs], [p[1] for p in probs], prm)
            cnt = ctx.debug_counters() if flags & 2 else None
            assert ctx.last_strip_blocks() == reached(L)
            graphs = [ctx.last_graph(b, len(p[0])) for b, p in enumerate(probs)]
        finally:
            ctx.set_flags(0)
        if cnt is not None:
            assert cnt["filter_mismatches"] == 0, f"L={L}"
        for b, (src, _, one, want) in enumerate(probs):
            what = f"L={L} flags {flags} problem {b} (n={len(src)})"
            assert sols[b:b + 1].tobytes()[:STAGE_OFF] == bytes(one["sol"])[:STAGE_OFF], what
            assert np.array_equal(cliques[b], one["clique"]), what
            assert np.array_equal(graphs[b][0], want[0]), f"{what}: bitset differs from the oracle's"
            assert np.array_equal(graphs[b][1], want[1]), f"{what}: degrees differ from the oracle's"
            assert int(sols[b]["n_edges"]) == want[2], what


# ------------------------------------------------------------------ 5. the automatic switch
DISTINCT = 3
SWITCH_N = 1000  # 8 row blocks, 36 blocks per problem


def _device_batch(B, n, prs):
    src = np.ascontiguousarray(np.stack([prs[b % DISTINCT]["src"] for b in range(B)]))
    dst = np.ascontiguousarray(np.stack([prs[b % DISTINCT]["dst"] for b in range(B)]))
    return torch.from_numpy(src).cuda(), torch.from_numpy(dst).cuda()


def _solve_dev(ctx, prm, B, n, src_d, dst_d, flags):
    sol_d = torch.zeros(B * capi.SOLUTION_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    ctx.set_flags(flags)
    try:
        ctx.solve_batch_dev(prm, B, n, src_d.data_ptr(), dst_d.data_ptr(), sol_d.data_ptr())
        ctx.synchronize()
        L = ctx.last_strip_blocks()
    finally:
        ctx.set_flags(0)
    sols = np.frombuffer(sol_d.cpu().numpy().tobytes(), dtype=capi.SOLUTION_DTYPE)
    sample = [0, 1, 2, B // 2, B - 3, B - 2, B - 1]
    return L, sols, {b: ctx.last_graph(b, n) for b in sample}


def test_automatic_switch_at_its_threshold(ctx):
    """launch_graph takes 6-block strips once every CTA slot (6 per SM) has 512 blocks to sweep.  One batch a problem
    below that threshold runs 4-block strips and one at it 6-block strips; each gives the bits of its length forced, and
    the oracle's."""
    n = SWITCH_N
    nt = (n + 127) // 128
    slots = torch.cuda.get_device_properties(0).multi_processor_count * 6
    B_at = -(-512 * slots // (nt * (nt + 1) // 2))
    prs = [synth.config_problem("C2", 60 + k, n=n) for k in range(DISTINCT)]
    nb = prs[0]["noise_bound"]
    prm = capi.default_params(noise_bound=nb, cbar2=1.0, estimate_scaling=0, rotation_cost_threshold=1e-12)
    want = [orc.build_graph_bits(pr["src"], pr["dst"], nb) for pr in prs]
    for B, L_auto in ((B_at - 1, AUTO_SHORT), (B_at, AUTO_LONG)):
        src_d, dst_d = _device_batch(B, n, prs)
        auto = _solve_dev(ctx, prm, B, n, src_d, dst_d, 0)
        forced = _solve_dev(ctx, prm, B, n, src_d, dst_d, capi.strip_flags(L_auto))
        del src_d, dst_d
        assert auto[0] == L_auto, f"B={B}: automatic choice {auto[0]} blocks, expected {L_auto}"
        assert forced[0] == L_auto
        rec = [s.view(np.uint8).reshape(B, -1)[:, :STAGE_OFF] for s in (auto[1], forced[1])]
        assert np.array_equal(rec[0], rec[1]), f"B={B}: solution records differ between the automatic and the forced length"
        ne = np.array([int(s["n_edges"]) for s in auto[1]])
        assert np.array_equal(ne, np.array([want[b % DISTINCT][2] for b in range(B)])), f"B={B}: edge counts"
        for b, (bits, deg) in auto[2].items():
            fb, fd = forced[2][b]
            assert np.array_equal(bits, fb) and np.array_equal(deg, fd), f"B={B} problem {b}: auto != forced"
            assert np.array_equal(bits, want[b % DISTINCT][0]), f"B={B} problem {b}: bitset differs from the oracle's"
            assert np.array_equal(deg, want[b % DISTINCT][1]), f"B={B} problem {b}: degrees differ from the oracle's"


# ------------------------------------------------------------------ 6. one large problem
def test_large_problem_long_strips(ctx):
    """n = 16385 (129 row blocks, the last with one row) in strips of 6 and 8 blocks against the oracle, production
    and verifying instances."""
    pr = synth.config_problem("C2", 5, n=16385)
    src, dst, nb = pr["src"], pr["dst"], pr["noise_bound"]
    want = orc.build_graph_bits(src, dst, nb)
    for L in (6, 8):
        assert_graph(build(ctx, src, dst, nb, 0, L), want, f"n=16385 L={L}")
        got = build(ctx, src, dst, nb, 2 | 4, L)
        assert got[3]["filter_mismatches"] == 0, f"L={L}"
        assert_graph(got, want, f"n=16385 L={L} verify")


# ------------------------------------------------------------------ 7. determinism
def test_long_strip_batch_is_deterministic(ctx, mixed):
    """The mixed batch in 7-block strips with a 64-entry re-check queue (warps race for it): two runs give byte-identical
    bitsets, degrees and solution records."""
    src, dst, _, want = mixed
    first = solve_array(ctx, src, dst, 16384 | 4, 7)
    second = solve_array(ctx, src, dst, 16384 | 4, 7)
    for b in range(src.shape[0]):
        assert first[2][b][0].tobytes() == second[2][b][0].tobytes(), f"problem {b}: bitsets differ between runs"
        assert first[2][b][1].tobytes() == second[2][b][1].tobytes(), f"problem {b}: degrees differ between runs"
        assert first[0][b:b + 1].tobytes()[:STAGE_OFF] == second[0][b:b + 1].tobytes()[:STAGE_OFF], f"problem {b}"
    assert_batch(first[0], first[2], want, "L=7 first run")
