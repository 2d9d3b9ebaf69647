"""The large clique route where it can be wrong (run on an H100: `pytest -m gpu`).

The route (n > 32768, or debug flag 524288 at any n) decides on the size of the peeled (L-1)-core: exactly L survivors
is the uniqueness shortcut, more than the cap is route -1 (heuristic clique, not proven), anything else is compacted
and searched.  These tests check that it decides on the core itself:
- slow peels: pendant paths numbered against the scan order, which lose one or two vertices per peel round, on both
  routes and under the 64-vertex test cap (debug flag 1048576);
- the cap at its edge: cores of 63, 64 and 65 vertices under the test cap, and of 32768 and 32769 at n = 65536;
- word edges through the relabelling: core and clique members at v % 32 in {0, 31}, at vertex 65535 and at compacted
  positions 31, 32, 63, 64, 1023 and 1024;
- a mixed batch at n = 36000 in both orders, each problem against its own single call;
- real-size solves that need a search: a two-motion scene at n = 40000 (single, batched and ragged) and the all-inlier
  problem at n = 65536.
Every expectation comes from tests/large_route_cases.py (closed forms and numpy cores; the CPU oracle on small graphs
and on the scene's core), whose premises tests/test_large_route_cases_cpu.py checks without a GPU.
"""
import importlib

import numpy as np
import pytest

import large_route_cases as C

capi = importlib.import_module("teaser-plusplus_b200.capi")
synth = importlib.import_module("teaser-plusplus_b200.synth")

pytestmark = pytest.mark.gpu

LARGE = 524288        # debug flag: the large clique route at any n
CAP64 = 1048576       # debug flag: compacted core capped at 64 vertices
SHORT_FIRST = 32768   # debug flag: first exact pass of 1 ns, so every searched problem meets the LP kernel
MAX_N = 65536


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0, max_n=MAX_N)
    yield c
    c.close()


@pytest.fixture()
def flags(ctx):
    yield ctx.set_flags
    ctx.set_flags(0)


def fixed(nb):
    return capi.default_params(noise_bound=nb, cbar2=1.0, estimate_scaling=0, rotation_cost_threshold=1e-12)


def bits_of(case):
    return C.to_bits(case["n"], case["edges"])


def batch(ctx, bits, mode=0, **kw):
    cl, proven, f = ctx.max_clique_batch(bits, mode=mode, **kw)
    return cl, proven, f, ctx.clique_route(bits.shape[0])


# ------------------------------------------------------------------ a. slow peels on both routes
@pytest.mark.parametrize("base", [0, SHORT_FIRST])
@pytest.mark.parametrize("name", ["one300", "lp260", "several"])
def test_slow_peel_both_routes(ctx, flags, name, base):
    case = C.slow_peel_case(name)
    bits = bits_of(case)[None]
    seen = {}
    for extra in (0, LARGE, LARGE | CAP64):
        flags(base | extra)
        cl, proven, f, route = batch(ctx, bits)
        got = (proven[0], f[0], route[0])
        assert np.array_equal(cl[0], case["clique"]), (extra, cl[0][:8], got)
        assert proven[0] == 1, (extra, got)
        assert route[0] == (len(case["core"]) if extra else 0), (extra, got)
        seen[extra] = int(f[0])
    assert len(set(seen.values())) == 1, seen  # the search flags do not depend on the route


@pytest.mark.parametrize("name", ["one300", "several"])
def test_slow_peel_kcore_heuristic(ctx, flags, name):
    case = C.slow_peel_case(name)
    bits = bits_of(case)[None]
    inner = C.innermost_core(case["n"], case["edges"])
    for extra in (0, LARGE):
        flags(extra)
        cl, proven, _, _ = batch(ctx, bits, mode=2, kcore_thr=1e-6)
        assert np.array_equal(cl[0], inner) and proven[0] == 0, extra


def test_extra_blocks_only_for_slow_peels(ctx, flags):
    """A graph whose core peel converges inside the first 48 rounds takes exactly the launches of an edgeless graph; a
    slow peel adds whole blocks of 48 rounds plus the survivors' listing."""
    flags(LARGE)

    def launches(case):
        before = ctx.kernel_launches()
        cl, proven, _, route = batch(ctx, bits_of(case)[None])
        assert np.array_equal(cl[0], case["clique"]) and proven[0] == 1
        return ctx.kernel_launches() - before

    n = 400
    edgeless = dict(n=n, edges=np.zeros((0, 2), dtype=np.int64), clique=np.zeros(0, dtype=np.int64))
    base = launches(edgeless)
    assert launches(C.pendant_paths(n, [0, 31, 399], [(32, 8), (64, 40)])) == base
    extra = launches(C.slow_peel_case("one300")) - base
    assert extra > 0 and extra % 49 == 0, extra


def test_slow_peel_65536(ctx):
    """250 paths of 256 on a triangle: 48 in-place rounds leave at least 39753 vertices, above the 32768 cap."""
    case = C.slow_peel_case("paths250")
    bits = bits_of(case)
    c, proven = ctx.max_clique(bits, case["n"])
    route = int(ctx.clique_route(1)[0])
    assert np.array_equal(c, case["clique"]) and proven and route == 3, (c[:8], proven, route)
    c2, _ = ctx.max_clique(bits, case["n"], mode=2, kcore_thr=1e-6)
    assert np.array_equal(c2, C.innermost_core(case["n"], case["edges"]))


# ------------------------------------------------------------------ b. the compaction cap at its edge
def _check_capped(case, cl, proven, f, route):
    assert np.array_equal(cl, case["clique"])  # the heuristic finds the planted clique (premise on the CPU)
    assert route == -1 and proven == 0 and f & 17 == 17, (route, proven, f)


@pytest.mark.parametrize("size", [63, 64, 65])
def test_cap64_edge(ctx, flags, size):
    case = C.cap_case(size, 256)
    bits = bits_of(case)[None]
    flags(0)
    small = batch(ctx, bits)
    assert np.array_equal(small[0][0], case["clique"]) and small[1][0] == 1 and small[3][0] == 0
    flags(LARGE)
    cl, proven, f, route = batch(ctx, bits)
    assert np.array_equal(cl[0], case["clique"]) and proven[0] == 1 and route[0] == size and f[0] == small[2][0]
    flags(LARGE | CAP64)
    cl, proven, f, route = batch(ctx, bits)
    if size <= 64:
        assert np.array_equal(cl[0], case["clique"]) and proven[0] == 1 and f[0] == small[2][0]
        assert route[0] == size
    else:
        _check_capped(case, cl[0], proven[0], f[0], route[0])
    for extra in (0, LARGE):
        flags(extra)
        kc, _, _, _ = batch(ctx, bits, mode=2, kcore_thr=1e-6)
        assert np.array_equal(kc[0], C.innermost_core(case["n"], case["edges"]))


@pytest.mark.parametrize("size", [32768, 32769])
def test_real_cap_edge(ctx, size):
    case = C.cap_case(size, MAX_N)
    cl, proven, f, route = batch(ctx, bits_of(case)[None])
    if size == 32768:
        assert np.array_equal(cl[0], case["clique"]) and proven[0] == 1 and route[0] == size, (proven[0], f[0], route[0])
    else:
        _check_capped(case, cl[0], proven[0], f[0], route[0])


# ------------------------------------------------------------------ c. word edges through the relabelling
@pytest.mark.parametrize("n", [4096, MAX_N])
def test_word_edges_through_relabelling(ctx, flags, n):
    case = C.word_edge_case(n)
    bits = bits_of(case)[None]
    results = []
    for extra in ((0, LARGE) if n <= 32768 else (0,)):
        flags(extra)
        cl, proven, f, route = batch(ctx, bits)
        assert np.array_equal(cl[0], case["clique"]) and proven[0] == 1, (extra, cl[0], proven[0], f[0])
        assert route[0] == (len(case["core"]) if (extra or n > 32768) else 0)
        results.append(int(f[0]))
    assert len(set(results)) == 1


# ------------------------------------------------------------------ d. a mixed large batch
def test_mixed_large_batch(ctx):
    cases = C.mixed_batch_cases()
    n = cases[0][1]["n"]
    bits = [bits_of(c) for _, c, _ in cases]
    single = []
    for (name, case, want), b in zip(cases, bits):
        cl, proven, f, route = batch(ctx, b[None])
        single.append((cl[0], int(proven[0]), int(f[0]), int(route[0])))
        assert np.array_equal(cl[0], case["clique"]), name
        assert route[0] == want and proven[0] == (0 if want < 0 else 1), (name, proven[0], f[0], route[0])
    for order in (list(range(len(cases))), list(range(len(cases)))[::-1]):
        cl, proven, f, route = batch(ctx, np.stack([bits[i] for i in order]))
        for j, i in enumerate(order):
            got = (cl[j], int(proven[j]), int(f[j]), int(route[j]))
            assert np.array_equal(got[0], single[i][0]) and got[1:] == single[i][1:], (cases[i][0], got[1:], single[i][1:])
    assert n == 36000


# ------------------------------------------------------------------ e. real-size solves that need a search
SCENE_N, SCENE_M = 40000, 24


@pytest.fixture(scope="module")
def scene():
    return C.two_motion_scene(SCENE_N, SCENE_M, 4)


def _check_scene(ctx, sc, clique, proven, R, t, b=0, B=1):
    assert np.array_equal(clique, sc["expect"]), clique
    assert proven == 1
    assert int(ctx.clique_route(B)[b]) == 2 * sc["m"]
    R0, t0 = sc["motion"]
    assert synth.angular_error(R, R0) < 0.02 and np.linalg.norm(t - t0) < 0.02


def test_two_motion_scene_solve(ctx, scene):
    sc = scene
    out = ctx.solve(sc["src"], sc["dst"], fixed(sc["nb"]))
    assert out["valid"]
    _check_scene(ctx, sc, out["clique"], int(out["sol"].clique_proven_optimal), out["R"], out["t"])
    rot, trans = ctx.last_inliers(0)
    assert np.array_equal(rot, out["rot_inliers"]) and np.array_equal(trans, out["trans_inliers"])
    bits, deg = ctx.last_graph(0, sc["n"])  # the device graph is the exact one (premise: no pair near the threshold)
    assert np.array_equal(C.edges_of_bits(bits, sc["n"]), sc["edges"])


def test_two_motion_scene_batches(ctx, scene):
    sc = scene
    p = fixed(sc["nb"])
    sols, cl = ctx.solve_batch([sc["src"]] * 2, [sc["dst"]] * 2, p)
    for b in range(2):
        _check_scene(ctx, sc, cl[b], int(sols[b]["clique_proven_optimal"]),
                     capi.rotation_from_solution_record(sols[b]), np.asarray(sols[b]["translation"]), b, 2)
    # ragged: the large problem between small ones, each small one against its own single solve
    small = [C.two_motion_scene(80, 20, 5), C.two_motion_scene(500, 30, 6)]
    srcs = [small[0]["src"], sc["src"], small[1]["src"]]
    dsts = [small[0]["dst"], sc["dst"], small[1]["dst"]]
    sols, cl = ctx.solve_batch(srcs, dsts, p)
    _check_scene(ctx, sc, cl[1], int(sols[1]["clique_proven_optimal"]), capi.rotation_from_solution_record(sols[1]),
                 np.asarray(sols[1]["translation"]), 1, 3)
    rot, trans = ctx.last_inliers(1)
    assert len(rot) == len(trans) == sc["m"]  # CHAIN: one TIM per clique member
    for b, s in ((0, small[0]), (2, small[1])):
        one = ctx.solve(s["src"], s["dst"], p)
        assert np.array_equal(cl[b], one["clique"]) and np.array_equal(one["clique"], s["expect"]), b
        assert int(sols[b]["clique_proven_optimal"]) == 1


def test_all_inliers_65536(ctx):
    n = MAX_N
    bits = np.full((n, C.words64(n)), np.uint64(0xFFFFFFFFFFFFFFFF), dtype=np.uint64)
    idx = np.arange(n)
    bits[idx, idx >> 6] &= ~(np.uint64(1) << (idx & 63).astype(np.uint64))
    c, proven = ctx.max_clique(bits, n)
    assert proven and np.array_equal(c, idx) and int(ctx.clique_route(1)[0]) == n
    del bits
    pr = synth.make_problem(n, 0.0, 65536, "ball", sigma=0.01, noise_bound=synth.NOISE_BOUND_SIGMA_001)
    out = ctx.solve(pr["src"], pr["dst"], fixed(pr["noise_bound"]))
    assert out["valid"] and out["proven"] and np.array_equal(out["clique"], idx)
    assert int(ctx.clique_route(1)[0]) == n and int(out["n_edges"]) == n * (n - 1) // 2
