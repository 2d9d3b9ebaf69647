"""Problems of up to 65536 correspondences and the large clique route (run on an H100: `pytest -m gpu`).

Route equivalence: debug flag 524288 sends any graph through the large route (heuristic on the full graph, (L-1)-core
on many CTAs, order-preserving compaction, the small route's search on the compacted core, map back).  On the clique
families of test_gpu_clique_boundary.py it must give the small route's cliques, proven codes and search flags, and on
whole solves the same solution records.  Debug flag 1048576 caps the compacted core at 64 vertices, so that the "core
too large" outcome (route -1, heuristic clique, not proven) is reachable at test sizes.  Real sizes: 32769 ... 65536
correspondences on the ball model, checked against float64 numpy rows, a numpy core and the CPU oracle.
"""
import importlib
import os
import sys

import numpy as np
import pytest

import oracle_lib as orc
import test_gpu_clique_boundary as cb

capi = importlib.import_module("teaser-plusplus_b200.capi")
synth = importlib.import_module("teaser-plusplus_b200.synth")

pytestmark = pytest.mark.gpu

LARGE = 524288      # debug flag: the large clique route at any n
CAP64 = 1048576     # debug flag: compacted core capped at 64 vertices
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


def fixed(nb, **kw):
    d = dict(noise_bound=nb, cbar2=1.0, estimate_scaling=0, rotation_cost_threshold=1e-12)
    d.update(kw)
    return capi.default_params(**d)


def both_routes(ctx, flags, bits, base=0, mode=0):
    """max_clique_batch under `base` and under base | LARGE: (small, large, large routes)."""
    flags(base)
    small = ctx.max_clique_batch(bits, mode=mode)
    assert np.all(ctx.clique_route(bits.shape[0]) == 0)
    flags(base | LARGE)
    large = ctx.max_clique_batch(bits, mode=mode)
    route = ctx.clique_route(bits.shape[0])
    assert np.all(route != 0)
    return small, large, route


def assert_same(small, large, exact_cliques=True):
    (c0, p0, f0), (c1, p1, f1) = small, large
    assert np.array_equal(p0, p1), (p0, p1)
    assert np.array_equal(f0, f1), (f0, f1)
    for b, (a, c) in enumerate(zip(c0, c1)):
        # after a Nemhauser-Trotter reduction (flag 8) the second pass keeps the first LARGER clique a warp finds:
        # its size is proven, which clique is not deterministic on either route
        if exact_cliques and not (f0[b] & 8):
            assert np.array_equal(a, c), b
        else:
            assert len(a) == len(c), b


# ------------------------------------------------------------------ route equivalence at small n
@pytest.mark.parametrize("word_edges", [False, True])
@pytest.mark.parametrize("n", [33, 64, 129, 1025])
def test_route_equivalence_multipartite_ties(ctx, flags, n, word_edges):
    rng = np.random.default_rng(1000 + n + 7 * word_edges)
    A, canon, _ = cb.tie_graph(n, rng, word_edges)
    small, large, _ = both_routes(ctx, flags, cb.bits_of(A)[None], cb.FLAG_ONE_PASS)
    assert_same(small, large)
    assert np.array_equal(large[0][0], canon) and large[1][0] == 1


@pytest.mark.parametrize("n", [65, 1024, 4097])
def test_route_equivalence_word_edges(ctx, flags, n):
    A, _ = cb.word_edge_graph(n, np.random.default_rng(2000 + n))
    small, large, route = both_routes(ctx, flags, cb.bits_of(A)[None])
    assert_same(small, large)
    cb.assert_clique(A, large[0][0])
    h = int(ctx.clique_info(1)["heuristic_best"][0])  # the incumbent whose (h-1)-core was compacted
    assert route[0] == cb._core_size(A, h - 1) or (route[0] == h == cb._core_size(A, h - 1))


@pytest.mark.parametrize("name", cb.SEARCH_CASES)
def test_route_equivalence_search_paths(ctx, flags, name):
    A = cb._search_case(name)
    small, large, _ = both_routes(ctx, flags, cb.bits_of(A)[None])
    assert_same(small, large)
    assert large[1][0] == 1


@pytest.mark.parametrize("pairs", [30, 64, 150])
def test_route_equivalence_lp_closes(ctx, flags, pairs):
    A = cb.cocktail_party(pairs, np.random.default_rng(pairs))
    small, large, route = both_routes(ctx, flags, cb.bits_of(A)[None], cb.FLAG_SHORT_FIRST)
    assert_same(small, large)
    assert large[2][0] == 4 and large[1][0] == 2 and route[0] == 2 * pairs


@pytest.mark.parametrize("T,leaves", [(2, [20, 20]), (10, [5, 5, 5, 5]), (40, [8] * 20)])
def test_route_equivalence_nt_reduction(ctx, flags, T, leaves):
    A, omega, lp_ub = cb.triangles_and_stars(T, leaves, np.random.default_rng(T))
    small, large, _ = both_routes(ctx, flags, cb.bits_of(A)[None], cb.FLAG_SHORT_FIRST)
    assert_same(small, large)
    cb._check_nt(A, omega, lp_ub, large[0][0], large[1][0], large[2][0])


@pytest.mark.parametrize("n", [1, 2, 63, 300])
def test_route_equivalence_edgeless_and_complete(ctx, flags, n):
    bits = np.stack([cb.bits_of(np.zeros((n, n), dtype=bool)), cb.bits_of(~np.eye(n, dtype=bool))])
    small, large, route = both_routes(ctx, flags, bits)
    assert_same(small, large)
    assert len(large[0][0]) == 0 and np.array_equal(large[0][1], np.arange(n if n > 1 else 0))
    assert route[1] == max(len(large[0][1]), 1)  # complete graph: the core is the clique, no search


@pytest.mark.parametrize("mode", [1, 2])
def test_route_equivalence_heuristic_modes(ctx, flags, mode):
    rng = np.random.default_rng(40 + mode)
    mats = [cb._search_case("gnp_2000_0.1"), cb.second_chance_graph(1500, 0.15, 15, rng)[0],
            cb.shortcut_graph(1500, rng)[0], cb.gnp(1500, 0.3, rng)]
    bits = np.stack([cb.bits_of(A[:1500, :1500]) for A in mats])
    small, large, _ = both_routes(ctx, flags, bits, mode=mode)
    assert_same(small, large)


def test_route_equivalence_mixed_batch(ctx, flags):
    n = 256
    probs = cb._batch_problems(n, np.random.default_rng(77))
    assert len(probs) >= 12
    for order in (list(range(len(probs))), list(range(len(probs)))[::-1]):
        bits = np.stack([cb.bits_of(probs[i][0]) for i in order])
        small, large, route = both_routes(ctx, flags, bits)
        assert_same(small, large)
        for j, i in enumerate(order):
            A, ref, kind = probs[i]
            cb.assert_clique(A, large[0][j])
            if ref is not None:
                assert np.array_equal(large[0][j], ref), (i, kind)


@pytest.mark.parametrize("model,n", [("ball", 2000), ("ball", 5000), ("incube", 3000), ("incube", 5000)])
def test_route_equivalence_solve(ctx, flags, model, n):
    pr = synth.make_problem(n, 0.95, 77 + n, model, sigma=0.01, noise_bound=synth.NOISE_BOUND_SIGMA_001)
    p = fixed(pr["noise_bound"])
    flags(cb.FLAG_ONE_PASS)  # whether the search finishes must not depend on the wall clock
    a = ctx.solve(pr["src"], pr["dst"], p)
    flags(cb.FLAG_ONE_PASS | LARGE)
    b = ctx.solve(pr["src"], pr["dst"], p)
    assert ctx.clique_route(1)[0] > 0
    ra, rb = bytes(a["sol"]), bytes(b["sol"])
    off = capi.Solution.stage_ms.offset
    assert ra[:off] == rb[:off]  # every field of tzr_solution but stage_ms, bit for bit
    assert np.array_equal(a["clique"], b["clique"])
    assert np.array_equal(a["rot_inliers"], b["rot_inliers"]) and np.array_equal(a["trans_inliers"], b["trans_inliers"])


# ------------------------------------------------------------------ the cap (flag 1048576)
def test_core_above_cap(ctx, flags):
    rng = np.random.default_rng(5)
    dense = cb.gnp(300, 0.5, rng)                      # (L-1)-core: all 300 vertices
    sparse, members = cb.shortcut_graph(300, rng)      # core = the planted clique
    bits = np.stack([cb.bits_of(dense), cb.bits_of(sparse)])
    flags(cb.FLAG_ONE_PASS)
    ref = ctx.max_clique_batch(bits)
    flags(cb.FLAG_ONE_PASS | LARGE | CAP64)
    cl, proven, f = ctx.max_clique_batch(bits)
    route = ctx.clique_route(2)
    heur = ctx.clique_info(2)["heuristic_best"]
    assert route[0] == -1 and proven[0] == 0 and f[0] & 17 == 17
    cb.assert_clique(dense, cl[0])
    assert len(cl[0]) == heur[0]
    assert route[1] == len(members) and np.array_equal(cl[1], members) and proven[1] == 1
    assert np.array_equal(cl[1], ref[0][1]) and f[1] == ref[2][1]


# ------------------------------------------------------------------ real sizes, fixed scale, ball model
def _core(bits, deg, k):
    """k-core of the bitset graph by peeling from {deg >= k}, on the rows of the candidates only."""
    alive = np.nonzero(deg >= k)[0]
    while True:
        rows = np.unpackbits(bits[alive].view(np.uint8), axis=1, bitorder="little")[:, alive]
        d = rows.sum(1)
        keep = d >= k
        if keep.all():
            return alive
        alive = alive[keep]


def _check_rows(pr, bits, n, seed=0):
    beta = 2 * pr["noise_bound"]
    for r in np.random.default_rng(seed).integers(0, n, size=6):
        ds = np.sqrt(((pr["src"] - pr["src"][r]) ** 2)[:, 0] + ((pr["src"] - pr["src"][r]) ** 2)[:, 1]
                     + ((pr["src"] - pr["src"][r]) ** 2)[:, 2])
        dd = np.sqrt(((pr["dst"] - pr["dst"][r]) ** 2)[:, 0] + ((pr["dst"] - pr["dst"][r]) ** 2)[:, 1]
                     + ((pr["dst"] - pr["dst"][r]) ** 2)[:, 2])
        want = np.abs(ds - dd) <= beta
        want[r] = False
        got = np.unpackbits(bits[r].view(np.uint8), bitorder="little")[:n].astype(bool)
        assert np.array_equal(got, want), r


def _check_large_solve(ctx, pr, out, n, b=0, B=1, oracle=False):
    assert out["valid"]
    clique = out["clique"]
    assert set(pr["inliers"].tolist()) <= set(clique.tolist())
    assert synth.angular_error(out["R"], pr["R"]) < 0.02 and np.linalg.norm(out["t"] - pr["t"]) < 0.02
    route = ctx.clique_route(B)[b]
    bits, deg = ctx.last_graph(b, n)
    assert int(deg.sum()) == 2 * out["n_edges"]
    _check_rows(pr, bits, n, seed=b)
    core = _core(bits, deg, len(clique) - 1)
    # the ball model's inliers are the whole (L-1)-core: the uniqueness shortcut, no search
    assert route == len(clique) and np.array_equal(core, clique), (route, len(core))
    if oracle:
        ref, info = orc.max_clique_bits(bits, n)
        assert not info["timed_out"] and np.array_equal(ref, clique)


@pytest.mark.parametrize("n", [32769, 40000, 65536])
def test_large_solve_ball(ctx, n):
    pr = synth.make_problem(n, 0.99, 9000 + n, "ball", sigma=0.01, noise_bound=synth.NOISE_BOUND_SIGMA_001)
    out = ctx.solve(pr["src"], pr["dst"], fixed(pr["noise_bound"]))
    assert out["proven"]
    _check_large_solve(ctx, pr, out, n, oracle=(n == 40000))


def test_large_solve_batch_dev(ctx):
    torch = pytest.importorskip("torch")
    n, B = MAX_N, 5
    prs = [synth.make_problem(n, 0.99, 7000 + b, "ball", sigma=0.01, noise_bound=synth.NOISE_BOUND_SIGMA_001)
           for b in range(B)]
    src = torch.tensor(np.stack([p["src"] for p in prs]), device="cuda")
    dst = torch.tensor(np.stack([p["dst"] for p in prs]), device="cuda")
    sols = torch.zeros((B, capi.SOLUTION_DTYPE.itemsize), dtype=torch.uint8, device="cuda")
    cliques = torch.full((B, n), -1, dtype=torch.int32, device="cuda")
    ctx.solve_batch_dev(fixed(prs[0]["noise_bound"]), B, n, src.data_ptr(), dst.data_ptr(), sols.data_ptr(),
                        cliques.data_ptr())
    ctx.synchronize()
    recs = np.frombuffer(sols.cpu().numpy().tobytes(), dtype=capi.SOLUTION_DTYPE)
    cl = cliques.cpu().numpy()
    for b in (0, B - 1):  # the first problem and the one that starts 2 GiB into the bitset
        m = int(recs[b]["clique_size"])
        out = dict(valid=bool(recs[b]["valid"]), clique=cl[b, :m], R=capi.rotation_from_solution_record(recs[b]),
                   t=np.asarray(recs[b]["translation"]), n_edges=int(recs[b]["n_edges"]))
        assert recs[b]["clique_proven_optimal"] == 1
        _check_large_solve(ctx, prs[b], out, n, b=b, B=B)


def test_size_limits(ctx):
    p = fixed(0.01)
    big = np.zeros((MAX_N + 1, 3))
    with pytest.raises(capi.TzrError, match="too large"):
        ctx.solve(big, big, p)
    with pytest.raises(capi.TzrError, match="invalid argument"):
        ctx.set_max_n(MAX_N + 1)
    with pytest.raises(capi.TzrError, match="invalid argument"):
        ctx.set_max_n(32767)
    c = capi.Context(0)
    try:
        pts = np.random.default_rng(0).uniform(size=(32769, 3))
        with pytest.raises(capi.TzrError, match="too large"):
            c.solve(pts, pts, p)
        c.set_max_n(32769)
        assert c.solve(pts, pts, p)["valid"]
    finally:
        c.close()


# ------------------------------------------------------------------ other modes and cases
def _sym_hash_bits(n, p, seed):
    """Bitset of a symmetric pseudo-random graph, edge (i, j) iff a hash of {i, j} falls below p (no n x n floats)."""
    W = (n + 63) // 64
    bits = np.zeros((n, W), dtype=np.uint64)
    j = np.arange(n, dtype=np.uint64)
    thr = np.uint64(int(p * 2 ** 32))
    for i0 in range(0, n, 2048):
        i = np.arange(i0, min(n, i0 + 2048), dtype=np.uint64)[:, None]
        lo, hi = np.minimum(i, j), np.maximum(i, j)
        h = (lo * np.uint64(0x9E3779B97F4A7C15) + hi * np.uint64(0xC2B2AE3D27D4EB4F) + np.uint64(seed)) \
            & np.uint64(0xFFFFFFFFFFFFFFFF)
        h ^= h >> np.uint64(31)
        h = (h * np.uint64(0xBF58476D1CE4E5B9)) & np.uint64(0xFFFFFFFFFFFFFFFF)
        h ^= h >> np.uint64(29)
        A = ((h & np.uint64(0xFFFFFFFF)) < thr) & (i != j)
        pad = np.zeros((A.shape[0], W * 64), dtype=np.uint8)
        pad[:, :n] = A
        bits[i0:i0 + A.shape[0]] = np.packbits(pad, axis=1, bitorder="little").view(np.uint64)
    return bits


def _bits_clique(bits, c):
    rows = np.unpackbits(bits[c].view(np.uint8), axis=1, bitorder="little")[:, c]
    return int(rows.sum()) == len(c) * (len(c) - 1)


def test_dense_large_graph_returns_heuristic(ctx):
    n = 33000
    bits = _sym_hash_bits(n, 0.15, 1)
    c, proven = ctx.max_clique(bits, n, mode=0)
    assert ctx.clique_route(1)[0] == -1 and not proven
    assert len(c) >= 2 and _bits_clique(bits, c) and np.all(np.diff(c) > 0)


def _plant_bits(bits, members):
    for a in members:
        for b in members:
            if a != b:
                bits[a, b >> 6] |= np.uint64(1) << np.uint64(b & 63)


def test_large_sparse_graph_kcore_and_compaction(ctx):
    """n = 33000, G(n, 0.0005) plus two tied 40-cliques.  KCORE_HEU returns the innermost core (numpy core numbers);
    the exact mode compacts the 39-core (both cliques, 80 vertices), searches it and returns the canonical clique."""
    n, k = 33000, 40
    bits = _sym_hash_bits(n, 0.0005, 2)
    pick = np.random.default_rng(3).choice(n, size=2 * k, replace=False)
    X, Y = np.sort(pick[:k]), np.sort(pick[k:])
    _plant_bits(bits, X)
    _plant_bits(bits, Y)
    deg = np.unpackbits(bits.view(np.uint8), axis=1, bitorder="little")[:, :n].sum(1)
    core = _core(bits, deg, k - 1)  # the innermost core: both cliques form the (k-1)-core, nothing has a k-core
    assert len(_core(bits, deg, k)) == 0 and np.array_equal(core, np.union1d(X, Y))
    c, _ = ctx.max_clique(bits, n, mode=2, kcore_thr=0.0005)
    assert np.array_equal(c, core)
    c, proven = ctx.max_clique(bits, n, mode=0)
    assert proven and ctx.clique_route(1)[0] == 2 * k
    assert np.array_equal(c, min(X.tolist(), Y.tolist()))


@pytest.mark.parametrize("mode", [1, 3])
def test_large_heuristic_and_none_modes(ctx, mode):
    n = 40000
    pr = synth.make_problem(n, 0.99, 41, "ball", sigma=0.01, noise_bound=synth.NOISE_BOUND_SIGMA_001)
    out = ctx.solve(pr["src"], pr["dst"], fixed(pr["noise_bound"], inlier_selection_mode=mode))
    assert out["valid"] and not out["proven"]
    if mode == 1:
        assert set(pr["inliers"].tolist()) <= set(out["clique"].tolist())
        assert synth.angular_error(out["R"], pr["R"]) < 0.02


def test_all_inliers_take_the_shortcut(ctx):
    n = 33000
    pr = synth.make_problem(n, 0.0, 42, "ball", sigma=0.01, noise_bound=synth.NOISE_BOUND_SIGMA_001)
    out = ctx.solve(pr["src"], pr["dst"], fixed(pr["noise_bound"]))
    assert out["proven"] and len(out["clique"]) == n
    assert ctx.clique_route(1)[0] == n


# ------------------------------------------------------------------ front ends and unknown scale
def test_teaserpp_python_40000():
    import subprocess
    host = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "teaser-plusplus_b200", "host")
    subprocess.check_call(["make", "-s", "-C", host])
    sys.path.insert(0, os.path.join(host, "python"))
    import teaserpp_python as tp
    pr = synth.make_problem(40000, 0.99, 43, "ball", sigma=0.01, noise_bound=synth.NOISE_BOUND_SIGMA_001)
    p = tp.RobustRegistrationSolver.Params()
    p.noise_bound = pr["noise_bound"]
    p.estimate_scaling = False
    s = tp.RobustRegistrationSolver(p)
    sol = s.solve(pr["src"].T, pr["dst"].T)
    assert sol.valid and s.isMaxCliqueProvenOptimal()
    assert set(pr["inliers"].tolist()) <= set(np.array(s.getInlierMaxClique()).tolist())
    assert synth.angular_error(np.asarray(sol.rotation), pr["R"]) < 0.02


def test_unknown_scale_33000(ctx):
    torch = pytest.importorskip("torch")
    n = 33000
    K = n * (n - 1) // 2
    need = K * 8 * 2 + 2 * K * 12 * 2  # TIM ratios and ranges, and the sort of their 2K end points (keys + payload, x2)
    free, _ = torch.cuda.mem_get_info()
    if free < need + (8 << 30):
        pytest.skip(f"unknown-scale stage needs about {need / 2**30:.0f} GiB, {free / 2**30:.0f} GiB free")
    # 80 % outliers, as the C2scale configuration: at 99 % the outlier pairs' ratios outnumber the inlier pairs' and
    # the scale TLS (here as in the reference) settles on their mode
    pr = synth.make_problem(n, 0.80, 44, "ball", sigma=0.01, noise_bound=synth.NOISE_BOUND_SIGMA_001)
    s = 1.7
    try:
        out = ctx.solve(pr["src"], pr["dst"] * s, capi.default_params(noise_bound=pr["noise_bound"] * s))
    except capi.TzrError as e:
        if "allocation failed" in str(e):
            pytest.skip(f"unknown-scale stage does not fit the free device memory: {e}")
        raise
    assert out["valid"] and abs(out["scale"] - s) < 0.02 * s
