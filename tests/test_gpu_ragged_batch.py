"""Ragged batches through padded size classes (run on an H100: `pytest -m gpu`).

tzr_solve_batch with differing sizes cuts the problems into size classes and runs each class as one padded device
batch with every problem's own n in Batch::nb.  Each problem must come out exactly as tzr_solve gives it alone: the
whole solution record byte for byte except stage_ms, the clique, and tzr_last_graph(b) equal to the single solve's
graph.  Every case runs with the default classes and under debug flag 16777216 (one class wherever the large-route
and scale-path rules allow), where n = 1 is padded to thousands of rows.
"""
import importlib

import numpy as np
import pytest

capi = importlib.import_module("teaser-plusplus_b200.capi")
synth = importlib.import_module("teaser-plusplus_b200.synth")

pytestmark = pytest.mark.gpu

ONE_CLASS = 16777216
VERIFY = 2
SHORT_QUEUE = 16384
SIZES = [1, 2, 3, 31, 32, 33, 127, 128, 129, 255, 256, 257, 1000, 4097]
STAGE_OFF = capi.SOLUTION_DTYPE.fields["stage_ms"][1]


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.set_flags(0)
    c.close()


def params(**kw):
    d = dict(noise_bound=synth.NOISE_BOUND_SIGMA_001, cbar2=1.0, estimate_scaling=0, rotation_cost_threshold=1e-12)
    d.update(kw)
    return capi.default_params(**d)


def problem(n, seed, outliers=0.9):
    pr = synth.make_problem(n, outliers if n > 2 else 0.0, 7000 + seed, "ball")
    return pr["src"], pr["dst"]


def batch(sizes, seed=0, outliers=0.9):
    return [problem(n, seed + i, outliers) for i, n in enumerate(sizes)]


def check(ctx, probs, prm, flags=0, graphs=True):
    """The ragged call against tzr_solve on every problem alone; returns the batch's solutions."""
    ctx.set_flags(flags)
    sols, cliques = ctx.solve_batch([p[0] for p in probs], [p[1] for p in probs], prm)
    got_graphs = [ctx.last_graph(b, len(p[0])) for b, p in enumerate(probs)] if graphs else None
    for b, (s, d) in enumerate(probs):
        one = ctx.solve(s, d, prm)
        assert sols[b:b + 1].tobytes()[:STAGE_OFF] == bytes(one["sol"])[:STAGE_OFF], (b, len(s))
        assert np.array_equal(cliques[b], one["clique"]), (b, len(s))
        if graphs:
            bits, deg = ctx.last_graph(0, len(s))
            assert np.array_equal(got_graphs[b][0], bits), (b, len(s))
            assert np.array_equal(got_graphs[b][1], deg), (b, len(s))
    ctx.set_flags(0)
    return sols


@pytest.mark.parametrize("flags", [0, ONE_CLASS])
@pytest.mark.parametrize("order", ["shuffled", "reversed"])
def test_sizes_at_every_edge(ctx, flags, order):
    sizes = list(SIZES)
    if order == "shuffled":
        np.random.default_rng(3).shuffle(sizes)
    else:
        sizes.reverse()
    check(ctx, batch(sizes), params(), flags)


@pytest.mark.parametrize("flags", [0, ONE_CLASS])
@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_inlier_selection_modes(ctx, flags, mode):
    # KCORE_HEU at 0.3: the n = 300 problem (half inliers, max core ~149) passes int(0.3 * 300) = 90 but would fail
    # against the padded class's int(0.3 * 4000) = 1200
    probs = batch([4000, 300, 1200, 90], seed=20, outliers=0.5) if mode == 2 else batch([4000, 300, 1200, 90], seed=20)
    sols = check(ctx, probs, params(inlier_selection_mode=mode, kcore_heuristic_threshold=0.3), flags)
    if mode == 2:
        assert sols[1]["clique_size"] > 90


@pytest.mark.parametrize("flags", [0, ONE_CLASS])
@pytest.mark.parametrize("alg", [0, 1, 2])
@pytest.mark.parametrize("tim", [0, 1])
def test_rotation_solvers(ctx, flags, alg, tim):
    check(ctx, batch([600, 150, 420, 33], seed=40, outliers=0.7),
          params(rotation_estimation_algorithm=alg, rotation_tim_graph=tim), flags)


@pytest.mark.parametrize("flags", [0, ONE_CLASS])
def test_unknown_scale_both_paths(ctx, flags):
    probs = []
    for i, n in enumerate([100, 200, 255, 256, 257, 300, 600, 2]):
        s, d = problem(n, 60 + i, 0.5)
        probs.append((s, 1.5 * d))
    check(ctx, probs, params(estimate_scaling=1), flags)


def c1_like(n, seed):
    # outliers moved 500 extents away: beta / D ~ 1e-5 fails the Gram test's guard, the interval test builds the graph
    pr = synth.make_problem(n, 0.9, 8000 + seed, "ball")
    d = pr["dst"].copy()
    out = np.setdiff1d(np.arange(n), pr["inliers"])
    d[out] *= 500.0
    return pr["src"], d


def edgeless(n):
    # grid points 0.1 apart, target scaled by 3: every |d2 - d1| = 2 d1 >= 0.2 exceeds beta
    g = np.stack(np.meshgrid(*[np.arange(8)] * 3, indexing="ij"), -1).reshape(-1, 3)[:n] * 0.1
    return np.ascontiguousarray(g, dtype=np.float64), np.ascontiguousarray(3.0 * g)


@pytest.mark.parametrize("flags", [0, ONE_CLASS])
def test_mixed_tests_exact_path_and_edgeless(ctx, flags):
    s, d = problem(700, 80)
    s = s.copy()
    s[5, 0] = np.nan
    probs = batch([1500, 900], seed=81) + [c1_like(1100, 1), (s, d), edgeless(400), edgeless(3)]
    sols = check(ctx, probs, params(), flags)
    assert sols[4]["n_edges"] == 0 and sols[5]["n_edges"] == 0


@pytest.mark.parametrize("flags", [VERIFY, SHORT_QUEUE, VERIFY | ONE_CLASS, SHORT_QUEUE | ONE_CLASS])
def test_debug_paths(ctx, flags):
    check(ctx, batch([2000, 1300, 257, 64, 5], seed=90) + [c1_like(800, 2)], params(), flags)
    if flags & VERIFY:
        ctx.set_flags(flags)
        ctx.solve_batch(*zip(*batch([2000, 1300, 257, 64, 5], seed=90)), params())
        assert ctx.filter_mismatches() == 0
        ctx.set_flags(0)


@pytest.mark.parametrize("flags", [0, ONE_CLASS])
def test_chunked_two_lane_batch(ctx, flags):
    sizes = np.random.default_rng(5).choice(np.arange(200, 1500), size=80, replace=False)
    check(ctx, batch([int(n) for n in sizes], seed=100), params(), flags, graphs=False)


@pytest.mark.parametrize("flags", [0, ONE_CLASS])
def test_large_route_problem_among_small_ones(flags):
    c = capi.Context(0, max_n=65536)
    try:
        probs = batch([500, 33000, 2000, 40], seed=200, outliers=0.97)
        check(c, probs, params(), flags)
        c.set_flags(flags)
        c.solve_batch([p[0] for p in probs], [p[1] for p in probs], params())
        c.set_flags(0)
        route = c.clique_route(4)  # in the caller's order: only the problem above 32768 takes the large route
        assert route[1] != 0 and route[0] == route[2] == route[3] == 0, route
    finally:
        c.close()


def test_device_entry_point_matches_host_call(ctx):
    torch = pytest.importorskip("torch")
    sizes = [900, 33, 2500, 1, 600, 257]
    probs = batch(sizes, seed=300)
    prm = params()
    sols, cliques = ctx.solve_batch([p[0] for p in probs], [p[1] for p in probs], prm)
    src = torch.from_numpy(np.concatenate([p[0] for p in probs])).cuda()
    dst = torch.from_numpy(np.concatenate([p[1] for p in probs])).cuda()
    sol_t = torch.zeros(len(sizes) * capi.SOLUTION_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    clq_t = torch.full((sum(sizes),), -7, dtype=torch.int32, device="cuda")
    ctx.solve_batch_ragged_dev(prm, sizes, src.data_ptr(), dst.data_ptr(), sol_t.data_ptr(), clq_t.data_ptr())
    ctx.synchronize()
    dev = np.frombuffer(sol_t.cpu().numpy().tobytes(), dtype=capi.SOLUTION_DTYPE)
    assert dev.tobytes() == sols.tobytes()
    flat = clq_t.cpu().numpy()
    at = 0
    for b, n in enumerate(sizes):
        m = len(cliques[b])
        assert np.array_equal(flat[at:at + m], cliques[b]) and np.all(flat[at + m:at + n] == -1), b
        at += n


def test_front_end_to_ragged_solve(ctx):
    rng = np.random.default_rng(11)
    clouds_s, clouds_d = [], []
    for n in [700, 450, 900, 520]:
        s = rng.uniform(size=(n, 3)).astype(np.float32)
        R = synth.random_rotation(rng)
        clouds_s.append(s)
        clouds_d.append((s @ R.T + rng.uniform(-0.5, 0.5, 3)).astype(np.float32))
    feats = ctx.compute_fpfh_batch(clouds_s + clouds_d, 0.1, 0.2)
    B = len(clouds_s)
    pairs = ctx.match_correspondences_batch(clouds_s, clouds_d, feats[:B], feats[B:])
    probs = [(np.ascontiguousarray(clouds_s[b][p[:, 0]], dtype=np.float64),
              np.ascontiguousarray(clouds_d[b][p[:, 1]], dtype=np.float64)) for b, p in enumerate(pairs)]
    assert len({len(p[0]) for p in probs}) > 1 and min(len(p[0]) for p in probs) > 2
    check(ctx, probs, params(noise_bound=0.01))
