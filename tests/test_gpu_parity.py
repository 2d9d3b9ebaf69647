"""GPU parity tests (run on an H100: `pytest -m gpu`).  Every call goes through the C-ABI
(libteaser_b200.so via ctypes); the oracle is the checker."""
import importlib
import os

import numpy as np
import pytest

import oracle_lib as orc

capi = importlib.import_module("teaser-plusplus_b200.capi")
synth = importlib.import_module("teaser-plusplus_b200.synth")

pytestmark = pytest.mark.gpu

ROT_TOL = 1e-4  # rad   (BASELINE.json north_star)
TRANS_TOL = 1e-4  # m


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


def fixed_params(nb, **kw):
    d = dict(noise_bound=nb, cbar2=1.0, estimate_scaling=0, rotation_estimation_algorithm=0,
             rotation_gnc_factor=1.4, rotation_max_iterations=100, rotation_cost_threshold=1e-12)
    d.update(kw)
    return d


# ------------------------------------------------------------------ stage 1: graph, bit-exact
GRAPH_CASES = [("C2", 700), ("C2cube", 900), ("C3", 1300), ("C4", 513), ("C5", 1000), ("C2", 128), ("C2", 129),
               ("C2cube", 257), ("C2", 31), ("C2", 2)]


@pytest.mark.parametrize("cfg,n", GRAPH_CASES)
def test_graph_bit_exact(ctx, cfg, n):
    pr = synth.config_problem(cfg, 3, n=n)
    beta = 2 * pr["noise_bound"]
    obits, odeg, oe = orc.build_graph_bits(pr["src"], pr["dst"], pr["noise_bound"])
    ctx.set_flags(2 | 4)  # verify FP32 filter against FP64 for every pair, count rechecks
    bits, deg, ne = ctx.graph_build(pr["src"], pr["dst"], beta)
    assert ctx.filter_mismatches() == 0
    rechecks = ctx.filter_rechecks()
    ctx.set_flags(0)
    assert np.array_equal(bits, obits)
    assert np.array_equal(deg, odeg)
    assert ne == oe
    assert rechecks < 0.02 * n * n + 64  # the exact path is the exception, not the rule
    # pure FP64 mode gives the same bits
    ctx.set_flags(1)
    bits64, _, _ = ctx.graph_build(pr["src"], pr["dst"], beta)
    ctx.set_flags(0)
    assert np.array_equal(bits64, obits)


@pytest.mark.parametrize("shift,scale,nb", [(1e4, 1.0, None), (0.0, 1e-3, 3.3682e-5), (-3e6, 50.0, None),
                                             (0.0, 1.0, 1e-9), (0.0, 1.0, 10.0)])
def test_graph_bit_exact_conditioning(ctx, shift, scale, nb):
    """Large offsets / tiny scales / degenerate bounds: the FP32 filter must degrade to the exact path,
    never to wrong bits."""
    pr = synth.config_problem("C2cube", 11, n=400)
    src = pr["src"] * scale + shift
    dst = pr["dst"] * scale - 0.5 * shift
    nbv = pr["noise_bound"] * scale if nb is None else nb
    obits, odeg, oe = orc.build_graph_bits(src, dst, nbv)
    ctx.set_flags(2)
    bits, deg, ne = ctx.graph_build(src, dst, 2 * nbv)
    assert ctx.filter_mismatches() == 0
    ctx.set_flags(0)
    assert np.array_equal(bits, obits)
    assert ne == oe


def test_graph_duplicates_and_nan(ctx):
    pr = synth.config_problem("C2", 5, n=300)
    src, dst = pr["src"].copy(), pr["dst"].copy()
    src[10] = src[11]
    dst[10] = dst[11]  # zero-length TIM
    src[20] = src[21]
    obits, _, oe = orc.build_graph_bits(src, dst, pr["noise_bound"])
    bits, _, ne = ctx.graph_build(src, dst, 2 * pr["noise_bound"])
    assert np.array_equal(bits, obits) and ne == oe
    src[5, 1] = np.nan
    obits, _, oe = orc.build_graph_bits(src, dst, pr["noise_bound"])
    bits, _, ne = ctx.graph_build(src, dst, 2 * pr["noise_bound"])
    assert np.array_equal(bits, obits) and ne == oe


def test_graph_full_size_c2(ctx):
    pr = synth.config_problem("C2", 0)
    obits, odeg, oe = orc.build_graph_bits(pr["src"], pr["dst"], pr["noise_bound"])
    bits, deg, ne = ctx.graph_build(pr["src"], pr["dst"], 2 * pr["noise_bound"])
    assert np.array_equal(bits, obits)
    assert np.array_equal(deg, odeg) and ne == oe


def _graph_properties(bits, deg, ne, n):
    b = np.unpackbits(bits.view(np.uint8), axis=1, bitorder="little")[:, :n].astype(bool)
    assert not b.diagonal().any()
    assert np.array_equal(b, b.T)
    assert np.array_equal(b.sum(1), deg)
    assert b.sum() == 2 * ne
    pad = np.unpackbits(bits.view(np.uint8), axis=1, bitorder="little")[:, n:]
    assert not pad.any()


@pytest.mark.parametrize("cfg", ["C3", "C5"])
def test_graph_full_size_properties(ctx, cfg):
    """Full BASELINE sizes through size-independent properties (symmetry, empty diagonal, degree sums),
    plus exact rows for a sample of vertices."""
    pr = synth.config_problem(cfg, 0)
    n = pr["src"].shape[0]
    bits, deg, ne = ctx.graph_build(pr["src"], pr["dst"], 2 * pr["noise_bound"])
    _graph_properties(bits, deg, ne, n)
    rng = np.random.default_rng(0)
    beta = 2 * pr["noise_bound"]
    for i in rng.choice(n, size=16, replace=False):
        d1 = np.sqrt((((pr["src"] - pr["src"][i]) ** 2)[:, 0] + ((pr["src"] - pr["src"][i]) ** 2)[:, 1])
                     + ((pr["src"] - pr["src"][i]) ** 2)[:, 2])
        d2 = np.sqrt((((pr["dst"] - pr["dst"][i]) ** 2)[:, 0] + ((pr["dst"] - pr["dst"][i]) ** 2)[:, 1])
                     + ((pr["dst"] - pr["dst"][i]) ** 2)[:, 2])
        row = np.abs(d1 - d2) <= beta
        row[i] = False
        got = np.unpackbits(bits[i].view(np.uint8), bitorder="little")[:n].astype(bool)
        assert np.array_equal(got, row)


# ------------------------------------------------------------------ stage 2: max clique
def _bits_from_dense(A):
    n = A.shape[0]
    W = (n + 63) // 64
    padded = np.zeros((n, W * 64), dtype=np.uint8)
    padded[:, :n] = A
    return np.packbits(padded, axis=1, bitorder="little").view(np.uint64).reshape(n, W)


@pytest.mark.parametrize("seed", range(8))
def test_clique_random_graphs(ctx, seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(40, 400))
    p = float(rng.uniform(0.05, 0.5))
    A = np.triu(rng.uniform(size=(n, n)) < p, 1)
    if seed % 2 == 0:
        k = int(rng.integers(10, 30))
        idx = rng.choice(n, size=k, replace=False)
        A[np.ix_(idx, idx)] = True
        A = np.triu(A, 1)
    A = A | A.T
    bits = _bits_from_dense(A)
    oc, info = orc.max_clique_bits(bits, n)
    gc, proven = ctx.max_clique(bits, n, mode=0)
    assert proven
    assert len(gc) == len(oc)
    assert all(A[a, b] for a in gc for b in gc if a != b)
    assert np.all(np.diff(gc) > 0)
    assert np.array_equal(gc, oc)  # canonical (lexicographically smallest) maximum clique, ties included


def test_clique_toy_graphs(ctx):
    # test/teaser/graph-test.cc:131-305
    A = ~np.eye(5, dtype=bool)
    gc, proven = ctx.max_clique(_bits_from_dense(A), 5)
    assert gc.tolist() == [0, 1, 2, 3, 4] and proven
    adj = {0: [2, 3], 1: [2], 2: [0, 1, 3], 3: [0, 2]}
    A = np.zeros((4, 4), dtype=bool)
    for a, l in adj.items():
        A[a, l] = True
    gc, proven = ctx.max_clique(_bits_from_dense(A), 4)
    assert gc.tolist() == [0, 2, 3]
    gc, proven = ctx.max_clique(_bits_from_dense(np.zeros((4, 4), dtype=bool)), 4)
    assert len(gc) == 0  # PMC reports lb = 0 on an edgeless graph; solve() then returns valid = false


def test_clique_canonical_tie_break(ctx):
    import itertools
    A = np.zeros((8, 8), dtype=bool)
    for K in ([0, 1, 2, 3], [4, 5, 6, 7]):
        for a, b in itertools.combinations(K, 2):
            A[a, b] = A[b, a] = True
    gc, proven = ctx.max_clique(_bits_from_dense(A), 8)
    assert gc.tolist() == [0, 1, 2, 3] and proven
    A = np.zeros((6, 6), dtype=bool)
    for K in ([2, 3, 4, 5], [0, 3, 4, 5]):
        for a, b in itertools.combinations(K, 2):
            A[a, b] = A[b, a] = True
    gc, proven = ctx.max_clique(_bits_from_dense(A), 6)
    assert gc.tolist() == [0, 3, 4, 5]


@pytest.mark.parametrize("cfg,n", [("C2", 1000), ("C2cube", 1500), ("C3", 3000), ("C5", 2000)])
def test_clique_on_inlier_graphs(ctx, cfg, n):
    pr = synth.config_problem(cfg, 1, n=n)
    bits, deg, ne = ctx.graph_build(pr["src"], pr["dst"], 2 * pr["noise_bound"])
    oc, info = orc.max_clique_bits(bits, n)
    gc, proven = ctx.max_clique(bits, n, mode=0)
    assert proven
    assert np.array_equal(gc, oc)  # identical index set (canonical tie-break on both sides)


# ------------------------------------------------------------------ stage 3: GNC-TLS rotation
def _gnc_problem(seed, m=300, outlier_frac=0.3, nb=0.05):
    rng = np.random.default_rng(seed)
    src = rng.normal(size=(m, 3))
    R = synth.random_rotation(rng)
    noise = rng.normal(size=(m, 3))
    noise *= (rng.uniform(0.3, 0.9, size=(m, 1)) * nb) / np.linalg.norm(noise, axis=1, keepdims=True)
    dst = src @ R.T + noise
    k = int(outlier_frac * m)
    dst[:k] = rng.normal(size=(k, 3)) * 2
    return src, dst, R


@pytest.mark.parametrize("seed", range(5))
def test_gnc_tls_iterating(ctx, seed):
    """Planted outlier TIMs so that the weight update / mu schedule really runs (SURVEY §4 coverage hole)."""
    src, dst, R = _gnc_problem(seed)
    o = orc.gnc_tls(src, dst, 100, 1e-12, 1.4, 0.05)
    g = ctx.gnc_tls_rotation(src, dst, 0.05, 1.4, 100, 1e-12)
    assert o["iterations"] > 3
    assert abs(g["iterations"] - o["iterations"]) <= 1
    # summation order differs (block tree vs sequential) and the 1e-12 stop rule may fire one iteration
    # apart: compare within a small fraction of the 1e-4 rad budget
    assert synth.angular_error(o["R"], g["R"]) < 1e-6
    assert np.mean(g["inliers"] != o["inliers"]) < 0.01
    assert abs(g["cost"] - o["cost"]) <= 1e-6 * max(1.0, abs(o["cost"]))
    assert synth.angular_error(R, g["R"]) < 0.05


def test_gnc_tls_kat(ctx):
    src = np.loadtxt(os.path.join(synth.GOLDEN_DIR, "registration_test", "rotation_only_src.csv"), delimiter=",")
    Rexp = np.array([[0.997379773225804, -0.019905935977315, -0.069551000516966],
                     [0.013777311189888, 0.996068297974922, -0.087510750572249],
                     [0.071019530105605, 0.086323226782879, 0.993732623426126]])
    g = ctx.gnc_tls_rotation(src, src @ Rexp.T, 1e-3, 1.4, 100, 1e-12)  # rotation-solver-test.cc:222-250
    assert synth.angular_error(Rexp, g["R"]) < 1e-5
    g = ctx.gnc_tls_rotation(src, src, 1e-3, 1.4, 100, 1e-12)
    assert synth.angular_error(np.eye(3), g["R"]) < 1e-5


# ------------------------------------------------------------------ stage 4: TLS translation / scalar TLS
def test_translation_kat(ctx):
    d = os.path.join(synth.GOLDEN_DIR, "registration_test")
    v1 = np.loadtxt(os.path.join(d, "translation_test_v1_inliers.csv"), delimiter=",").T
    v2 = np.loadtxt(os.path.join(d, "translation_test_v2_inliers.csv"), delimiter=",").T
    t, inl = ctx.tls_translation(v1, v2, 0.00673642835, 1.0)
    exp = np.array([-0.098430131086161, 0.008679113091532, 0.197317864174211])
    assert np.linalg.norm(t - exp) < 1e-5  # translation-solver-test.cc:98-110
    ot, oinl = orc.tls_translation(v1, v2, 0.00673642835, 1.0)
    assert np.array_equal(t, ot) and np.array_equal(inl, oinl)  # same accumulation order -> bit-exact


@pytest.mark.parametrize("seed", range(4))
def test_translation_random(ctx, seed):
    rng = np.random.default_rng(seed)
    m = int(rng.integers(5, 700))
    src = rng.normal(size=(m, 3))
    t0 = rng.normal(size=3)
    dst = src + t0 + rng.uniform(-0.01, 0.01, size=(m, 3))
    k = m // 4
    dst[:k] += rng.normal(size=(k, 3)) * 3
    t, inl = ctx.tls_translation(src, dst, 0.02, 1.0)
    ot, oinl = orc.tls_translation(src, dst, 0.02, 1.0)
    assert np.allclose(t, ot, atol=1e-12)
    assert np.array_equal(inl, oinl)


@pytest.mark.parametrize("X,r,ref", [
    ([0.5, 1, 0.6, 0.7, 1.2], [0.9, 0.9, 0.4, 0.5, 0.4], 0.8383),
    ([0.5, 1, 0.6, 0.7, 1.2, 10], [0.9, 0.9, 0.4, 0.5, 0.4, 0.5], 0.8383),
    ([0.5, 1, 0.6, 20, 16, 10], [0.9, 0.9, 0.4, 0.5, 0.4, 0.5], 0.6425)])
def test_scalar_tls_kat(ctx, X, r, ref):  # tls-test.cc:21-86
    est, inl = ctx.scalar_tls(X, r)
    oest, oinl = orc.scalar_tls(X, r)
    assert abs(est - ref) < 1e-3
    assert est == oest and np.array_equal(inl, oinl)


# ------------------------------------------------------------------ whole path
SOLVE_CASES = [("C2", 800), ("C2cube", 1200), ("C3", 2500), ("C4", 600), ("C5", 1500)]


@pytest.mark.parametrize("cfg,n", SOLVE_CASES)
def test_solve_vs_oracle(ctx, cfg, n):
    pr = synth.config_problem(cfg, 2, n=n)
    kw = fixed_params(pr["noise_bound"])
    o = orc.solve(pr["src"], pr["dst"], orc.default_params(**kw))
    g = ctx.solve(pr["src"], pr["dst"], capi.default_params(**kw))
    assert g["valid"] and o["valid"]
    assert np.array_equal(g["clique"], o["clique"])  # identical max-clique inlier index set
    assert g["proven"]
    assert g["n_edges"] == o["sol"].n_edges
    assert synth.angular_error(o["R"], g["R"]) <= ROT_TOL
    assert np.linalg.norm(o["t"] - g["t"]) <= TRANS_TOL
    assert g["scale"] == 1.0
    assert np.array_equal(g["trans_inliers"], o["trans_inliers"])
    assert np.mean(g["rot_inliers"] != o["rot_inliers"]) <= 0.01


def test_solve_bunny_c1(ctx):
    """BASELINE config C1 (examples/teaser_cpp_ply/teaser_cpp_ply.cc) with a fixed seed."""
    pr = synth.bunny_problem(os.path.join(synth.GOLDEN_DIR, "bun_zipper_res3.ply"))
    kw = fixed_params(pr["noise_bound"], rotation_cost_threshold=0.005)
    o = orc.solve(pr["src"], pr["dst"], orc.default_params(**kw))
    g = ctx.solve(pr["src"], pr["dst"], capi.default_params(**kw))
    assert np.array_equal(g["clique"], o["clique"])
    assert synth.angular_error(o["R"], g["R"]) <= ROT_TOL
    assert np.linalg.norm(o["t"] - g["t"]) <= TRANS_TOL
    assert synth.angular_error(pr["R"], g["R"]) < 0.01 and np.linalg.norm(pr["t"] - g["t"]) < 0.01


def test_solve_invalid_when_no_clique(ctx):
    rng = np.random.default_rng(0)
    src = rng.uniform(size=(50, 3))
    dst = rng.uniform(size=(50, 3)) * 100
    kw = fixed_params(1e-6)
    g = ctx.solve(src, dst, capi.default_params(**kw))
    o = orc.solve(src, dst, orc.default_params(**kw))
    assert g["valid"] == o["valid"]
    if not o["valid"]:
        assert len(g["clique"]) <= 1


def test_solve_outlier_detection_identity(ctx):  # registration-test.cc:394-467
    for n_out in range(1, 6):
        rng = np.random.default_rng(100 + n_out)
        N = 20
        src = rng.uniform(-1, 1, size=(N, 3))
        R = synth.random_rotation(rng)
        t = rng.uniform(-1, 1, size=3)
        dst = src @ R.T + t
        out_idx = np.sort(rng.choice(N, size=n_out, replace=False))
        dst[out_idx] += rng.uniform(5, 10, size=(n_out, 3))
        g = ctx.solve(src, dst, capi.default_params(**fixed_params(1e-3, rotation_cost_threshold=0.005)))
        assert synth.angular_error(R, g["R"]) <= 0.2 and np.linalg.norm(g["t"] - t) <= 0.1
        assert g["clique"].tolist() == sorted(set(range(N)) - set(out_idx.tolist()))


def test_solve_none_mode(ctx):
    pr = synth.config_problem("C2", 9, n=300)
    src, dst = pr["src"][pr["inliers"]], pr["dst"][pr["inliers"]]
    kw = fixed_params(pr["noise_bound"], inlier_selection_mode=3)
    o = orc.solve(src, dst, orc.default_params(**kw))
    g = ctx.solve(src, dst, capi.default_params(**kw))
    assert len(g["clique"]) == len(src)
    assert synth.angular_error(o["R"], g["R"]) <= ROT_TOL and np.linalg.norm(o["t"] - g["t"]) <= TRANS_TOL


def test_solve_batch_matches_single(ctx):
    prs = [synth.config_problem("C4", b, n=500) for b in range(12)]
    p = capi.default_params(**fixed_params(prs[0]["noise_bound"]))
    sols, cliques = ctx.solve_batch([q["src"] for q in prs], [q["dst"] for q in prs], p)
    for b, q in enumerate(prs):
        g = ctx.solve(q["src"], q["dst"], p)
        assert np.array_equal(cliques[b], g["clique"])
        assert np.array_equal(capi.rotation_from_solution_record(sols[b]), g["R"])
        assert np.array_equal(sols[b]["translation"], g["t"])
        assert np.array_equal(cliques[b], q["inliers"])


def test_solve_batch_array_matches_list_api(ctx):
    prs = [synth.config_problem("C4", 100 + b, n=400) for b in range(70)]  # >= 64 -> chunked copy/compute overlap
    src = np.ascontiguousarray(np.stack([q["src"] for q in prs]))
    dst = np.ascontiguousarray(np.stack([q["dst"] for q in prs]))
    p = capi.default_params(**fixed_params(prs[0]["noise_bound"]))
    sols, cl = ctx.solve_batch_array(src, dst, p)
    sols2, cliques2 = ctx.solve_batch([q["src"] for q in prs], [q["dst"] for q in prs], p)
    for b in range(len(prs)):
        m = sols[b]["clique_size"]
        assert np.array_equal(cl[b, :m], cliques2[b]) and np.array_equal(cl[b, :m], prs[b]["inliers"])
        assert np.array_equal(sols[b]["rotation"], sols2[b]["rotation"])
        assert np.array_equal(sols[b]["translation"], sols2[b]["translation"])


def test_solve_batch_ragged(ctx):
    prs = [synth.config_problem("C2", b, n=n) for b, n in enumerate([200, 333, 64, 500])]
    p = capi.default_params(**fixed_params(prs[0]["noise_bound"]))
    sols, cliques = ctx.solve_batch([q["src"] for q in prs], [q["dst"] for q in prs], p)
    for b, q in enumerate(prs):
        o = orc.solve(q["src"], q["dst"], orc.default_params(**fixed_params(q["noise_bound"])))
        assert np.array_equal(cliques[b], o["clique"])
        assert synth.angular_error(o["R"], capi.rotation_from_solution_record(sols[b])) <= ROT_TOL


def test_solve_batch_ragged_groups_by_size(ctx):
    """Mixed sizes with repeats: problems of equal n travel as one device batch, results return in caller order."""
    sizes = [300, 150, 300, 64, 150, 300, 2, 150]
    prs = [synth.config_problem("C2", b, n=n) for b, n in enumerate(sizes)]
    p = capi.default_params(**fixed_params(prs[0]["noise_bound"]))
    sols, cliques = ctx.solve_batch([q["src"] for q in prs], [q["dst"] for q in prs], p)
    for b, q in enumerate(prs):
        one = ctx.solve(q["src"], q["dst"], p)
        assert bool(sols[b]["valid"]) == one["valid"]
        assert np.array_equal(cliques[b], one["clique"])
        if one["valid"]:
            assert np.allclose(capi.rotation_from_solution_record(sols[b]), one["R"], atol=1e-12)


def test_solve_full_size_c2(ctx):
    pr = synth.config_problem("C2", 0)
    kw = fixed_params(pr["noise_bound"])
    o = orc.solve(pr["src"], pr["dst"], orc.default_params(**kw))
    g = ctx.solve(pr["src"], pr["dst"], capi.default_params(**kw))
    assert np.array_equal(g["clique"], o["clique"]) and np.array_equal(g["clique"], pr["inliers"])
    assert synth.angular_error(o["R"], g["R"]) <= ROT_TOL and np.linalg.norm(o["t"] - g["t"]) <= TRANS_TOL


# ------------------------------------------------------------------ unknown scale (Params default) + golden fixtures
BENCH_TOL = {1: (1e-5,) * 6, 2: (1e-5,) * 6, 3: (1e-5,) * 6, 4: (1e-5,) * 6, 5: (1e-5,) * 6,
             6: (1e-2, 1e-2, 2e-2, 1e-5, 1e-3, 1e-3)}  # registration-benchmark.cc:276-374


def _load_benchmark(i):
    d = os.path.join(synth.GOLDEN_DIR, f"benchmark_{i}")
    src = synth.read_ply_vertices(os.path.join(d, "src.ply"))
    dst = synth.read_ply_vertices(os.path.join(d, "dst.ply"))
    nb = [float(l.split(":")[1]) for l in open(os.path.join(d, "parameters.txt")) if l.startswith("Noise Bound")][0]
    g = {k: np.loadtxt(os.path.join(d, f"{k}.csv"), delimiter=",", ndmin=2)
         for k in ("R_ref", "R_est", "t_ref", "t_est", "s_ref", "s_est")}
    return src, dst, nb, g


@pytest.mark.parametrize("i", [1, 2, 3, 4, 5, 6])
def test_benchmark_fixture_gpu(ctx, i):
    """The reference's end-to-end known-answer fixtures (test/benchmark/registration-benchmark.cc) through the
    GPU path with the reference's own parameters (estimate_scaling = true, GNC-TLS, cost_thr 1e-12)."""
    src, dst, nb, g = _load_benchmark(i)
    kw = dict(noise_bound=nb, cbar2=1.0, estimate_scaling=1, rotation_max_iterations=100, rotation_gnc_factor=1.4,
              rotation_estimation_algorithm=0, rotation_cost_threshold=1e-12)
    out = ctx.solve(src, dst, capi.default_params(**kw))
    o = orc.solve(src, dst, orc.default_params(**kw))
    tol = BENCH_TOL[i]
    assert out["valid"]
    assert abs(out["scale"] - g["s_ref"].item()) <= tol[0]
    assert synth.angular_error(g["R_ref"], out["R"]) <= tol[1]
    assert np.linalg.norm(out["t"] - g["t_ref"].ravel()) <= tol[2]
    assert abs(out["scale"] - g["s_est"].item()) <= tol[3]
    assert synth.angular_error(g["R_est"], out["R"]) <= tol[4]
    assert np.linalg.norm(out["t"] - g["t_est"].ravel()) <= tol[5]
    # and against the oracle on identical inputs
    assert np.array_equal(out["clique"], o["clique"])
    assert abs(out["scale"] - o["scale"]) <= 1e-12
    assert synth.angular_error(o["R"], out["R"]) <= ROT_TOL and np.linalg.norm(o["t"] - out["t"]) <= TRANS_TOL


def test_unknown_scale_object_scene(ctx):
    d = os.path.join(synth.GOLDEN_DIR, "registration_test")
    obj = np.loadtxt(os.path.join(d, "objectIn.csv"), delimiter=",").T
    scene = np.loadtxt(os.path.join(d, "sceneIn.csv"), delimiter=",").T
    kw = dict(noise_bound=0.0067364, estimate_scaling=1, rotation_cost_threshold=1e-12)
    g = ctx.solve(obj, scene, capi.default_params(**kw))
    o = orc.solve(obj, scene, orc.default_params(**kw))
    assert abs(g["scale"] - 0.955885) < 1e-4  # registration-test.cc:313
    assert abs(g["scale"] - o["scale"]) <= 1e-12
    assert np.array_equal(g["clique"], o["clique"])
    assert synth.angular_error(o["R"], g["R"]) <= ROT_TOL and np.linalg.norm(o["t"] - g["t"]) <= TRANS_TOL


@pytest.mark.parametrize("scale", [0.5, 1.0, 2.7])
def test_unknown_scale_synthetic(ctx, scale):
    pr = synth.make_problem(400, 0.5, 4242, "ball")
    dst = pr["dst"] * scale
    kw = dict(noise_bound=pr["noise_bound"] * scale, estimate_scaling=1, rotation_cost_threshold=1e-12)
    g = ctx.solve(pr["src"], dst, capi.default_params(**kw))
    o = orc.solve(pr["src"], dst, orc.default_params(**kw))
    assert abs(g["scale"] - o["scale"]) <= 1e-10 and abs(g["scale"] - scale) < 0.02 * scale
    assert np.array_equal(g["clique"], o["clique"])
    assert g["n_edges"] == o["sol"].n_edges
    assert synth.angular_error(o["R"], g["R"]) <= ROT_TOL and np.linalg.norm(o["t"] - g["t"]) <= TRANS_TOL


def test_unknown_scale_outlier_dominated(ctx):
    """90 % ball outliers: the TLS scale consensus is NOT the true scale — GPU and oracle must still agree."""
    pr = synth.config_problem("C4", 4, n=500)
    kw = dict(noise_bound=pr["noise_bound"], estimate_scaling=1, rotation_cost_threshold=1e-12)
    g = ctx.solve(pr["src"], pr["dst"], capi.default_params(**kw))
    o = orc.solve(pr["src"], pr["dst"], orc.default_params(**kw))
    assert abs(g["scale"] - o["scale"]) <= 1e-10
    assert np.array_equal(g["clique"], o["clique"]) and g["n_edges"] == o["sol"].n_edges
    assert g["valid"] == o["valid"]
    if o["valid"]:
        assert synth.angular_error(o["R"], g["R"]) <= ROT_TOL and np.linalg.norm(o["t"] - g["t"]) <= TRANS_TOL




# ------------------------------------------------------------------ drop-in surfaces above the C-ABI
def test_pybind_facade_matches_capi(ctx):
    """teaserpp_python (pybind11 over the C++ façade) gives the same answer as the raw C-ABI call."""
    import subprocess
    import sys
    host = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "teaser-plusplus_b200", "host")
    subprocess.check_call(["make", "-s", "-C", host])
    sys.path.insert(0, os.path.join(host, "python"))
    import teaserpp_python as tp
    pr = synth.config_problem("C4", 7, n=700)
    p = tp.RobustRegistrationSolver.Params()
    p.noise_bound = pr["noise_bound"]
    p.estimate_scaling = False
    p.rotation_cost_threshold = 1e-12
    s = tp.RobustRegistrationSolver(p)
    sol = s.solve(pr["src"].T, pr["dst"].T)  # the reference API takes (3, N)
    g = ctx.solve(pr["src"], pr["dst"], capi.default_params(**fixed_params(pr["noise_bound"])))
    assert sol.valid and np.array_equal(np.array(s.getInlierMaxClique()), g["clique"])
    assert np.array_equal(sol.rotation, g["R"]) and np.array_equal(sol.translation, g["t"]) and sol.scale == 1.0
    assert np.array_equal(s.getTranslationInliersMask(), g["trans_inliers"])
    assert np.array_equal(s.getRotationInliersMask(), g["rot_inliers"])
    assert s.getTranslationInliers() == np.nonzero(g["trans_inliers"])[0].tolist()
    assert s.isMaxCliqueProvenOptimal()
    # lazy O(N^2) getters agree with the oracle's materialised versions
    adj = s.getInlierGraph()
    obits, odeg, oe = orc.build_graph_bits(pr["src"], pr["dst"], pr["noise_bound"])
    assert [len(a) for a in adj] == odeg.tolist() and s.getNumInlierGraphEdges() == oe
    mask = s.getScaleInliersMask()
    tims = s.getSrcTIMs()
    assert mask.shape[0] == 700 * 699 // 2 and int(mask.sum()) == oe and tims.shape == (3, 700 * 699 // 2)
    assert np.array_equal(tims[:, 0], pr["src"][1] - pr["src"][0])
    # a second solve on the same object is clean (the reference compounds state, SURVEY Q2)
    sol2 = s.solve(pr["src"].T, pr["dst"].T)
    assert np.array_equal(sol2.rotation, sol.rotation) and s.getRotationInliers() == np.nonzero(g["rot_inliers"])[0].tolist()
    # decoupled sub-solver entry points
    t = s.solveForTranslation(pr["src"][pr["inliers"]].T, (pr["src"][pr["inliers"]] + np.array([1.0, 2.0, 3.0])).T) \
        if hasattr(s, "solveForTranslation") else None


def test_cpp_example_bunny():
    """The reference's C++ quick-start, compiled against the drop-in header, runs on the GPU."""
    import subprocess
    host = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "teaser-plusplus_b200", "host")
    subprocess.check_call(["make", "-s", "-C", host])
    out = subprocess.run([os.path.join(host, "example_cpp_ply"), os.path.join(synth.GOLDEN_DIR, "bun_zipper_res3.ply")],
                         capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    vals = {l.split(":")[0]: float(l.split(":")[1]) for l in out.stdout.strip().splitlines()}
    assert vals["rotation error (rad)"] < 0.01 and vals["translation error (m)"] < 0.01
    assert vals["clique size"] > 500


# ------------------------------------------------------------------ other rotation back-ends / TIM graphs (SURVEY §8f-2)
@pytest.mark.parametrize("i", [1, 2, 3, 4, 5, 6])
def test_benchmark_fixture_gpu_fgr(ctx, i):
    """registration-benchmark.cc runs every fixture with FGR too (cost threshold 0.005)."""
    src, dst, nb, g = _load_benchmark(i)
    kw = dict(noise_bound=nb, cbar2=1.0, estimate_scaling=1, rotation_max_iterations=100, rotation_gnc_factor=1.4,
              rotation_estimation_algorithm=1, rotation_cost_threshold=0.005)
    out = ctx.solve(src, dst, capi.default_params(**kw))
    o = orc.solve(src, dst, orc.default_params(**kw))
    tol = BENCH_TOL[i]
    assert abs(out["scale"] - g["s_ref"].item()) <= tol[0]
    assert synth.angular_error(g["R_ref"], out["R"]) <= tol[1]
    assert np.linalg.norm(out["t"] - g["t_ref"].ravel()) <= tol[2]
    assert synth.angular_error(g["R_est"], out["R"]) <= tol[4]
    assert np.linalg.norm(out["t"] - g["t_est"].ravel()) <= tol[5]
    assert np.array_equal(out["clique"], o["clique"])
    assert synth.angular_error(o["R"], out["R"]) <= ROT_TOL and np.linalg.norm(o["t"] - out["t"]) <= TRANS_TOL
    assert out["gnc_iterations"] == o["gnc_iterations"]


def test_object_scene_fgr(ctx):  # registration-test.cc:256-392
    d = os.path.join(synth.GOLDEN_DIR, "registration_test")
    obj = np.loadtxt(os.path.join(d, "objectIn.csv"), delimiter=",").T
    scene = np.loadtxt(os.path.join(d, "sceneIn.csv"), delimiter=",").T
    Rexp = np.array([[0.9974, -0.0199, -0.0696], [0.0138, 0.9961, -0.0875], [0.0710, 0.0863, 0.9937]])
    texp = np.array([-0.1011, 0.0908, 0.1344])
    for es, rtol, ttol in ((1, 0.25, 0.15), (0, 0.2, 0.1)):
        kw = dict(noise_bound=0.0067364, estimate_scaling=es, rotation_estimation_algorithm=1,
                  rotation_cost_threshold=0.005)
        g = ctx.solve(obj, scene, capi.default_params(**kw))
        o = orc.solve(obj, scene, orc.default_params(**kw))
        assert synth.angular_error(Rexp, g["R"]) < rtol and np.linalg.norm(g["t"] - texp) < ttol
        assert synth.angular_error(o["R"], g["R"]) <= ROT_TOL and np.linalg.norm(o["t"] - g["t"]) <= TRANS_TOL
        assert np.array_equal(g["clique"], o["clique"])
        assert np.array_equal(g["rot_inliers"], o["rot_inliers"])  # l_pq.cast<bool>()


@pytest.mark.parametrize("alg,graph", [(1, 0), (2, 0), (0, 1), (1, 1), (2, 1)])
def test_solve_rotation_variants(ctx, alg, graph):
    """FGR / Quatro back-ends and the COMPLETE TIM graph, against the oracle on identical inputs."""
    rng = np.random.default_rng(50 + alg * 2 + graph)
    n = 400
    src = rng.uniform(size=(n, 3))
    if alg == 2:  # Quatro estimates yaw only
        a = 0.6
        R = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1.0]])
    else:
        R = synth.random_rotation(rng)
    t = rng.uniform(-1, 1, size=3)
    nb = 0.02
    noise = rng.normal(size=(n, 3))
    noise *= (rng.uniform(0, 0.9, size=(n, 1)) * nb) / np.linalg.norm(noise, axis=1, keepdims=True)
    dst = src @ R.T + t + noise
    out_idx = rng.choice(n, size=int(0.8 * n), replace=False)
    dst[out_idx] = rng.uniform(-3, 3, size=(len(out_idx), 3))
    kw = dict(noise_bound=nb, estimate_scaling=0, rotation_estimation_algorithm=alg, rotation_tim_graph=graph,
              rotation_cost_threshold=0.005 if alg == 1 else 1e-9)
    g = ctx.solve(src, dst, capi.default_params(**kw))
    o = orc.solve(src, dst, orc.default_params(**kw))
    assert g["valid"] and np.array_equal(g["clique"], o["clique"])
    assert synth.angular_error(o["R"], g["R"]) <= ROT_TOL and np.linalg.norm(o["t"] - g["t"]) <= TRANS_TOL
    assert len(g["rot_inliers"]) == len(o["rot_inliers"])
    assert np.mean(g["rot_inliers"] != o["rot_inliers"]) <= 0.01
    assert synth.angular_error(R, g["R"]) < 0.05 and np.linalg.norm(t - g["t"]) < 0.05


# ------------------------------------------------------------------ KCORE_HEU / PMC_HEU inlier selection modes
def test_kcore_heu_shortcut(ctx):  # graph.cc:66-81
    rng = np.random.default_rng(5)
    n = 300
    A = np.triu(rng.uniform(size=(n, n)) < 0.05, 1)
    idx = rng.choice(n, size=200, replace=False)
    A[np.ix_(idx, idx)] = True
    A = np.triu(A, 1)
    A = A | A.T
    bits = _bits_from_dense(A)
    oc, info = orc.max_clique_bits(bits, n, mode=2, kcore_thr=0.5)
    gc, proven = ctx.max_clique(bits, n, mode=2, kcore_thr=0.5)
    assert info["max_core"] > 150
    assert np.array_equal(gc, oc) and not proven
    # threshold 1 short-circuits the comparison -> heuristic clique (valid, maybe not maximum)
    gc, proven = ctx.max_clique(bits, n, mode=2, kcore_thr=1.0)
    assert len(gc) >= 150 and all(A[a, b] for a in gc for b in gc if a != b)


def test_kcore_heu_below_threshold_and_pmc_heu(ctx):
    pr = synth.config_problem("C2cube", 3, n=900)
    bits, deg, ne = ctx.graph_build(pr["src"], pr["dst"], 2 * pr["noise_bound"])
    b = np.unpackbits(bits.view(np.uint8), axis=1, bitorder="little")[:, :900].astype(bool)
    for mode in (1, 2):
        gc, proven = ctx.max_clique(bits, 900, mode=mode, kcore_thr=0.5)
        assert not proven and len(gc) >= len(pr["inliers"])
        assert all(b[x, y] for x in gc for y in gc if x != y)


def test_solve_kcore_heu_mode(ctx):
    pr = synth.make_problem(500, 0.3, 99, "ball")  # 70 % inliers: max_core = 349 > 0.5 * 500
    kw = fixed_params(pr["noise_bound"], inlier_selection_mode=2, kcore_heuristic_threshold=0.5)
    o = orc.solve(pr["src"], pr["dst"], orc.default_params(**kw))
    g = ctx.solve(pr["src"], pr["dst"], capi.default_params(**kw))
    assert np.array_equal(g["clique"], o["clique"]) and not g["proven"]
    assert synth.angular_error(o["R"], g["R"]) <= ROT_TOL and np.linalg.norm(o["t"] - g["t"]) <= TRANS_TOL


def test_unknown_scale_large_n(ctx):
    """n above the single-CTA limit: radix-sort + deterministic-scan TLS (K = 2 M pairs here)."""
    pr = synth.make_problem(2000, 0.6, 777, "ball")
    scale = 1.7
    dst = pr["dst"] * scale
    kw = dict(noise_bound=pr["noise_bound"] * scale, estimate_scaling=1, rotation_cost_threshold=1e-12)
    g = ctx.solve(pr["src"], dst, capi.default_params(**kw))
    o = orc.solve(pr["src"], dst, orc.default_params(**kw))
    assert abs(g["scale"] - o["scale"]) <= 1e-9 * scale  # different association of the running sums
    assert abs(g["scale"] - scale) < 0.02 * scale
    assert np.array_equal(g["clique"], o["clique"])
    # The inlier graph may differ from the oracle's ONLY on pairs whose exact predicate margin
    # | |d2/d1 - s| - beta/d1 | is below the difference of the two scale estimates (the predicate is evaluated with the
    # reference's exact sequence on both sides; only s differs, by the association of the running sums).
    n = pr["src"].shape[0]
    W = (n + 63) // 64
    gb = np.zeros((n, W), dtype=np.uint64)
    ctx._ck(capi.lib().tzr_last_graph(ctx._h, 0, capi._p(gb, capi.C.c_uint64), None))
    ob = orc.solve(pr["src"], dst, orc.default_params(**kw), want_adj=True)["adj_bits"]
    diff = np.unpackbits((gb ^ ob).view(np.uint8), axis=1, bitorder="little")[:, :n]
    ii, jj = np.nonzero(diff)
    assert len(ii) <= 2 * abs(g["n_edges"] - o["sol"].n_edges) + 8 and len(ii) <= 16
    beta = 2 * kw["noise_bound"]
    for i, j in zip(ii, jj):
        d1 = np.sqrt(((pr["src"][j] - pr["src"][i]) ** 2).sum())
        d2 = np.sqrt(((dst[j] - dst[i]) ** 2).sum())
        margin = abs(abs(d2 / d1 - o["scale"]) - beta / d1)
        assert margin <= 2 * abs(g["scale"] - o["scale"]) + 1e-14, (i, j, margin)
    assert synth.angular_error(o["R"], g["R"]) <= ROT_TOL and np.linalg.norm(o["t"] - g["t"]) <= TRANS_TOL


# ------------------------------------------------------------------ full-size stress configs (BASELINE C3 / C5)
@pytest.mark.parametrize("cfg", ["C3", "C5", "C2cube"])
def test_solve_full_size_stress(ctx, cfg):
    """BASELINE configs C3 (N=10000, 99 % in-cube outliers: max-clique stress), C5 (N=8000, 97 %) and the in-cube
    variant of C2 at full size: identical clique vs the oracle, rotation/translation within tolerance."""
    pr = synth.config_problem(cfg, 0)
    kw = fixed_params(pr["noise_bound"])
    g = ctx.solve(pr["src"], pr["dst"], capi.default_params(**kw))
    o = orc.solve(pr["src"], pr["dst"], orc.default_params(**kw))
    print(cfg, "gpu stage ms", [round(x, 3) for x in g["stage_ms"][:7]], "clique", len(g["clique"]),
          "oracle stage ms", [round(x, 1) for x in o["stage_ms"][:7]])
    assert g["proven"]
    assert np.array_equal(g["clique"], o["clique"])
    assert g["n_edges"] == o["sol"].n_edges
    assert synth.angular_error(o["R"], g["R"]) <= ROT_TOL and np.linalg.norm(o["t"] - g["t"]) <= TRANS_TOL


def test_clique_time_limit_is_honoured(ctx):
    """A tiny max_clique_time_limit stops the exact search: the result is a valid clique, flagged as not proven."""
    rng = np.random.default_rng(1)
    n = 600
    A = np.triu(rng.uniform(size=(n, n)) < 0.5, 1)
    A = A | A.T
    bits = _bits_from_dense(A)
    gc, proven = ctx.max_clique(bits, n, mode=0, time_limit=1e-6)
    assert not proven and len(gc) >= 2
    assert all(A[a, b] for a in gc for b in gc if a != b)


def test_batch_c4_shape(ctx):
    """BASELINE config C4 shape (N=2000, 90 % outliers) as a batch: every problem recovers its planted inlier set
    (or a superset containing it) and the ground-truth pose; a sample is compared with the oracle."""
    B = 96
    prs = [synth.config_problem("C4", b) for b in range(B)]
    src = np.ascontiguousarray(np.stack([q["src"] for q in prs]))
    dst = np.ascontiguousarray(np.stack([q["dst"] for q in prs]))
    p = capi.default_params(**fixed_params(prs[0]["noise_bound"]))
    sols, cl = ctx.solve_batch_array(src, dst, p)
    for b in range(B):
        m = sols[b]["clique_size"]
        assert sols[b]["valid"] and sols[b]["clique_proven_optimal"] == 1
        assert set(prs[b]["inliers"].tolist()) <= set(cl[b, :m].tolist())
        R = capi.rotation_from_solution_record(sols[b])
        assert synth.angular_error(prs[b]["R"], R) < 0.02 and np.linalg.norm(prs[b]["t"] - sols[b]["translation"]) < 0.02
    for b in (0, 17, 95):
        o = orc.solve(prs[b]["src"], prs[b]["dst"], orc.default_params(**fixed_params(prs[b]["noise_bound"])))
        m = sols[b]["clique_size"]
        assert np.array_equal(cl[b, :m], o["clique"])
        assert synth.angular_error(o["R"], capi.rotation_from_solution_record(sols[b])) <= ROT_TOL
        assert np.linalg.norm(o["t"] - sols[b]["translation"]) <= TRANS_TOL


def test_standalone_rotation_backends_kat(ctx):
    """FGR and Quatro on caller-supplied TIMs (rotation-solver-test.cc:23-135, registration-test.cc:144-218)."""
    src = np.loadtxt(os.path.join(synth.GOLDEN_DIR, "registration_test", "rotation_only_src.csv"), delimiter=",")
    Rexp = np.array([[0.997379773225804, -0.019905935977315, -0.069551000516966],
                     [0.013777311189888, 0.996068297974922, -0.087510750572249],
                     [0.071019530105605, 0.086323226782879, 0.993732623426126]])
    g = ctx.rotation_solve(1, src, src @ Rexp.T, 1e-3, 1.4, 100, 1e-12)
    o = orc.fgr(src, src @ Rexp.T, 100, 1e-12, 1.4, 1e-3)
    # acos near 1 resolves angles only to ~sqrt(eps) = 1.5e-8 rad
    assert synth.angular_error(Rexp, g["R"]) < 1e-5 and synth.angular_error(o["R"], g["R"]) < 1e-6
    assert abs(g["iterations"] - o["iterations"]) <= 3  # the cost < 1e-12 stop acts on rounding noise here
    Ryaw = np.array([[0.997379773225804, -0.072343541246221, 0.0], [0.072343541246221, 0.997379773225804, 0.0],
                     [0.0, 0.0, 1.0]])
    g = ctx.rotation_solve(2, src, src @ Ryaw.T, 0.0067364, 1.4, 100, 0.005)
    assert synth.angular_error(Ryaw, g["R"]) < 1e-5
    rng = np.random.default_rng(3)
    dst = src @ Ryaw.T
    dst[:40] += rng.normal(size=(40, 3))
    g = ctx.rotation_solve(2, src, dst, 0.01, 1.4, 100, 1e-9)
    o = orc.quatro(src, dst, 100, 1e-9, 1.4, 0.01)
    assert synth.angular_error(o["R"], g["R"]) < 1e-6 and np.mean(g["inliers"] != o["inliers"]) < 0.02


# ------------------------------------------------------------------ size edges
@pytest.mark.parametrize("n", [1, 2, 3, 4])
def test_tiny_problems_match_oracle(ctx, n):
    """n = 1 has no TIM at all, n = 2 a single one: validity and values must follow registration.cc:643-647."""
    rng = np.random.default_rng(n)
    R = synth.random_rotation(rng)
    src = rng.uniform(size=(n, 3))
    dst = (R @ src.T).T + 0.3
    kw = fixed_params(0.01)
    out = ctx.solve(src, dst, capi.default_params(**kw))
    o = orc.solve(src, dst, orc.default_params(**kw))
    assert out["valid"] == o["valid"]
    assert np.array_equal(out["clique"], o["clique"])
    if o["valid"]:
        assert synth.angular_error(out["R"], o["R"]) < ROT_TOL
        assert np.linalg.norm(out["t"] - o["t"]) < TRANS_TOL


def test_maximum_size_problem(ctx):
    """kMaxN = 32768 correspondences: graph properties + planted clique recovered; one more is TZR_ERR_TOO_LARGE."""
    n = 32768
    pr = synth.make_problem(n, 0.995, seed=7, model="ball", sigma=0.01, noise_bound=synth.NOISE_BOUND_SIGMA_001)
    p = capi.default_params(**fixed_params(pr["noise_bound"]))
    out = ctx.solve(pr["src"], pr["dst"], p)
    assert out["valid"]
    inl = np.sort(pr["inliers"])
    assert len(out["clique"]) >= len(inl)
    assert set(inl.tolist()) <= set(out["clique"].tolist())
    assert synth.angular_error(out["R"], pr["R"]) < 0.02 and np.linalg.norm(out["t"] - pr["t"]) < 0.02
    bits, deg = ctx.last_graph(0, n)
    assert int(deg.sum()) == 2 * out["n_edges"]
    rows = np.random.default_rng(0).integers(0, n, size=6)
    # exact rows against a direct float64 evaluation of the predicate (registration.cc:427-443)
    beta = 2 * pr["noise_bound"]
    for r in rows:
        ds = np.sqrt(((pr["src"] - pr["src"][r]) ** 2)[:, 0] + ((pr["src"] - pr["src"][r]) ** 2)[:, 1]
                     + ((pr["src"] - pr["src"][r]) ** 2)[:, 2])
        dd = np.sqrt(((pr["dst"] - pr["dst"][r]) ** 2)[:, 0] + ((pr["dst"] - pr["dst"][r]) ** 2)[:, 1]
                     + ((pr["dst"] - pr["dst"][r]) ** 2)[:, 2])
        want = np.abs(ds - dd) <= beta
        want[r] = False
        got = np.unpackbits(bits[r].view(np.uint8), bitorder="little")[:n].astype(bool)
        assert np.array_equal(got, want)
    with pytest.raises(capi.TzrError):
        big = np.zeros((n + 1, 3))
        ctx.solve(big, big, p)


@pytest.mark.parametrize("ratio,n", [(0.0, 2000), (0.5, 2500), (0.999, 3000)])
def test_outlier_ratio_extremes_vs_oracle(ctx, ratio, n):
    """All-inlier input (complete graph, clique = everything), half outliers, and a 3-inlier needle."""
    pr = synth.make_problem(n, ratio, seed=int(ratio * 1000) + n, model="ball", sigma=0.01,
                            noise_bound=synth.NOISE_BOUND_SIGMA_001)
    kw = fixed_params(pr["noise_bound"])
    out = ctx.solve(pr["src"], pr["dst"], capi.default_params(**kw))
    o = orc.solve(pr["src"], pr["dst"], orc.default_params(**kw))
    assert out["valid"] == o["valid"]
    assert np.array_equal(out["clique"], o["clique"])
    assert out["n_edges"] == int(o["sol"].n_edges)
    if ratio < 0.9:
        assert set(pr["inliers"].tolist()) <= set(out["clique"].tolist())
    assert synth.angular_error(out["R"], o["R"]) < ROT_TOL
    assert np.linalg.norm(out["t"] - o["t"]) < TRANS_TOL


def test_python_example_bunny():
    """host/examples/teaser_python_ply.py: the reference's Python quick-start through the pybind module."""
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    host = os.path.join(root, "teaser-plusplus_b200", "host")
    subprocess.check_call(["make", "-s", "-C", host])
    out = subprocess.run([sys.executable, os.path.join(host, "examples", "teaser_python_ply.py"),
                          os.path.join(synth.GOLDEN_DIR, "bun_zipper_res3.ply")], capture_output=True, text=True,
                         timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    vals = {l.split(":")[0]: float(l.split(":")[1]) for l in out.stdout.strip().splitlines()}
    # noise bound 0.05 on a 0.15 m object (the reference example's own numbers): a loose pose, but a large clique
    # (597 = the optimum, see test_dense_graph_is_closed_by_the_vertex_cover_bound)
    assert vals["rotation error (rad)"] < 0.2 and vals["translation error (m)"] < 0.03
    assert vals["clique size"] == 597
    assert vals["time (s)"] < 5.0


def _python_example_problem():
    rng = np.random.default_rng(1889)
    src = np.transpose(synth.read_ply_vertices(os.path.join(synth.GOLDEN_DIR, "bun_zipper_res3.ply")).astype(np.float64))
    N = src.shape[1]
    T = np.array([[9.96926560e-01, 6.68735757e-02, -4.06664421e-02, -1.15576939e-01],
                  [-6.61289946e-02, 9.97617877e-01, 1.94008687e-02, -3.87705398e-02],
                  [4.18675510e-02, -1.66517807e-02, 9.98977765e-01, 1.14874890e-01], [0, 0, 0, 1]])
    dst = T[:3, :3] @ src + T[:3, 3:4]
    dst += (rng.random((3, N)) - 0.5) * 2 * 0.05
    oi = rng.integers(1700, size=1700)
    for i in range(oi.size):
        dst[:, oi[i]] += (5 + rng.random((3, 1)) * 5).squeeze()
    return np.ascontiguousarray(src.T), np.ascontiguousarray(dst.T)


def test_dense_graph_is_closed_by_the_vertex_cover_bound(ctx):
    """The reference's Python example (noise bound 0.05 on the 0.15 m bunny): 99 % dense graph on ~810 surviving
    vertices, heuristic 596, core bound 742.  Colouring-bound search does not finish (the restatement neither); the
    maximum is 597 (independent check: exact vertex cover of the complement by MILP, 810 - 213).  The NT bound /
    reduction closes it after the first 50 ms pass; the result is a valid clique of that size, flagged 2."""
    import time
    S, D = _python_example_problem()
    p = capi.default_params(noise_bound=0.05, cbar2=1.0, estimate_scaling=0, rotation_cost_threshold=1e-12,
                            max_clique_time_limit=60.0)
    ctx.solve(S, D, p)
    t0 = time.time()
    r = ctx.solve(S, D, p)
    dt = time.time() - t0
    assert r["valid"] and len(r["clique"]) == 597
    assert int(r["sol"].clique_proven_optimal) == 2
    assert dt < 3.0
    bits, _ = ctx.last_graph(0, S.shape[0])
    Adj = np.unpackbits(bits.view(np.uint8), axis=1, bitorder="little")[:, :S.shape[0]].astype(bool)
    c = r["clique"]
    sub = Adj[np.ix_(c, c)]
    assert sub.sum() == len(c) * (len(c) - 1)          # a clique indeed
    obits, _, _ = orc.build_graph_bits(S, D, 0.05)
    assert np.array_equal(bits, obits)                  # on the same graph as the restatement's
    # the restatement takes the same two-pass route (3 s first pass, LP bound, NT reduction, beat-only second pass)
    o = orc.solve(S, D, orc.default_params(noise_bound=0.05, cbar2=1.0, estimate_scaling=0,
                                           rotation_cost_threshold=1e-12, max_clique_time_limit=600.0))
    assert len(o["clique"]) == 597 and int(o["sol"].clique_proven_optimal) == 2


def test_dense_small_instance_same_size_as_oracle(ctx):
    """A 360-point dense instance (tests/test_oracle_dense_cpu.py checks the restatement's answer against a MILP):
    the device returns a valid clique of the same, maximum, size."""
    rng = np.random.default_rng(5)
    n, n_out = 360, 110
    src = rng.uniform(0, 0.15, size=(n, 3))
    dst = src + (rng.random((n, 3)) - 0.5) * 0.1
    dst[:n_out] += 7.0
    bits, deg, ne = ctx.graph_build(src, dst, 0.1)
    obits, _, _ = orc.build_graph_bits(src, dst, 0.05)
    assert np.array_equal(bits, obits)
    c, proven = ctx.max_clique(bits, n, mode=0, time_limit=120.0)
    oc, info = orc.max_clique_bits(obits, n, mode=0, time_limit=300.0)
    A = np.unpackbits(bits.view(np.uint8), axis=1, bitorder="little")[:, :n].astype(bool)
    assert A[np.ix_(c, c)].sum() == len(c) * (len(c) - 1)
    assert proven and not info["timed_out"]
    assert len(c) == len(oc)
