"""tzr_register_cloud_pairs against the chain of existing calls (run on an H100: `pytest -m gpu`).

The chain is the one a caller builds by hand today: tzr_compute_fpfh_batch over the clouds, tzr_match_correspondences_batch
over the pairs whose clouds did not overflow (same seeds), the float points at the correspondences converted to
float64, and tzr_solve_batch over the pairs that can be solved.  For every pair the new call must give the same
correspondences and global scale, and for every solved pair the same record (byte for byte except stage_ms) and clique;
the retained solve (masks, graphs, certification) must be the chain's solve.
"""
import importlib
import os
import subprocess
import sys

import numpy as np
import pytest

capi = importlib.import_module("teaser-plusplus_b200.capi")

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "teaser-plusplus_b200", "host")
STAGE_OFF = capi.SOLUTION_DTYPE.fields["stage_ms"][1]
REC = capi.SOLUTION_DTYPE.itemsize
TOO_LARGE, INVALID = capi.TZR_ERR_TOO_LARGE, capi.TZR_ERR_INVALID_ARG
RN, RF = 0.1, 0.15
NB = 0.01
EXAMPLE = (False, True, False, 0.0)  # examples/teaser_cpp_fpfh: absolute scale off, cross check on, no tuple test
GOLDEN = 0x9E3779B97F4A7C15


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.set_flags(0)
    c.close()


def params(**kw):
    d = dict(noise_bound=NB, cbar2=1.0, estimate_scaling=0, rotation_cost_threshold=1e-12)
    d.update(kw)
    return capi.default_params(**d)


def surface(rng, n):
    uv = rng.uniform(-1, 1, size=(n, 2))
    pts = np.stack([uv[:, 0], uv[:, 1], 0.3 * np.sin(3 * uv[:, 0]) * np.cos(2 * uv[:, 1])], axis=1)
    return (pts + rng.normal(scale=0.003, size=pts.shape) + np.array([0.5, -0.2, 2.0])).astype(np.float32)


def moved(rng, src, n):
    """A scan of the same surface: 2/3 of src's points (when n allows), new samples for the rest, permuted, moved."""
    keep = min(len(src), n - n // 3)
    dst = np.concatenate([src[:keep], surface(rng, n - keep)])[rng.permutation(n)].astype(np.float64)
    a = rng.normal(size=3)
    a *= 0.05 / np.linalg.norm(a)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    R = np.eye(3) + np.sin(0.05) * K / 0.05 + (1 - np.cos(0.05)) * (K @ K) / 0.05 ** 2
    return (dst @ R.T + np.array([0.05, 0.0, 0.0])).astype(np.float32)


def sequence(sizes, seed):
    """Scans k = 0 .. len(sizes) - 1, each a moved partial copy of the one before; pair k is (k, k + 1)."""
    rng = np.random.default_rng(seed)
    clouds = [surface(rng, sizes[0])]
    for n in sizes[1:]:
        clouds.append(moved(rng, clouds[-1], n))
    return clouds, [(k, k + 1) for k in range(len(sizes) - 1)]


def sequence_problem():
    """A small float64 problem for tzr_solve: points of one scan against themselves."""
    clouds, _ = sequence([200], seed=5)
    p = np.ascontiguousarray(clouds[0], dtype=np.float64)
    return p, p.copy()


def chain(ctx, clouds, pairs, prm, flags, seeds, max_n=32768):
    try:
        feats = ctx.compute_fpfh_batch(clouds, RN, RF)
        ovf = np.zeros(len(clouds), dtype=np.int32)
    except capi.TzrError as e:
        feats, ovf = e.result, e.status
    P = len(pairs)
    matched = [p for p, (a, b) in enumerate(pairs) if ovf[a] == 0 and ovf[b] == 0]
    corr, scales = [None] * P, [None] * P
    if matched:
        m, g = ctx.match_correspondences_batch([clouds[pairs[p][0]] for p in matched],
                                               [clouds[pairs[p][1]] for p in matched],
                                               [feats[pairs[p][0]] for p in matched],
                                               [feats[pairs[p][1]] for p in matched], *flags,
                                               tuple_seeds=[seeds[p] for p in matched], return_scale=True)
        for k, p in enumerate(matched):
            corr[p], scales[p] = m[k], g[k]
    solved = [p for p in matched if 0 < len(corr[p]) <= max_n and not (prm.estimate_scaling and len(corr[p]) >= 46341)]
    sols = cliques = None
    if solved:
        src = [np.ascontiguousarray(clouds[pairs[p][0]][corr[p][:, 0]], dtype=np.float64) for p in solved]
        dst = [np.ascontiguousarray(clouds[pairs[p][1]][corr[p][:, 1]], dtype=np.float64) for p in solved]
        sols, cliques = ctx.solve_batch(src, dst, prm)
    return dict(ovf=ovf, corr=corr, scales=scales, solved=solved, sols=sols, cliques=cliques)


def retained(ctx, sizes, certify):
    masks = [ctx.last_inliers(b) for b in range(len(sizes))]
    graphs = [ctx.last_graph(b, n) for b, n in enumerate(sizes)]
    cert = ctx.certify_last(noise_bound=2 * NB, cbar2=1.0) if certify else None
    return masks, graphs, cert


def check(ctx, clouds, pairs, prm, flags=EXAMPLE, seeds=None, retention=False, certify=False):
    """The new call against the chain; returns (status, problem_index, the chain's results)."""
    P = len(pairs)
    seeds = list(range(100, 100 + P)) if seeds is None else seeds
    sols, status, index, corr, cliques, scales = ctx.register_cloud_pairs(clouds, pairs, prm, RN, RF, *flags,
                                                                          tuple_seeds=seeds)
    n_solved = int((index >= 0).sum())
    got = retained(ctx, [len(corr[p]) for p in np.argsort(index) if index[p] >= 0], certify) \
        if retention and n_solved else None
    want = chain(ctx, clouds, pairs, prm, flags, seeds)
    solved = want["solved"]
    for p, (a, b) in enumerate(pairs):
        if want["ovf"][a] or want["ovf"][b]:
            assert status[p] == TOO_LARGE and len(corr[p]) == 0 and index[p] == -1, p
            assert sols[p:p + 1].tobytes() == bytes(REC), p
            continue
        assert np.array_equal(corr[p], want["corr"][p]), p
        assert np.float32(scales[p]).tobytes() == np.float32(want["scales"][p]).tobytes(), p
        if p in solved:
            k = solved.index(p)
            assert status[p] == 0 and index[p] == k, p
            assert sols[p:p + 1].tobytes()[:STAGE_OFF] == want["sols"][k:k + 1].tobytes()[:STAGE_OFF], p
            assert np.array_equal(cliques[p], want["cliques"][k]), p
        else:
            assert status[p] == (INVALID if len(corr[p]) == 0 else TOO_LARGE) and index[p] == -1, p
            assert sols[p:p + 1].tobytes() == bytes(REC) and len(cliques[p]) == 0, p
    assert n_solved == len(solved)
    if got is not None:
        exp = retained(ctx, [len(want["corr"][p]) for p in solved], certify)
        for k in range(len(solved)):
            for x, y in zip(got[0][k], exp[0][k]):
                assert np.array_equal(x, y), k
            for x, y in zip(got[1][k], exp[1][k]):
                assert np.array_equal(x, y), k
        if certify:
            for x, y in zip(got[2], exp[2]):
                assert x["status"] == y["status"] and x["is_optimal"] == y["is_optimal"]
                assert x["best_suboptimality"] == y["best_suboptimality"]
                assert np.array_equal(x["suboptimality_traj"], y["suboptimality_traj"])
    return status, index, want


def test_topology_shared_self_and_both_directions(ctx):
    """One cloud in five pairs, a self pair, (a, b) next to (b, a), ragged sizes on both radius-search routes."""
    rng = np.random.default_rng(3)
    c0 = surface(rng, 700)
    c1 = moved(rng, c0, 650)
    c2 = moved(rng, c0, 900)
    c3 = surface(rng, 4500)            # grid route (n >= 4096)
    c4 = moved(rng, c3, 5000)
    c5 = moved(rng, c3, 1200)          # brute force next to its grid-route source
    clouds = [c0, c1, c2, c3, c4, c5]
    pairs = [(0, 1), (1, 0), (0, 2), (2, 0), (0, 0), (3, 4), (4, 3), (1, 2), (3, 5), (5, 3), (0, 4)]
    status, index, _ = check(ctx, clouds, pairs, params())
    assert (status == 0).all() and list(index) == list(range(len(pairs)))


FLAG_CASES = [(abs_s, cc, tt, ts) for abs_s in (False, True) for cc in (False, True)
              for (tt, ts) in ((False, 0.0), (True, 0.95), (True, 0.0), (False, 0.95))]


@pytest.mark.parametrize("abs_scale,crosscheck,tuple_test,tuple_scale", FLAG_CASES)
def test_every_matcher_flag_combination(ctx, abs_scale, crosscheck, tuple_test, tuple_scale):
    clouds, pairs = sequence([500, 620, 450, 700], seed=11)
    pairs = pairs + [(1, 0), (2, 2)]
    seeds = [7, 7, 2 ** 40 + 17, GOLDEN, 5]   # equal and distinct seeds
    check(ctx, clouds, pairs, params(), flags=(abs_scale, crosscheck, tuple_test, tuple_scale), seeds=seeds)


@pytest.mark.parametrize("solver", [
    dict(estimate_scaling=1),
    dict(rotation_estimation_algorithm=1),
    dict(rotation_estimation_algorithm=2, inlier_selection_mode=2),
    dict(inlier_selection_mode=3),
    dict(inlier_selection_mode=1, estimate_scaling=1),
], ids=["scaling", "fgr", "quatro_kcore", "none", "pmc_heu_scaling"])
def test_solver_settings(ctx, solver):
    clouds, pairs = sequence([400, 520, 300, 640, 480], seed=23)
    check(ctx, clouds, pairs + [(0, 2)], params(**solver))


@pytest.mark.parametrize("solver", [dict(), dict(estimate_scaling=1)], ids=["fixed_scale", "scaling"])
def test_retention_equals_the_chains_solve(ctx, solver):
    """last_inliers, last_graph and certify_last(noise_bound = 2 nb) after the call equal the chain's."""
    clouds, pairs = sequence([300, 360, 280, 330], seed=31)
    check(ctx, clouds, pairs + [(2, 0)], params(**solver), retention=True, certify=True)


def test_overflowing_cloud(ctx):
    rng = np.random.default_rng(41)
    clouds, pairs = sequence([500, 600, 550], seed=41)
    clouds.append(rng.uniform(0, 0.01, size=(5000, 3)).astype(np.float32))  # every point has 5000 neighbours
    pairs = [(0, 1), (3, 0), (1, 2), (3, 3), (2, 3), (2, 0)]
    status, index, want = check(ctx, clouds, pairs, params(), retention=True)
    assert want["ovf"][3] != 0
    assert list(status) == [0, TOO_LARGE, 0, TOO_LARGE, TOO_LARGE, 0]
    assert list(index) == [0, -1, 1, -1, -1, 2]


def test_pair_without_correspondences(ctx):
    """A 1-point pair under the tuple test keeps no correspondence (its only triple is degenerate)."""
    clouds, pairs = sequence([500, 600, 550], seed=43)
    clouds += [np.array([[0.1, 0.2, 0.3]], dtype=np.float32), np.array([[0.4, 0.1, 0.2]], dtype=np.float32)]
    pairs = [(3, 4), (0, 1), (1, 2), (4, 3)]
    status, index, want = check(ctx, clouds, pairs, params(), flags=(False, True, True, 0.95), retention=True)
    assert status[0] == INVALID and status[3] == INVALID and index[0] == index[3] == -1
    assert index[1] == 0 and len(want["corr"][1]) > 0


def test_tuple_scale_one_keeps_nothing(ctx):
    """tuple_scale = 1: the strict tests li * s < lj < li / s never pass, so no pair has a correspondence and no solve
    is retained."""
    clouds, pairs = sequence([500, 600, 550], seed=47)
    ctx.solve(*sequence_problem(), params())   # a solve is retained before the call
    ctx.register_cloud_pairs(clouds, pairs, params(), RN, RF, False, True, True, 1.0)
    with pytest.raises(capi.TzrError):
        ctx.last_inliers(0)
    status, index, _ = check(ctx, clouds, pairs, params(), flags=(False, True, True, 1.0))
    assert (status == INVALID).all() and (index == -1).all()


def test_pair_above_the_context_limit(ctx):
    """Without cross check every target row of the smaller cloud is its own correspondence: two clouds of 33000 points
    give more than 32768, written but not solved, among pairs that are solved."""
    rng = np.random.default_rng(53)
    big_a = rng.uniform(0, 1, size=(33000, 3)).astype(np.float32)
    big_b = rng.uniform(0, 1, size=(33000, 3)).astype(np.float32)
    clouds, pairs = sequence([500, 600], seed=53)
    clouds += [big_a, big_b]
    pairs = pairs + [(2, 3), (1, 0)]
    status, index, want = check(ctx, clouds, pairs, params(), flags=(False, False, False, 0.0), retention=True)
    assert len(want["corr"][1]) > 32768
    assert list(status) == [0, TOO_LARGE, 0] and list(index) == [0, -1, 1]


def test_launch_count(ctx):
    """The call launches what the three batch calls launch plus the two gathers, for any number of pairs."""
    for sizes in ([400, 520, 300, 640], [400 + 37 * k for k in range(17)]):
        clouds, pairs = sequence(sizes, seed=61)
        pairs = pairs + [(0, 2)]
        l0 = ctx.kernel_launches()
        sols, status, index, *_ = ctx.register_cloud_pairs(clouds, pairs, params(), RN, RF, *EXAMPLE)
        new = ctx.kernel_launches() - l0
        assert (status == 0).all()
        l0 = ctx.kernel_launches()
        want = chain(ctx, clouds, pairs, params(), EXAMPLE, [0] * len(pairs))
        assert len({len(c) for c in want["corr"]}) > 1   # a ragged solve in the chain too
        assert new == ctx.kernel_launches() - l0 + 2


def test_cpp_facade_equals_the_facade_chain(tmp_path):
    """RobustRegistrationSolver::solveCloudPairs against FPFHEstimation::computeFPFHFeaturesBatch, a seeded
    Matcher::calculateCorrespondencesBatch and solve(src_cloud, dst_cloud, correspondences) per pair
    (tests/cpp/register_pairs_test.cc)."""
    subprocess.check_call(["make", "-s", "-C", HOST])
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    exe = str(tmp_path / "register_pairs_test")
    csrc = os.path.join(ROOT, "teaser-plusplus_b200", "csrc")
    subprocess.check_call([cxx, "-std=c++17", "-O1", "-I", os.path.join(HOST, "include"), "-I",
                           os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "register_pairs_test.cc"),
                           "-L", HOST, "-lteaser_registration", "-L", csrc, "-lteaser_b200",
                           f"-Wl,-rpath,{HOST}:{csrc}", "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr


def test_pybind_solve_cloud_pairs(ctx):
    subprocess.check_call(["make", "-s", "-C", HOST])
    sys.path.insert(0, os.path.join(HOST, "python"))
    import teaserpp_python as tpp
    clouds, pairs = sequence([400, 520, 300, 640], seed=71)
    pairs = pairs + [(0, 2), (2, 2)]
    seed = 12345
    flags = (False, True, True, 0.95)
    solver = tpp.RobustRegistrationSolver(noise_bound=NB, estimate_scaling=False, rotation_cost_threshold=1e-12)
    out = solver.solve_cloud_pairs(clouds, pairs, RN, RF, *flags, seed)
    seeds = [(seed + GOLDEN * p) % 2 ** 64 for p in range(len(pairs))]
    want = chain(ctx, clouds, pairs, params(), flags, seeds)
    assert len(out) == len(pairs)
    for p, r in enumerate(out):
        assert np.array_equal(np.asarray(r["correspondences"], dtype=np.int32).reshape(-1, 2), want["corr"][p]), p
        assert np.float32(r["global_scale"]).tobytes() == np.float32(want["scales"][p]).tobytes(), p
        if p in want["solved"]:
            k = want["solved"].index(p)
            rec = want["sols"][k]
            assert r["status"] == 0, p
            assert r["solution"].valid == bool(rec["valid"]) and r["solution"].scale == rec["scale"], p
            assert np.array_equal(np.asarray(r["solution"].rotation), capi.rotation_from_solution_record(rec)), p
            assert np.array_equal(np.asarray(r["solution"].translation).ravel(), rec["translation"]), p
            assert np.array_equal(np.asarray(r["max_clique"]), want["cliques"][k]), p
        else:
            assert r["status"] != 0 and not r["solution"].valid and len(r["max_clique"]) == 0, p
