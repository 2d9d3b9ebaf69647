"""Open3D's line process on the device (run on an H100: `pytest -m gpu`): tzr_pose_graph_optimize_line_process against
the numpy restatement (tests/line_process_reference.py) on small graphs, wrong closures, a chain of 200, a complete graph
of 64 nodes and the K = 1024 cap; every stop rule; determinism; the refusals; the launch count; the retained solve; the
chained multiway entry against the chain of public calls, with and without colours."""
import importlib
import os
import subprocess
import sys

import numpy as np
import pytest

import line_process_reference as lp
import pose_graph_reference as pg
from line_process_graphs import graph, rigid
from test_gpu_icp import PAIR_FLAGS, _retained, _sequence
from test_gpu_icp_colored import colours_of

capi = importlib.import_module("teaser-plusplus_b200.capi")

pytestmark = pytest.mark.gpu

R_CORR = 0.05


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


def check(got, want, pose_atol=1e-8):
    assert (got["iterations"], got["trials"], got["stop_reason"]) == \
        (want["iterations"], want["trials"], want["stop_reason"])
    assert np.array_equal(got["kept"], want["kept"]) and got["pruned"] == want["pruned"]
    np.testing.assert_allclose(got["poses"], want["poses"], rtol=0, atol=pose_atol)
    np.testing.assert_allclose(got["confidence"], want["confidence"], rtol=0, atol=1e-8)
    np.testing.assert_allclose(got["mu"], want["mu"], rtol=1e-15, atol=0)
    assert abs(got["residual"] - want["residual"]) <= 1e-8 * max(1.0, abs(want["residual"]))
    np.testing.assert_allclose(got["residuals"], want["residuals"], rtol=1e-6, atol=1e-10)


CASES = {
    "chain": (11, 6, [], []),
    "loops": (12, 12, [(11, 0), (8, 0), (9, 3), (7, 2)], []),
    "complete6": (13, 6, None, []),
    "wrong": (21, 16, [(15, 0), (8, 0), (12, 4)], [(10, 2), (14, 6)]),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_against_the_restatement(ctx, name):
    seed, K, extra, wrong = CASES[name]
    gt, edges, T, L, unc = graph(seed, K, extra or [], wrong=wrong, noise=0.004, complete=extra is None)
    want = lp.optimize(K, edges, T, L, R_CORR, unc)
    got = ctx.global_optimization(K, edges, T, L, R_CORR, uncertain=unc)
    check(got, want)
    if wrong:
        assert not got["kept"][-len(wrong):].any() and got["kept"][:-len(wrong)].all()


def test_chain_of_200(ctx):
    gt, edges, T, L, unc = graph(41, 200, [(199, 0), (150, 20), (100, 60)], wrong=[(120, 10)], noise=0.003)
    check(ctx.global_optimization(200, edges, T, L, R_CORR, uncertain=unc), lp.optimize(200, edges, T, L, R_CORR, unc))


def test_complete_64(ctx):
    gt, edges, T, L, unc = graph(43, 64, None, noise=0.003, complete=True, points=(60, 120))
    check(ctx.global_optimization(64, edges, T, L, R_CORR, uncertain=unc), lp.optimize(64, edges, T, L, R_CORR, unc))


def cap_graph():
    extra = [(k + 37, k) for k in range(0, 980, 61)]
    return graph(47, 1024, extra, wrong=[(500, 3), (900, 450)], noise=0.002, points=(60, 120))


def test_cap_1024_against_the_restatement(ctx):
    gt, edges, T, L, unc = cap_graph()
    got = ctx.global_optimization(1024, edges, T, L, R_CORR, uncertain=unc)
    check(got, lp.optimize(1024, edges, T, L, R_CORR, unc), pose_atol=1e-8)
    assert not got["kept"][-2:].any()


# ---- the stop rules -------------------------------------------------------------------------------------------------------
def test_consistent_graph_stops_on_the_right_term(ctx):
    gt, edges, T, L, unc = graph(51, 7, [(6, 0), (4, 1)], noise=0.0)
    got = ctx.global_optimization(7, edges, T, L, R_CORR, uncertain=unc)
    assert got["iterations"] == [0, 0] and got["trials"] == [0, 0]
    assert got["stop_reason"] == [lp.STOP["right_term"]] * 2
    start = pg.bfs(7, edges, T, [True] * len(edges), unc, 0)
    assert got["poses"].tobytes() == np.stack(start).tobytes()


RULES = {
    "relative_increment": dict(min_relative_residual_increment=0.0),
    "relative_residual": dict(min_relative_increment=0.0),
    "lm_trials": dict(max_iteration_lm=1),
    "min_residual": dict(min_residual=1e12),
    "max_iteration": dict(max_iteration=2, min_relative_increment=0.0, min_relative_residual_increment=0.0),
}


@pytest.mark.parametrize("rule", sorted(RULES))
def test_every_stop_rule(ctx, rule):
    gt, edges, T, L, unc = graph(61, 10, [(9, 0), (7, 2)], wrong=[(8, 1)], noise=0.01)
    want = lp.optimize(10, edges, T, L, R_CORR, unc, **RULES[rule])
    got = ctx.global_optimization(10, edges, T, L, R_CORR, uncertain=unc, **RULES[rule])
    assert want["stop_reason"][0] == lp.STOP[rule]
    check(got, want)


# ---- determinism, defaults, compensation -----------------------------------------------------------------------------------
def test_deterministic_and_explicit_start_equals_the_default(ctx):
    gt, edges, T, L, unc = graph(71, 12, [(11, 0), (6, 1)], wrong=[(9, 3)], noise=0.005)
    a = ctx.global_optimization(12, edges, T, L, R_CORR, uncertain=unc)
    b = ctx.global_optimization(12, edges, T, L, R_CORR, uncertain=unc)
    init = pg.bfs(12, edges, T, [True] * len(edges), unc, 0)
    c = ctx.global_optimization(12, edges, T, L, R_CORR, uncertain=unc, initial_poses=init)
    for k in a:
        assert np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes() == np.asarray(c[k]).tobytes(), k


def test_reference_node_and_compensation(ctx):
    gt, edges, T, L, unc = graph(73, 9, [(8, 0)], noise=0.01)
    rng = np.random.default_rng(5)
    init = [rigid(rng, 0.02, 0.02) @ g for g in gt]
    for ref in (-1, 4):
        got = ctx.global_optimization(9, edges, T, L, R_CORR, uncertain=unc, initial_poses=init, reference_node=ref)
        check(got, lp.optimize(9, edges, T, L, R_CORR, unc, init=init, reference_node=ref))
        if ref >= 0:
            np.testing.assert_allclose(got["poses"][ref], init[ref], rtol=0, atol=1e-12)


# ---- refusals ---------------------------------------------------------------------------------------------------------------
BAD = [dict(max_correspondence_distance=0.0), dict(max_correspondence_distance=np.inf),
       dict(edge_prune_threshold=-0.1), dict(edge_prune_threshold=1.5), dict(preference_loop_closure=0.0),
       dict(preference_loop_closure=np.nan), dict(reference_node=-2), dict(reference_node=5), dict(max_iteration=0),
       dict(max_iteration_lm=0), dict(min_relative_increment=-1.0), dict(min_relative_residual_increment=np.inf),
       dict(min_right_term=np.nan), dict(min_residual=-1e-9), dict(lower_scale_factor=0.0),
       dict(upper_scale_factor=0.2), dict(upper_scale_factor=np.inf)]


@pytest.mark.parametrize("kw", BAD, ids=[next(iter(k)) + "=" + str(next(iter(k.values()))) for k in BAD])
def test_parameter_ranges(ctx, kw):
    gt, edges, T, L, unc = graph(81, 5, [])
    kw = dict(kw)
    c = kw.pop("max_correspondence_distance", R_CORR)
    with pytest.raises(capi.TzrError):
        ctx.global_optimization(5, edges, T, L, c, **kw)


def test_graph_refusals(ctx):
    gt, edges, T, L, unc = graph(83, 5, [])
    with pytest.raises(capi.TzrError):
        ctx.global_optimization(6, edges, T, L, R_CORR)  # node 5 has no edge
    with pytest.raises(capi.TzrError):
        ctx.global_optimization(1025, edges, T, L, R_CORR)
    bad = [t.copy() for t in T]
    bad[2][:3, :3] *= 1.001
    with pytest.raises(capi.TzrError):
        ctx.global_optimization(5, edges, bad, L, R_CORR)
    bad = [t.copy() for t in T]
    bad[1][0, 3] = np.nan
    with pytest.raises(capi.TzrError):
        ctx.global_optimization(5, edges, bad, L, R_CORR)
    badL = [x.copy() for x in L]
    badL[0][2, 2] = np.nan
    with pytest.raises(capi.TzrError):
        ctx.global_optimization(5, edges, T, badL, R_CORR)


# ---- launches and the retained solve ----------------------------------------------------------------------------------------
def enqueued(trials, cap):
    """Trials enqueued for a pass that ran `trials`: chunks of 1, 2, 4, then 8 until one ends at or past the last trial
    (include/teaser_b200.h), at most cap."""
    end, chunk = 0, 1
    while True:
        end += min(chunk, cap - end)
        chunk = min(2 * chunk, 8)
        if end >= max(1, trials) or end >= cap:
            return end


@pytest.mark.parametrize("ref", [0, -1])
def test_launch_count(ctx, ref):
    gt, edges, T, L, unc = graph(91, 9, [(8, 0), (5, 2)], wrong=[(7, 1)], noise=0.01)
    for kw in (dict(), dict(max_iteration=1, max_iteration_lm=3)):
        cap = kw.get("max_iteration", 100) * kw.get("max_iteration_lm", 20)
        l0 = ctx.kernel_launches()
        got = ctx.global_optimization(9, edges, T, L, R_CORR, uncertain=unc, reference_node=ref, **kw)
        want = sum(4 + 7 * enqueued(t, cap) for t in got["trials"]) + 1 + (ref >= 0)
        assert ctx.kernel_launches() - l0 == want


def test_retained_solve_survives(ctx):
    clouds = _sequence([600, 900, 700], seed=3)
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=0, rotation_cost_threshold=1e-12)
    res = ctx.register_cloud_pairs(clouds, [(0, 1), (1, 2)], prm, **PAIR_FLAGS)
    S = int((res[2] >= 0).sum())
    before = _retained(ctx, S)
    gt, edges, T, L, unc = graph(93, 8, [(7, 0)], noise=0.01)
    ctx.global_optimization(8, edges, T, L, R_CORR, uncertain=unc)
    assert _retained(ctx, S) == before


# ---- the chained entry ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("colored", [False, True])
def test_multiway_equals_the_chain_of_public_calls(ctx, colored):
    clouds = _sequence([600, 900, 700, 800, 650], seed=7)
    cols = [colours_of(c, seed=k) for k, c in enumerate(clouds)] if colored else None
    pairs = [(0, 1), (1, 2), (2, 3), (3, 4), (4, 0), (3, 1)]
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=0, rotation_cost_threshold=1e-12)
    kw = dict(colors=cols, lambda_geometric=0.9, kernel=("cauchy", 0.02)) if colored else {}
    plain = ctx.register_cloud_pairs(clouds, pairs, prm, **PAIR_FLAGS)
    S = int((plain[2] >= 0).sum())
    ret_plain = _retained(ctx, S)
    got = ctx.register_multiway(clouds, pairs, prm, R_CORR, optimizer="line_process", **kw, **PAIR_FLAGS)
    assert _retained(ctx, S) == ret_plain
    if colored:
        chain = ctx.register_cloud_pairs_icp(clouds, pairs, prm, R_CORR, method="colored", **kw, **PAIR_FLAGS)
    else:
        chain = ctx.register_cloud_pairs_icp(clouds, pairs, prm, R_CORR, method="point_to_plane", **PAIR_FLAGS)
    for a, b in zip(got[:7], chain):
        if isinstance(a, np.ndarray):
            assert a.tobytes() == b.tobytes()
        else:
            assert all(np.array_equal(x, y) for x, y in zip(a, b))
    mw, icp = got[7], chain[6]
    refined = [p for p in range(len(pairs)) if icp[p]["transform"]["scale"] > 0]
    assert len(refined) > 0
    trs = [dict(scale=float(icp[p]["transform"]["scale"]), rotation=icp[p]["transform"]["rotation"],
                translation=icp[p]["transform"]["translation"]) for p in refined]
    L, n = ctx.information_matrix_batch([clouds[pairs[p][0]] for p in refined], [clouds[pairs[p][1]] for p in refined],
                                        trs, R_CORR)
    for j, p in enumerate(refined):
        assert mw["information"][p].tobytes() == L[j].tobytes() and mw["counts"][p] == n[j]
    unc = [0 if b == a + 1 else 1 for a, b in pairs]
    want = ctx.global_optimization(len(clouds), [pairs[p] for p in refined], trs, L, R_CORR,
                                   uncertain=[unc[p] for p in refined])
    assert mw["status"] == 0
    assert mw["poses"].tobytes() == want["poses"].tobytes()
    assert mw["confidence"][refined].tobytes() == want["confidence"].tobytes()
    assert np.array_equal(mw["kept"][refined], want["kept"])
    for k in ("iterations", "trials", "stop_reason", "mu", "pruned", "residual"):
        assert mw[k] == want[k], k


def test_multiway_refusals(ctx):
    clouds = _sequence([600, 900], seed=8)
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=0)
    with pytest.raises(capi.TzrError):  # a robust kernel without colours
        ctx.register_multiway(clouds, [(0, 1)], prm, R_CORR, optimizer="line_process", kernel=("cauchy", 0.02),
                              **PAIR_FLAGS)
    with pytest.raises(capi.TzrError):
        ctx.register_multiway(clouds, [(0, 1)], prm, R_CORR, optimizer="line_process",
                              line_process=capi.line_process_params(R_CORR, max_iteration=0), **PAIR_FLAGS)
    with pytest.raises(capi.TzrError):
        ctx.register_multiway(clouds, [(0, 1)], prm, R_CORR, optimizer="levenberg", **PAIR_FLAGS)
    with pytest.raises(capi.TzrError):  # the other optimiser's parameters
        ctx.register_multiway(clouds, [(0, 1)], prm, R_CORR, optimizer="line_process",
                              pose_graph=capi.pose_graph_params(R_CORR), **PAIR_FLAGS)
    with pytest.raises(capi.TzrError):
        ctx.register_multiway(clouds, [(0, 1)], prm, R_CORR, line_process=capi.line_process_params(R_CORR),
                              **PAIR_FLAGS)


# ---- façades ----------------------------------------------------------------------------------------------------------
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "teaser-plusplus_b200", "host")
CSRC = os.path.join(ROOT, "teaser-plusplus_b200", "csrc")


def test_cpp_facade_equals_the_c_abi(tmp_path):
    """GlobalOptimization::optimize and the line-process solveMultiway against the C-ABI (tests/cpp/line_process_test.cc)."""
    subprocess.check_call(["make", "-s", "-C", HOST])
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    exe = str(tmp_path / "line_process_test")
    subprocess.check_call([cxx, "-std=c++17", "-O1", "-I", os.path.join(HOST, "include"), "-I",
                           os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "line_process_test.cc"),
                           "-L", HOST, "-lteaser_registration", "-L", CSRC, "-lteaser_b200",
                           f"-Wl,-rpath,{HOST}:{CSRC}", "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr


def test_pybind_equals_ctypes(ctx):
    subprocess.check_call(["make", "-s", "-C", HOST])
    sys.path.insert(0, os.path.join(HOST, "python"))
    import teaserpp_python as tpp
    gt, edges, T, L, unc = graph(21, 16, [(15, 0), (8, 0), (12, 4)], wrong=[(10, 2), (14, 6)], noise=0.004)
    g = tpp.GlobalOptimization(R_CORR, reference_node=-1).optimize(16, [tuple(e) for e in edges.tolist()], T, L,
                                                                     [bool(u) for u in unc])
    c = ctx.global_optimization(16, edges, T, L, R_CORR, uncertain=unc, reference_node=-1)
    assert np.stack(g["poses"]).tobytes() == c["poses"].tobytes()
    assert np.asarray(g["confidence"]).tobytes() == c["confidence"].tobytes()
    assert np.array_equal(np.asarray(g["kept"]), c["kept"])
    assert np.asarray(g["residuals"]).tobytes() == c["residuals"].tobytes()
    for k in ("iterations", "trials", "stop_reason", "mu", "pruned", "residual"):
        assert g[k] == c[k], k
    clouds = _sequence([600, 900, 700, 800], seed=7)
    pairs = [(0, 1), (1, 2), (2, 3), (3, 0)]
    solver = tpp.RobustRegistrationSolver(noise_bound=0.01, estimate_scaling=False, rotation_cost_threshold=1e-12)
    res = solver.solve_multiway(clouds, pairs, R_CORR, normal_search_radius=PAIR_FLAGS["normal_search_radius"],
                                fpfh_search_radius=PAIR_FLAGS["fpfh_search_radius"],
                                use_absolute_scale=PAIR_FLAGS["use_absolute_scale"],
                                use_crosscheck=PAIR_FLAGS["use_crosscheck"], use_tuple_test=PAIR_FLAGS["use_tuple_test"],
                                global_optimization=tpp.GlobalOptimization(R_CORR))
    assert res["pose_graph_status"] == 0
    mw = ctx.register_multiway(clouds, pairs, capi.default_params(noise_bound=0.01, estimate_scaling=0,
                                                                  rotation_cost_threshold=1e-12), R_CORR,
                               tuple_seeds=[0x7ea5e2 + 0x9E3779B97F4A7C15 * p & (2 ** 64 - 1) for p in range(4)],
                               optimizer="line_process", **PAIR_FLAGS)[7]
    assert np.stack(res["poses"]).tobytes() == mw["poses"].tobytes()
    assert np.asarray(res["edge_weights"]).tobytes() == mw["confidence"].tobytes()
    assert np.array_equal(np.asarray(res["edge_inliers"]), mw["kept"])
    for k in ("iterations", "trials", "stop_reason", "mu", "pruned", "residual"):
        assert res["line_process"][k] == mw[k], k
    with pytest.raises(ValueError):  # the GNC-TLS arguments do not apply
        solver.solve_multiway(clouds, pairs, R_CORR, gnc_factor=2.0, global_optimization=tpp.GlobalOptimization(R_CORR))
