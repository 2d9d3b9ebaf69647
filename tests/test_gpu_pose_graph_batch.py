"""The batched GNC-TLS pose graph on the device (run on an H100: `pytest -m gpu`): tzr_pose_graph_optimize_batch against
the numpy restatement (tests/pose_graph_reference.py) and against the single entry; each graph's independence from the
batch around it; per-graph and call-level refusals; the launch count; the all-certain, weight-0 and failed-factorisation
cases; 256 fragment graphs in one call; the retained solve; the C++ and pybind façades against the C ABI."""
import importlib
import os
import subprocess
import sys

import numpy as np
import pytest

import pose_graph_reference as ref
from line_process_fragments import fragment
from line_process_graphs import graph as lp_graph
from test_gpu_icp import PAIR_FLAGS, _retained, _sequence
from test_gpu_pose_graph import CASES, R_CORR, graph, rigid
from test_gpu_pose_graph_boundary import check_margins, compare, indefinite_graph
from test_pose_graph_batch_cpu import call

capi = importlib.import_module("teaser-plusplus_b200.capi")

pytestmark = pytest.mark.gpu

DECISIONS = ("iterations", "inner_iterations")


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


def gd(g, init=None, with_unc=True):
    gt, edges, T, L, unc = g
    return dict(K=len(gt), edges=edges, transforms=T, information=L, uncertain=unc if with_unc else None,
                initial_poses=init)


def restate(d, **kw):
    if "reference_node" in kw:
        kw["ref"] = kw.pop("reference_node")
    return ref.optimize(d["K"], d["edges"], d["transforms"], d["information"], R_CORR, d["uncertain"],
                        init=d["initial_poses"], **kw)


def single(ctx, d, **kw):
    return ctx.optimize_pose_graph(d["K"], d["edges"], d["transforms"], d["information"], R_CORR,
                                   uncertain=d["uncertain"], initial_poses=d["initial_poses"], **kw)


def check(got, want):
    """test_pose_graph_against_reference's checks"""
    assert (got["iterations"], got["inner_iterations"]) == (want["iterations"], want["inner_iterations"])
    assert np.array_equal(got["mask"], want["mask"])
    np.testing.assert_allclose(got["poses"], want["poses"], rtol=0, atol=1e-8)
    np.testing.assert_allclose(got["weights"], want["weights"], rtol=0, atol=1e-8)
    np.testing.assert_allclose(got["residuals"], want["residuals"], rtol=1e-6, atol=1e-12)
    assert abs(got["cost"] - want["cost"]) <= 1e-8 * max(1.0, want["cost"])


def same_bytes(a, b):
    for k in ("poses", "weights", "mask", "residuals", "iterations", "inner_iterations", "cost", "status"):
        if k in a and k in b:
            assert np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes(), k


def the_batch():
    """(graphs, n_wrong per graph): every CASES graph, a chain of 100, a complete graph of 32, fragments of 100 with
    wrong closures."""
    out = []
    for name in sorted(CASES):
        seed, K, extra = CASES[name]
        out.append((gd(graph(seed, K, extra or [], complete=extra is None)), 0))
    out.append((gd(lp_graph(101, 100, [], noise=0.003)), 0))
    out.append((gd(lp_graph(103, 32, None, noise=0.003, complete=True, points=(60, 120))), 0))
    for i in range(2):
        out.append((gd(fragment(105 + i, 100, n_wrong=2)), 2))
    return out


@pytest.fixture(scope="module")
def batch(ctx):
    graphs = the_batch()
    big = gd(lp_graph(41, 200, [(199, 0), (150, 20), (100, 60)], wrong=[(120, 10)], noise=0.003))
    ds = [g for g, _ in graphs] + [big]
    return graphs, big, ctx.optimize_pose_graph_batch(ds, R_CORR)


def test_against_the_restatement(batch):
    graphs, _, got = batch
    for (d, n_wrong), r in zip(graphs, got):
        assert r["status"] == 0
        check(r, restate(d))
        if n_wrong:
            assert not r["mask"][-n_wrong:].any()


def test_against_the_single_entry(ctx, batch):
    graphs, big, got = batch
    for (d, _), r in zip(graphs, got):
        s = single(ctx, d)
        for k in DECISIONS:
            assert r[k] == s[k], k
        assert np.array_equal(r["mask"], s["mask"])
    r = dict(got[-1])
    assert r.pop("status") == 0
    same_bytes(r, single(ctx, big))


def mixed():
    rng = np.random.default_rng(9)
    g1 = graph(73, 9, [(8, 0)], noise=0.01)
    init = [rigid(rng, 0.02, 0.02) @ g for g in g1[0]]
    return [gd(g1, init=init), gd(fragment(5, 60, n_wrong=1)), gd(graph(12, 12, [(11, 0), (8, 0)], noise=0.004),
                                                                  with_unc=False),
            gd(fragment(6, 128, n_wrong=2)), gd(graph(21, 16, [(15, 0), (8, 0)], wrong=[(10, 2)], noise=0.004)),
            gd(lp_graph(103, 32, None, noise=0.003, complete=True, points=(60, 120)))]


@pytest.mark.parametrize("ref_node", [0, 3])
def test_independent_of_the_batch_and_deterministic(ctx, ref_node):
    ds = mixed()
    a = ctx.optimize_pose_graph_batch(ds, R_CORR, reference_node=ref_node)
    b = ctx.optimize_pose_graph_batch(ds, R_CORR, reference_node=ref_node)
    rev = ctx.optimize_pose_graph_batch(ds[::-1], R_CORR, reference_node=ref_node)[::-1]
    for j, d in enumerate(ds):
        one = ctx.optimize_pose_graph_batch([d], R_CORR, reference_node=ref_node)[0]
        same_bytes(a[j], b[j])
        same_bytes(a[j], rev[j])
        same_bytes(a[j], one)
        check(a[j], restate(d, reference_node=ref_node))


def single_rc(ctx, d, **kw):
    try:
        single(ctx, d, **kw)
        return capi.TZR_OK
    except capi.TzrError as e:
        for code in (capi.TZR_ERR_INVALID_ARG, capi.TZR_ERR_TOO_LARGE):
            if str(e).startswith(capi.lib().tzr_status_string(code).decode() + ":"):
                return code
        raise


def test_per_graph_status(ctx):
    """Each refusal through its own check: the disconnected and non-rigid graphs contain the reference node, so they
    reach pg_start; the status is the single entry's code, with zeroed outputs, and the other graphs are unaffected."""
    good = [gd(graph(83, 12, [(11, 0)], noise=0.004)), gd(fragment(7, 30, n_wrong=1)), gd(graph(84, 9, [(8, 0)]))]
    g10 = graph(85, 10, [])
    disc = dict(gd(g10), K=11)  # node 10 has no edge
    bad_T = [t.copy() for t in g10[2]]
    bad_T[2][:3, :3] *= 1.001
    nonrigid = dict(gd(g10), transforms=bad_T)
    huge = dict(gd(g10), K=1025)
    small = gd(graph(86, 6, [(5, 0)]))  # reference_node 8 is not one of its nodes
    ds = [good[0], disc, good[1], nonrigid, huge, small, good[2]]
    messages = {"disc": "do not connect", "nonrigid": "not rigid", "huge": "more than 1024", "small": "reference_node"}
    for name, d in (("disc", disc), ("nonrigid", nonrigid), ("huge", huge), ("small", small)):
        with pytest.raises(capi.TzrError, match=messages[name]):
            single(ctx, d, reference_node=8)
        ctx.optimize_pose_graph_batch([d], R_CORR, reference_node=8)
        assert messages[name] in capi.lib().tzr_last_error(ctx._h).decode(), name
    got = ctx.optimize_pose_graph_batch(ds, R_CORR, reference_node=8)
    alone = [ctx.optimize_pose_graph_batch([d], R_CORR, reference_node=8)[0] for d in good]
    for d, r in zip(ds, got):
        assert r["status"] == single_rc(ctx, d, reference_node=8)
        if r["status"] != 0:
            assert not r["poses"][:, :3, :].any() and not r["weights"].any() and not r["mask"].any()
            assert not r["residuals"].any() and r["iterations"] == r["inner_iterations"] == 0 and r["cost"] == 0
    assert [r["status"] for r in got] == [0, capi.TZR_ERR_INVALID_ARG, 0, capi.TZR_ERR_INVALID_ARG,
                                          capi.TZR_ERR_TOO_LARGE, capi.TZR_ERR_INVALID_ARG, 0]
    for j, a, d in zip([0, 2, 6], alone, good):
        same_bytes(got[j], a)
        check(got[j], restate(d, reference_node=8))


@pytest.mark.parametrize("case", ["G0", "K", "E", "edges", "transforms", "information", "poses", "status",
                                  "distance", "gnc_factor", "max_iterations", "max_inner_iterations"])
def test_call_level_refusals(ctx, case):
    """With a context: G < 1, each NULL required array and each parameter the single entry refuses is
    TZR_ERR_INVALID_ARG from the batch's own check, with nothing written"""
    prm = capi.pose_graph_params(R_CORR)
    null, G = {}, 1
    if case == "G0":
        G = 0
    elif case == "distance":
        prm.max_correspondence_distance = 0.0
    elif case == "gnc_factor":
        prm.gnc_factor = 1.0
    elif case in ("max_iterations", "max_inner_iterations"):
        setattr(prm, case, 0)
    else:
        null = {case: True}
    rc, status, wrote_poses = call(ctx._h, prm, G, **null)
    assert rc == capi.TZR_ERR_INVALID_ARG and not wrote_poses
    if case != "status":
        assert status == 7
    assert capi.lib().tzr_last_error(ctx._h).decode().startswith("pose graph batch: invalid arguments")
    # the same graph with every argument given is solved
    assert call(ctx._h, capi.pose_graph_params(R_CORR))[:2] == (capi.TZR_OK, capi.TZR_OK)


def test_failed_factorisation_in_the_batch(ctx):
    """The first damped H of this graph is indefinite by a clear margin, so the batched Cholesky fails (on the first
    inner iteration of the call, before any candidate exists), the step is rejected and the damping climbs until the
    factorisation succeeds: the restatement's decisions and the single entry's, in a batch beside another graph."""
    edges, T, L = indefinite_graph()
    tr = []
    want = ref.optimize(3, edges, T, L, R_CORR, None, trace=tr, max_inner_iterations=12)
    inner = [x for x in tr if x["kind"] == "inner"]
    assert not inner[0]["factored"] and sum(not x["factored"] for x in inner) >= 3
    check_margins(tr)
    d = dict(K=3, edges=edges, transforms=T, information=L, uncertain=None, initial_poses=None)
    for ds in ([d], [gd(fragment(9, 40, n_wrong=1)), d]):
        got = ctx.optimize_pose_graph_batch(ds, R_CORR, max_inner_iterations=12)[-1]
        assert got["status"] == 0
        compare(got, want)
        s = single(ctx, d, max_inner_iterations=12)
        assert (got["iterations"], got["inner_iterations"]) == (s["iterations"], s["inner_iterations"])


def test_launch_count(ctx):
    for kw in (dict(), dict(max_iterations=1, max_inner_iterations=1)):
        counts = []
        for B in (1, 64):
            ds = [gd(fragment(200 + b, 40 + (b % 5) * 20, n_wrong=b % 3)) for b in range(B)]
            l0 = ctx.kernel_launches()
            got = ctx.optimize_pose_graph_batch(ds, R_CORR, **kw)
            counts.append(ctx.kernel_launches() - l0)
            assert all(r["status"] == 0 for r in got)
        assert counts == [1, 1]


def test_all_certain_runs_no_gnc_step(ctx):
    d = gd(graph(31, 8, [(7, 0)]), with_unc=False)
    got = ctx.optimize_pose_graph_batch([d, gd(fragment(9, 30, n_wrong=1))], R_CORR)[0]
    assert got["iterations"] == 1 and (got["weights"] == 1).all() and got["mask"].all()
    check(got, restate(d))


def test_singular_node_block_does_not_stop_the_graph(ctx):
    rng = np.random.default_rng(8)
    gt, edges, T, L, unc = graph(71, 7, [(6, 0)])
    Lsing = np.zeros((6, 6))
    Lsing[5, 5] = 100.0
    edges2 = np.vstack([edges, [[7, 3]]]).astype(np.int32)
    T2, L2, unc2 = T + [ref.inv(gt[3]) @ rigid(rng)], L + [Lsing], unc + [1]
    d2 = dict(K=8, edges=edges2, transforms=T2, information=L2, uncertain=unc2, initial_poses=None)
    got, base = ctx.optimize_pose_graph_batch([d2, gd((gt, edges, T, L, unc))], R_CORR)
    want = restate(d2)
    assert (got["iterations"], got["inner_iterations"]) == (want["iterations"], want["inner_iterations"])
    np.testing.assert_allclose(got["poses"], want["poses"], rtol=0, atol=1e-8)
    np.testing.assert_allclose(got["poses"][:7], base["poses"], rtol=0, atol=1e-8)


def test_256_fragments_in_one_call(ctx):
    ds = [gd(fragment(300 + b, 128, n_wrong=2)) for b in range(256)]
    got = ctx.optimize_pose_graph_batch(ds, R_CORR)
    assert all(r["status"] == 0 for r in got)
    for b in range(0, 256, 32):
        check(got[b], restate(ds[b]))
        assert not got[b]["mask"][-2:].any()


def test_retained_solve_survives(ctx):
    clouds = _sequence([600, 900, 700], seed=3)
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=0, rotation_cost_threshold=1e-12)
    res = ctx.register_cloud_pairs(clouds, [(0, 1), (1, 2)], prm, **PAIR_FLAGS)
    S = int((res[2] >= 0).sum())
    before = _retained(ctx, S)
    ctx.optimize_pose_graph_batch([gd(graph(93, 8, [(7, 0)], noise=0.01)), gd(fragment(8, 50, n_wrong=1))], R_CORR)
    assert _retained(ctx, S) == before


# ---- façades ----------------------------------------------------------------------------------------------------------
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "teaser-plusplus_b200", "host")
CSRC = os.path.join(ROOT, "teaser-plusplus_b200", "csrc")


def test_cpp_facade_equals_the_c_abi(tmp_path):
    """PoseGraph::optimizeBatch against the C ABI (tests/cpp/pose_graph_batch_test.cc)."""
    subprocess.check_call(["make", "-s", "-C", HOST])
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    exe = str(tmp_path / "pose_graph_batch_test")
    subprocess.check_call([cxx, "-std=c++17", "-O1", "-I", os.path.join(HOST, "include"), "-I",
                           os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "pose_graph_batch_test.cc"),
                           "-L", HOST, "-lteaser_registration", "-L", CSRC, "-lteaser_b200",
                           f"-Wl,-rpath,{HOST}:{CSRC}", "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr


def test_pybind_equals_ctypes(ctx):
    subprocess.check_call(["make", "-s", "-C", HOST])
    sys.path.insert(0, os.path.join(HOST, "python"))
    import teaserpp_python as tpp
    ds = [gd(fragment(31, 40, n_wrong=1)), gd(graph(21, 16, [(15, 0), (8, 0)], wrong=[(10, 2)], noise=0.004))]
    rng = np.random.default_rng(4)
    ds.append(gd(graph(73, 9, [(8, 0)], noise=0.01), init=[rigid(rng, 0.02, 0.02) @ np.eye(4) for _ in range(9)]))
    ds.append(dict(gd(graph(85, 5, [])), K=6))  # refused: node 5 has no edge
    graphs = [dict(num_nodes=d["K"], edges=[tuple(e) for e in d["edges"].tolist()], transforms=d["transforms"],
                   information=d["information"], uncertain=[bool(u) for u in d["uncertain"]],
                   initial_poses=d["initial_poses"] if d["initial_poses"] is not None else [])
              for d in ds]
    g = tpp.PoseGraph(R_CORR, reference_node=2).optimize_batch(graphs)
    c = ctx.optimize_pose_graph_batch(ds, R_CORR, reference_node=2)
    assert [a["status"] for a in g] == [b["status"] for b in c] == [0, 0, 0, capi.TZR_ERR_INVALID_ARG]
    assert g[3]["poses"] == []
    for a, b in zip(g[:3], c[:3]):
        assert np.stack(a["poses"]).tobytes() == b["poses"].tobytes()
        assert np.asarray(a["weights"]).tobytes() == b["weights"].tobytes()
        assert np.array_equal(np.asarray(a["inliers"]), b["mask"])
        assert np.asarray(a["residuals"]).tobytes() == b["residuals"].tobytes()
        for k in ("iterations", "inner_iterations", "cost"):
            assert a[k] == b[k], k
