"""The batched line process on the device (run on an H100: `pytest -m gpu`):
tzr_pose_graph_optimize_line_process_batch against the numpy restatement (tests/line_process_reference.py) and against
the single entry; each graph's independence from the batch around it; per-graph refusals; the launch count; 256
fragment graphs in one call; the retained solve; the C++ and pybind façades against the C ABI."""
import importlib
import os
import subprocess
import sys

import numpy as np
import pytest

import line_process_reference as lp
from line_process_fragments import fragment
from line_process_graphs import graph, rigid
from test_gpu_icp import PAIR_FLAGS, _retained, _sequence
from test_gpu_line_process import CASES, R_CORR, RULES, check

capi = importlib.import_module("teaser-plusplus_b200.capi")

pytestmark = pytest.mark.gpu

DECISIONS = ("iterations", "trials", "stop_reason", "pruned")


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
    return lp.optimize(d["K"], d["edges"], d["transforms"], d["information"], R_CORR, d["uncertain"],
                       init=d["initial_poses"], **kw)


def single(ctx, d, **kw):
    return ctx.global_optimization(d["K"], d["edges"], d["transforms"], d["information"], R_CORR,
                                   uncertain=d["uncertain"], initial_poses=d["initial_poses"], **kw)


def same_bytes(a, b):
    for k in ("poses", "confidence", "kept", "residuals", "iterations", "trials", "stop_reason", "mu", "pruned",
              "residual", "status"):
        if k in a and k in b:
            assert np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes(), k


def the_batch():
    """(graphs, n_wrong per graph): every CASES graph, a chain of 100, a complete graph of 32, fragments of 100 with
    wrong closures."""
    out = []
    for name in sorted(CASES):
        seed, K, extra, wrong = CASES[name]
        out.append((gd(graph(seed, K, extra or [], wrong=wrong, noise=0.004, complete=extra is None)), len(wrong)))
    out.append((gd(graph(101, 100, [], noise=0.003)), 0))
    out.append((gd(graph(103, 32, None, noise=0.003, complete=True, points=(60, 120))), 0))
    for i in range(2):
        out.append((gd(fragment(105 + i, 100, n_wrong=2)), 2))
    return out


@pytest.fixture(scope="module")
def batch(ctx):
    graphs = the_batch()
    big = gd(graph(41, 200, [(199, 0), (150, 20), (100, 60)], wrong=[(120, 10)], noise=0.003))
    ds = [g for g, _ in graphs] + [big]
    return graphs, big, ctx.global_optimization_batch(ds, R_CORR)


def test_against_the_restatement(batch):
    graphs, _, got = batch
    for (d, n_wrong), r in zip(graphs, got):
        assert r["status"] == 0
        check(r, restate(d))
        if n_wrong:
            assert not r["kept"][-n_wrong:].any() and r["pruned"] >= n_wrong


@pytest.mark.parametrize("rule", sorted(RULES))
def test_every_stop_rule(ctx, rule):
    d = gd(graph(61, 10, [(9, 0), (7, 2)], wrong=[(8, 1)], noise=0.01))
    want = restate(d, **RULES[rule])
    assert want["stop_reason"][0] == lp.STOP[rule]
    got = ctx.global_optimization_batch([d, gd(fragment(3, 40, n_wrong=1))], R_CORR, **RULES[rule])
    check(got[0], want)
    check(got[1], restate(gd(fragment(3, 40, n_wrong=1)), **RULES[rule]))


def test_against_the_single_entry(ctx, batch):
    graphs, big, got = batch
    for (d, _), r in zip(graphs, got):
        s = single(ctx, d)
        for k in DECISIONS:
            assert r[k] == s[k], k
        assert np.array_equal(r["kept"], s["kept"])
        assert np.asarray(r["mu"]).tobytes() == np.asarray(s["mu"]).tobytes()
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
            gd(graph(103, 32, None, noise=0.003, complete=True, points=(60, 120)))]


@pytest.mark.parametrize("ref", [0, -1])
def test_independent_of_the_batch_and_deterministic(ctx, ref):
    ds = mixed()
    a = ctx.global_optimization_batch(ds, R_CORR, reference_node=ref)
    b = ctx.global_optimization_batch(ds, R_CORR, reference_node=ref)
    rev = ctx.global_optimization_batch(ds[::-1], R_CORR, reference_node=ref)[::-1]
    for j, d in enumerate(ds):
        one = ctx.global_optimization_batch([d], R_CORR, reference_node=ref)[0]
        same_bytes(a[j], b[j])
        same_bytes(a[j], rev[j])
        same_bytes(a[j], one)
        check(a[j], restate(d, reference_node=ref))


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
    good = [gd(graph(83, 12, [(11, 0)], noise=0.004)), gd(fragment(7, 30, n_wrong=1)), gd(graph(84, 9, [(8, 0)]))]
    g5 = graph(85, 5, [])
    disc = dict(gd(g5), K=6)  # node 5 has no edge
    bad_T = [t.copy() for t in g5[2]]
    bad_T[2][:3, :3] *= 1.001
    nonrigid = dict(gd(g5), transforms=bad_T)
    huge = dict(gd(g5), K=1025)
    small = gd(graph(86, 6, [(5, 0)]))  # reference_node 8 is not one of its nodes
    ds = [good[0], disc, good[1], nonrigid, huge, small, good[2]]
    got = ctx.global_optimization_batch(ds, R_CORR, reference_node=8)
    alone = [ctx.global_optimization_batch([d], R_CORR, reference_node=8)[0] for d in good]
    for d, r in zip(ds, got):
        assert r["status"] == single_rc(ctx, d, reference_node=8)
        if r["status"] != 0:
            assert not r["poses"][:, :3, :].any() and not r["confidence"].any() and not r["kept"].any()
            assert not r["residuals"].any() and r["iterations"] == [0, 0] and r["mu"] == [0.0, 0.0]
    assert [r["status"] for r in got] == [0, capi.TZR_ERR_INVALID_ARG, 0, capi.TZR_ERR_INVALID_ARG,
                                          capi.TZR_ERR_TOO_LARGE, capi.TZR_ERR_INVALID_ARG, 0]
    for r, a in zip([got[0], got[2], got[6]], alone):
        same_bytes(r, a)
    # call-level refusals: raise, write nothing
    with pytest.raises(capi.TzrError):
        ctx.global_optimization_batch([], R_CORR)
    with pytest.raises(capi.TzrError):
        ctx.global_optimization_batch(good, R_CORR, max_iteration=0)
    with pytest.raises(capi.TzrError):
        ctx.global_optimization_batch(good, 0.0)


def test_launch_count(ctx):
    for kw in (dict(), dict(max_iteration=1, max_iteration_lm=3)):
        counts = []
        for B in (1, 64):
            ds = [gd(fragment(200 + b, 40 + (b % 5) * 20, n_wrong=b % 3)) for b in range(B)]
            l0 = ctx.kernel_launches()
            got = ctx.global_optimization_batch(ds, R_CORR, **kw)
            counts.append(ctx.kernel_launches() - l0)
            assert all(r["status"] == 0 for r in got)
        assert counts == [2, 2]


def test_256_fragments_in_one_call(ctx):
    ds = [gd(fragment(300 + b, 128, n_wrong=2)) for b in range(256)]
    got = ctx.global_optimization_batch(ds, R_CORR)
    assert all(r["status"] == 0 for r in got)
    for b in range(0, 256, 16):
        check(got[b], restate(ds[b]))
        assert not got[b]["kept"][-2:].any()


def test_retained_solve_survives(ctx):
    clouds = _sequence([600, 900, 700], seed=3)
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=0, rotation_cost_threshold=1e-12)
    res = ctx.register_cloud_pairs(clouds, [(0, 1), (1, 2)], prm, **PAIR_FLAGS)
    S = int((res[2] >= 0).sum())
    before = _retained(ctx, S)
    ctx.global_optimization_batch([gd(graph(93, 8, [(7, 0)], noise=0.01)), gd(fragment(8, 50, n_wrong=1))], R_CORR)
    assert _retained(ctx, S) == before


# ---- façades ----------------------------------------------------------------------------------------------------------
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "teaser-plusplus_b200", "host")
CSRC = os.path.join(ROOT, "teaser-plusplus_b200", "csrc")


def test_cpp_facade_equals_the_c_abi(tmp_path):
    """GlobalOptimization::optimizeBatch against the C ABI (tests/cpp/line_process_batch_test.cc)."""
    subprocess.check_call(["make", "-s", "-C", HOST])
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    exe = str(tmp_path / "line_process_batch_test")
    subprocess.check_call([cxx, "-std=c++17", "-O1", "-I", os.path.join(HOST, "include"), "-I",
                           os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "line_process_batch_test.cc"),
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
    graphs = [dict(num_nodes=d["K"], edges=[tuple(e) for e in d["edges"].tolist()], transforms=d["transforms"],
                   information=d["information"], uncertain=[bool(u) for u in d["uncertain"]],
                   initial_poses=d["initial_poses"] if d["initial_poses"] is not None else [])
              for d in ds]
    g = tpp.GlobalOptimization(R_CORR, reference_node=-1).optimize_batch(graphs)
    c = ctx.global_optimization_batch(ds, R_CORR, reference_node=-1)
    for a, b in zip(g, c):
        assert a["status"] == b["status"] == 0
        assert np.stack(a["poses"]).tobytes() == b["poses"].tobytes()
        assert np.asarray(a["confidence"]).tobytes() == b["confidence"].tobytes()
        assert np.array_equal(np.asarray(a["kept"]), b["kept"])
        assert np.asarray(a["residuals"]).tobytes() == b["residuals"].tobytes()
        for k in ("iterations", "trials", "stop_reason", "mu", "pruned", "residual"):
            assert a[k] == b[k], k
