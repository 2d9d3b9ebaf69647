"""Coloured ICP inside the chained cloud-pair and multiway calls (run on an H100: `pytest -m gpu`).

The chained entry against the chain of public calls it stands for (register_cloud_pairs, estimate_normals_batch,
icp_colored_batch) bit for bit, for several lambdas, with and without a kernel and with both scale settings; lambda = 1
against the point-to-plane and robust chained entries; lambda's range and the refusals, with nothing launched; the
gradient pass's launches; multiway against its chain of public calls and, at lambda = 1, against the point-to-plane
multiway call; the C++ and pybind façades against the C ABI.
"""
import ctypes as C
import importlib
import os
import subprocess
import sys

import numpy as np
import pytest

from test_gpu_icp import PAIR_FLAGS, RN, _retained, _sequence
from test_gpu_icp_colored import colours_of

capi = importlib.import_module("teaser-plusplus_b200.capi")

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "teaser-plusplus_b200", "host")
CSRC = os.path.join(ROOT, "teaser-plusplus_b200", "csrc")

R_CORR = 0.05
ITERS = 40


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.set_flags(0)
    c.close()


def _scene(sizes=(600, 1500, 500, 700), seed=5):
    """Clouds 0 ... 3 of a scan sequence, a far copy of cloud 0 (4) and a two-point cloud (5), with colours.  Cloud 1 is
    the target of two pairs, cloud 5 of none; the two-point cloud's pair is not solved."""
    clouds = _sequence(list(sizes), seed=seed)
    cols = [colours_of(c, seed=k) for k, c in enumerate(clouds)]
    clouds.append((clouds[0] + np.float32(40.0)).astype(np.float32))
    cols.append(cols[0].copy())
    clouds.append(clouds[2][:2].copy())
    cols.append(cols[2][:2].copy())
    pairs = [(0, 1), (1, 2), (2, 3), (3, 1), (1, 0), (0, 4), (5, 2)]
    return clouds, cols, pairs


def _seeds(sols, pairs_idx):
    return [dict(scale=sols[p]["scale"], rotation=sols[p]["rotation"], translation=sols[p]["translation"])
            for p in pairs_idx]


def _colored(ctx, clouds, cols, pairs, prm, lam=0.968, kernel=None):
    return ctx.register_cloud_pairs_icp(clouds, pairs, prm, R_CORR, max_iteration=ITERS, method="colored", colors=cols,
                                        lambda_geometric=lam, kernel=kernel, **PAIR_FLAGS)


def _gradient_launches(sizes):
    return 1 + (4 if max(sizes) >= 4096 else 0)


# ---- the chained entry ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("estimate_scaling", [0, 1])
@pytest.mark.parametrize("kernel", [None, ("huber", 0.02)], ids=["l2", "huber"])
@pytest.mark.parametrize("lam", [0.968, 0.0, 1.0])
def test_chained_entry_equals_the_chain(ctx, lam, kernel, estimate_scaling):
    clouds, cols, pairs = _scene()
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=estimate_scaling, rotation_cost_threshold=1e-12)
    plain = ctx.register_cloud_pairs(clouds, pairs, prm, **PAIR_FLAGS)
    S = int((plain[2] >= 0).sum())
    ret_plain = _retained(ctx, S)
    chained = _colored(ctx, clouds, cols, pairs, prm, lam, kernel)
    stage = capi.SOLUTION_DTYPE.fields["stage_ms"][1]
    for a, b in zip(plain[0], chained[0]):
        assert a.tobytes()[:stage] == b.tobytes()[:stage]
    assert np.array_equal(plain[1], chained[1]) and np.array_equal(plain[2], chained[2])
    assert all(np.array_equal(a, b) for a, b in zip(plain[3], chained[3]))
    assert all(np.array_equal(a, b) for a, b in zip(plain[4], chained[4]))
    assert plain[5] == chained[5]
    assert _retained(ctx, S) == ret_plain
    icp_res = chained[6]
    refined = [p for p in range(len(pairs)) if plain[1][p] == 0 and plain[0][p]["valid"]]
    assert len(refined) >= 3 and 6 not in refined
    for p in set(range(len(pairs))) - set(refined):
        assert not icp_res[p].tobytes().strip(b"\0"), p
    normals = ctx.estimate_normals_batch(clouds, RN)
    want, _ = ctx.icp_colored_batch([clouds[pairs[p][0]] for p in refined], [clouds[pairs[p][1]] for p in refined],
                                    [normals[pairs[p][1]] for p in refined], [cols[pairs[p][0]] for p in refined],
                                    [cols[pairs[p][1]] for p in refined], R_CORR, _seeds(plain[0], refined),
                                    lambda_geometric=lam, max_iteration=ITERS, kernel=kernel)
    for k, p in enumerate(refined):
        assert icp_res[p].tobytes() == want[k].tobytes(), p
        # the scans' colours follow each scan's own frame, so a purely photometric step (lambda 0) may walk a pair off
        assert icp_res[p]["iterations"] >= 1 and (lam == 0 or icp_res[p]["n_correspondences"] > 0)


@pytest.mark.parametrize("kernel", [None, ("tukey", 0.03)], ids=["l2", "tukey"])
def test_lambda_one_is_point_to_plane(ctx, kernel):
    clouds, cols, pairs = _scene(seed=6)
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=0, rotation_cost_threshold=1e-12)
    got = _colored(ctx, clouds, cols, pairs, prm, 1.0, kernel)
    plane = ctx.register_cloud_pairs_icp(clouds, pairs, prm, R_CORR, max_iteration=ITERS, method="point_to_plane",
                                         kernel=kernel, **PAIR_FLAGS)
    assert got[6].tobytes() == plane[6].tobytes()
    if kernel is None:  # and the robust entry with an explicit L2 kernel
        robust = ctx.register_cloud_pairs_icp(clouds, pairs, prm, R_CORR, max_iteration=ITERS,
                                              method="point_to_plane", kernel=("l2", 0.0), **PAIR_FLAGS)
        assert got[6].tobytes() == robust[6].tobytes()
    # the photometric rows move the result below lambda = 1
    other = _colored(ctx, clouds, cols, pairs, prm, 0.5, kernel)
    assert other[6].tobytes() != got[6].tobytes()


def test_lambda_out_of_range_and_refusals(ctx):
    clouds, cols, pairs = _scene(seed=7)
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=0, rotation_cost_threshold=1e-12)
    assert _colored(ctx, clouds, cols, pairs, prm, 2.0)[6].tobytes() == \
        _colored(ctx, clouds, cols, pairs, prm, 0.968)[6].tobytes()
    assert _colored(ctx, clouds, cols, pairs, prm, -0.5)[6].tobytes() == \
        _colored(ctx, clouds, cols, pairs, prm, 0.968)[6].tobytes()
    l0 = ctx.kernel_launches()
    with pytest.raises(capi.TzrError):
        _colored(ctx, clouds, cols, pairs, prm, float("nan"))
    with pytest.raises(capi.TzrError):
        _colored(ctx, clouds, cols, pairs, prm, float("inf"))
    with pytest.raises(capi.TzrError):
        _colored(ctx, clouds, cols, pairs, prm, 0.968, capi.RobustKernel(99, 0, 1.0))
    with pytest.raises(capi.TzrError):
        _colored(ctx, clouds, cols, pairs, prm, 0.968, ("huber", -1.0))
    # a NULL colour entry and a NULL colour array, through the C ABI directly
    L = capi.lib()
    fpp = C.POINTER(C.c_float)
    cl = [np.ascontiguousarray(c, dtype=np.float32) for c in clouds]
    K = [np.ascontiguousarray(c, dtype=np.float32) for c in cols]
    pc = np.ascontiguousarray(pairs, dtype=np.int32)
    P = len(pairs)
    n = np.array([len(c) for c in cl], dtype=np.int32)
    fpar = capi.FrontendParams(PAIR_FLAGS["normal_search_radius"], PAIR_FLAGS["fpfh_search_radius"], 0, 1, 0, 0.0)
    icp = capi.icp_params(R_CORR)
    sols = np.zeros(P, dtype=capi.SOLUTION_DTYPE)
    st, idx, cnt = np.zeros(P, np.int32), np.zeros(P, np.int32), np.zeros(P, np.int64)
    res = np.zeros(P, dtype=capi.ICP_RESULT_DTYPE)
    for colour_ptrs in ((fpp * len(K))(*([capi._p(k, C.c_float) for k in K[:-1]] + [None])), None):
        rc = L.tzr_register_cloud_pairs_icp_colored(
            ctx._h, C.byref(fpar), C.byref(prm), len(cl), capi._p(n, C.c_int32),
            (fpp * len(cl))(*[capi._p(c, C.c_float) for c in cl]), P, capi._p(pc, C.c_int32), None,
            sols.ctypes.data_as(C.POINTER(capi.Solution)), capi._p(st, C.c_int32), capi._p(idx, C.c_int32),
            capi._p(cnt, C.c_int64), None, None, None, C.byref(icp), colour_ptrs, 0.968, None,
            res.ctypes.data_as(C.POINTER(capi.IcpResult)))
        assert rc == capi.TZR_ERR_INVALID_ARG
    assert ctx.kernel_launches() == l0


@pytest.mark.parametrize("sizes", [(600, 1500, 500, 700), (600, 4200, 500, 700)], ids=["small", "grid"])
def test_launch_count(ctx, sizes):
    clouds, cols, pairs = _scene(sizes, seed=8)
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=0, rotation_cost_threshold=1e-12)
    l0 = ctx.kernel_launches()
    plane = ctx.register_cloud_pairs_icp(clouds, pairs, prm, R_CORR, max_iteration=ITERS, method="point_to_plane",
                                         **PAIR_FLAGS)
    l1 = ctx.kernel_launches()
    col = _colored(ctx, clouds, cols, pairs, prm)
    l2 = ctx.kernel_launches()
    assert np.array_equal(plane[2], col[2]) and (col[2] >= 0).any()
    assert (l2 - l1) - (l1 - l0) == _gradient_launches([len(c) for c in clouds])
    # the FPFH stage's route flag forces the gradient pass's grid at any size
    ctx.set_flags(capi.FLAG_FPFH_GRID)
    try:
        l3 = ctx.kernel_launches()
        ctx.register_cloud_pairs_icp(clouds, pairs, prm, R_CORR, max_iteration=ITERS, method="point_to_plane",
                                     **PAIR_FLAGS)
        l4 = ctx.kernel_launches()
        forced = _colored(ctx, clouds, cols, pairs, prm)
        l5 = ctx.kernel_launches()
    finally:
        ctx.set_flags(0)
    assert (l5 - l4) - (l4 - l3) == 5
    assert forced[6].tobytes() == col[6].tobytes()


# ---- multiway ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stray", [False, True])
def test_multiway_equals_the_chain_of_public_calls(ctx, stray):
    clouds = _sequence([600, 900, 700, 800, 650], seed=7)
    cols = [colours_of(c, seed=k) for k, c in enumerate(clouds)]
    pairs = [(0, 1), (1, 2), (2, 3), (3, 4), (4, 0), (3, 1)]
    if stray:  # a two-point cloud: its pair is not solved, so its node is not connected
        clouds.append(clouds[2][:2].copy())
        cols.append(cols[2][:2].copy())
        pairs.append((5, 2))
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=0, rotation_cost_threshold=1e-12)
    plain = ctx.register_cloud_pairs(clouds, pairs, prm, **PAIR_FLAGS)
    S = int((plain[2] >= 0).sum())
    ret_plain = _retained(ctx, S)
    kernel = ("cauchy", 0.02)
    got = ctx.register_multiway(clouds, pairs, prm, R_CORR, colors=cols, lambda_geometric=0.9, kernel=kernel,
                                **PAIR_FLAGS)
    assert _retained(ctx, S) == ret_plain
    chain = ctx.register_cloud_pairs_icp(clouds, pairs, prm, R_CORR, method="colored", colors=cols,
                                         lambda_geometric=0.9, kernel=kernel, **PAIR_FLAGS)
    for a, b in zip(got[:7], chain):
        if isinstance(a, np.ndarray):
            assert a.tobytes() == b.tobytes()
        else:
            assert all(np.array_equal(x, y) for x, y in zip(a, b))
    mw = got[7]
    icp = chain[6]
    refined = [p for p in range(len(pairs)) if icp[p]["transform"]["scale"] > 0]
    assert 0 < len(refined) <= len(pairs) - stray
    trs = [dict(scale=float(icp[p]["transform"]["scale"]), rotation=icp[p]["transform"]["rotation"],
                translation=icp[p]["transform"]["translation"]) for p in refined]
    L, n = ctx.information_matrix_batch([clouds[pairs[p][0]] for p in refined], [clouds[pairs[p][1]] for p in refined],
                                        trs, R_CORR)
    for j, p in enumerate(refined):
        assert mw["information"][p].tobytes() == L[j].tobytes() and mw["counts"][p] == n[j]
    for p in set(range(len(pairs))) - set(refined):
        assert not mw["information"][p].any() and mw["weights"][p] == 0
    unc = [0 if b == a + 1 else 1 for a, b in pairs]
    if stray:
        with pytest.raises(capi.TzrError):
            ctx.optimize_pose_graph(len(clouds), [pairs[p] for p in refined], trs, L, R_CORR,
                                    uncertain=[unc[p] for p in refined])
        assert mw["status"] == capi.TZR_ERR_INVALID_ARG and not mw["poses"][:, :3].any() and not mw["weights"].any()
        return
    pg = ctx.optimize_pose_graph(len(clouds), [pairs[p] for p in refined], trs, L, R_CORR,
                                 uncertain=[unc[p] for p in refined])
    assert mw["status"] == 0
    assert mw["poses"].tobytes() == pg["poses"].tobytes()
    assert mw["weights"][refined].tobytes() == pg["weights"].tobytes()
    assert np.array_equal(mw["mask"][refined], pg["mask"])
    assert (mw["iterations"], mw["inner_iterations"], mw["cost"]) == (pg["iterations"], pg["inner_iterations"],
                                                                      pg["cost"])


def _same_multiway(a, b):
    for x, y in zip(a[:7], b[:7]):
        if isinstance(x, np.ndarray):
            assert x.tobytes() == y.tobytes()
        else:
            assert all(np.array_equal(u, v) for u, v in zip(x, y))
    for k in ("information", "counts", "weights", "mask", "poses"):
        assert a[7][k].tobytes() == b[7][k].tobytes(), k
    assert [a[7][k] for k in ("status", "iterations", "inner_iterations", "cost")] == \
        [b[7][k] for k in ("status", "iterations", "inner_iterations", "cost")]


def test_multiway_lambda_one_is_point_to_plane_multiway(ctx):
    clouds = _sequence([600, 900, 700, 800, 650], seed=9)
    cols = [colours_of(c, seed=k) for k, c in enumerate(clouds)]
    pairs = [(0, 1), (1, 2), (2, 3), (3, 4), (4, 0), (3, 1)]
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=0, rotation_cost_threshold=1e-12)
    plane = ctx.register_multiway(clouds, pairs, prm, R_CORR, **PAIR_FLAGS)
    col = ctx.register_multiway(clouds, pairs, prm, R_CORR, colors=cols, lambda_geometric=1.0, **PAIR_FLAGS)
    assert plane[7]["status"] == 0
    _same_multiway(plane, col)


def test_multiway_rejects_estimated_scale(ctx):
    clouds = _sequence([600, 900], seed=8)
    cols = [colours_of(c) for c in clouds]
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=1)
    l0 = ctx.kernel_launches()
    with pytest.raises(capi.TzrError):
        ctx.register_multiway(clouds, [(0, 1)], prm, R_CORR, colors=cols, **PAIR_FLAGS)
    assert ctx.kernel_launches() == l0


# ---- façades ----------------------------------------------------------------------------------------------------------
def test_cpp_facade_equals_the_c_abi(tmp_path):
    """solveCloudPairsColoredICP and the coloured solveMultiway against the C-ABI (tests/cpp/register_colored_test.cc)."""
    subprocess.check_call(["make", "-s", "-C", HOST])
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    exe = str(tmp_path / "register_colored_test")
    subprocess.check_call([cxx, "-std=c++17", "-O1", "-I", os.path.join(HOST, "include"), "-I",
                           os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "register_colored_test.cc"),
                           "-L", HOST, "-lteaser_registration", "-L", CSRC, "-lteaser_b200",
                           f"-Wl,-rpath,{HOST}:{CSRC}", "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr


def test_pybind_equals_ctypes(ctx):
    subprocess.check_call(["make", "-s", "-C", HOST])
    sys.path.insert(0, os.path.join(HOST, "python"))
    import teaserpp_python as tpp
    clouds = _sequence([600, 900, 700, 800, 650], seed=10)
    cols = [colours_of(c, seed=k) for k, c in enumerate(clouds)]
    pairs = [(0, 1), (1, 2), (2, 3), (3, 4), (4, 0), (3, 1)]
    solver = tpp.RobustRegistrationSolver(noise_bound=0.01, estimate_scaling=False, rotation_cost_threshold=1e-12)
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=0, rotation_cost_threshold=1e-12)
    flags = dict(PAIR_FLAGS)  # no tuple test: the tuple seeds play no part
    tkernel = tpp.RobustKernel(tpp.RobustKernel.Type.HUBER, 0.02)
    for kernel, tk in ((None, None), (("huber", 0.02), tkernel)):
        got = solver.solve_cloud_pairs_icp(clouds, pairs, R_CORR, method="colored", colors=cols, lambda_geometric=0.9,
                                           kernel=tk, **flags)
        want = ctx.register_cloud_pairs_icp(clouds, pairs, prm, R_CORR, method="colored", colors=cols,
                                            lambda_geometric=0.9, kernel=kernel, **flags)[6]
        assert sum(r["refined"] for r in got) >= 5
        for r, w in zip(got, want):
            if not r["refined"]:
                assert w["transform"]["scale"] == 0
                continue
            d = capi.icp_result_dict(w)
            assert np.array_equal(np.asarray(r["icp"]["solution"].rotation), d["R"])
            assert np.array_equal(np.asarray(r["icp"]["solution"].translation).ravel(), d["t"])
            assert (r["icp"]["fitness"], r["icp"]["inlier_rmse"], r["icp"]["iterations"]) == \
                (d["fitness"], d["inlier_rmse"], d["iterations"])
    mw = solver.solve_multiway(clouds, pairs, R_CORR, colors=cols, lambda_geometric=0.9, kernel=tkernel, **flags)
    want = ctx.register_multiway(clouds, pairs, prm, R_CORR, colors=cols, lambda_geometric=0.9,
                                 kernel=("huber", 0.02), **flags)[7]
    assert mw["pose_graph_status"] == want["status"] == 0
    for k in range(len(clouds)):
        assert np.array_equal(np.asarray(mw["poses"][k]), want["poses"][k])
    for p in range(len(pairs)):
        assert np.array_equal(np.asarray(mw["information"][p]), want["information"][p])
    assert np.array_equal(np.asarray(mw["edge_weights"]), want["weights"])
    with pytest.raises(ValueError):
        solver.solve_cloud_pairs_icp(clouds, pairs, R_CORR, method="point_to_plane", colors=cols, **flags)
    with pytest.raises(ValueError):
        solver.solve_multiway(clouds, pairs, R_CORR, kernel=tkernel, **flags)
