"""Multiway registration on the device (run on an H100: `pytest -m gpu`): information matrices against the numpy
restatement (tests/pose_graph_reference.py) bit for bit, on both search routes, batch against single, edge inputs and the
retained solve; the GNC-TLS pose graph against the restatement on synthetic graphs, a wrong loop closure rejected, the
error cases, explicit initial poses and the launch count; the chained entry against the chain of public calls."""
import importlib
import os
import subprocess
import sys

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import pose_graph_reference as ref
from test_gpu_icp import PAIR_FLAGS, _retained, _sequence, scan_pair

capi = importlib.import_module("teaser-plusplus_b200.capi")

pytestmark = pytest.mark.gpu

BRUTE, GRID = capi.FLAG_ICP_BRUTE_FORCE, capi.FLAG_ICP_GRID
R_CORR = 0.05


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.set_flags(0)
    c.close()


def with_flags(ctx, flags, fn):
    ctx.set_flags(flags)
    try:
        return fn()
    finally:
        ctx.set_flags(0)


def sim(R, t, s=1.0):
    return dict(scale=s, rotation=np.asarray(R), translation=np.asarray(t))


# ---- information matrices ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed,ns,nd", [(1, 700, 900), (2, 3000, 2500), (3, 5000, 400)])
def test_information_against_reference(ctx, seed, ns, nd):
    src, dst, R, t = scan_pair(seed, ns, nd)
    want, wc = ref.information(src, dst, 1.0, R, t, R_CORR)
    got, gc = ctx.information_matrix(src, dst, sim(R, t), R_CORR)
    assert gc == wc > 100 and got[5, 5] == gc
    assert np.array_equal(got, want)
    assert np.array_equal(got, got.T)


def test_information_routes_bit_identical(ctx):
    src, dst, R, t = scan_pair(4, 2000, 3000)
    a = with_flags(ctx, BRUTE, lambda: ctx.information_matrix(src, dst, sim(R, t), R_CORR))
    b = with_flags(ctx, GRID, lambda: ctx.information_matrix(src, dst, sim(R, t), R_CORR))
    c = ctx.information_matrix(src, dst, sim(R, t), R_CORR)
    assert a[1] == b[1] == c[1] and a[0].tobytes() == b[0].tobytes() == c[0].tobytes()


def test_information_batch_equals_single(ctx):
    probs = [scan_pair(s, ns, nd) for s, ns, nd in [(5, 300, 2000), (6, 1200, 800), (7, 40, 60), (8, 2600, 1500)]]
    singles = [ctx.information_matrix(p[0], p[1], sim(p[2], p[3]), R_CORR) for p in probs]
    for order in ([0, 1, 2, 3], [3, 2, 1, 0]):
        L, n = ctx.information_matrix_batch([probs[k][0] for k in order], [probs[k][1] for k in order],
                                            [sim(probs[k][2], probs[k][3]) for k in order], R_CORR)
        for j, k in enumerate(order):
            assert L[j].tobytes() == singles[k][0].tobytes() and n[j] == singles[k][1]


def test_information_edges(ctx):
    rng = np.random.default_rng(9)
    dst = rng.uniform(-1, 1, size=(500, 3)).astype(np.float32)
    src = dst.copy()
    src[::7] = np.nan
    dst[::11] = np.nan
    want, wc = ref.information(src, dst, 1.0, np.eye(3), np.zeros(3), 0.05)
    got, gc = ctx.information_matrix(src, dst, None, 0.05)
    assert gc == wc and np.array_equal(got, want)
    # points at exactly r: no correspondence (strict d^2 < r^2)
    y = np.array([[0.0, 0.0, 0.0]], dtype=np.float32)
    x = np.array([[0.5, 0.0, 0.0], [0.25, 0.0, 0.0]], dtype=np.float32)
    L, n = ctx.information_matrix(x, y, None, 0.5)
    assert n == 1 and L[5, 5] == 1.0
    # no correspondence at all: Lambda = 0
    L, n = ctx.information_matrix(x + np.float32(10), y, None, 0.5)
    assert n == 0 and not L.any()
    with pytest.raises(capi.TzrError):
        ctx.information_matrix(x, y, None, 0.0)


def test_information_keeps_the_retained_solve(ctx):
    clouds = _sequence([600, 900, 700], seed=3)
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=0, rotation_cost_threshold=1e-12)
    res = ctx.register_cloud_pairs(clouds, [(0, 1), (1, 2)], prm, **PAIR_FLAGS)
    S = int((res[2] >= 0).sum())
    before = _retained(ctx, S)
    ctx.information_matrix(clouds[0], clouds[1], None, R_CORR)
    assert _retained(ctx, S) == before


# ---- pose graph ---------------------------------------------------------------------------------------------------------
def rigid(rng, angle=0.3, shift=0.5):
    T = np.eye(4)
    T[:3, :3] = Rotation.from_rotvec(rng.normal(size=3) * angle).as_matrix()
    T[:3, 3] = rng.normal(size=3) * shift
    return T


def graph(seed, K, extra, wrong=(), noise=0.002, complete=False):
    rng = np.random.default_rng(seed)
    gt = [np.eye(4)] + [rigid(rng) for _ in range(K - 1)]
    pairs = [(a, b) for a in range(K) for b in range(K) if a < b] if complete else \
        [(k, k + 1) for k in range(K - 1)] + list(extra)
    edges, T, L, unc = [], [], [], []
    for s, d in list(pairs) + list(wrong):
        Tsd = ref.inv(gt[d]) @ gt[s]
        Tsd = (rigid(rng, 0.5, 1.0) if (s, d) in wrong else rigid(rng, noise, noise)) @ Tsd
        pts = rng.uniform(-1, 1, size=(int(rng.integers(100, 400)), 3))
        G = [np.hstack([-ref.skew(q), np.eye(3)]) for q in pts]
        edges.append((s, d))
        T.append(Tsd)
        L.append(sum(g.T @ g for g in G))
        unc.append(0 if d == s + 1 else 1)
    return gt, np.array(edges, dtype=np.int32), T, L, unc


CASES = {
    "chain": (11, 6, []),
    "loops": (12, 12, [(11, 0), (8, 0), (9, 3), (7, 2)]),
    "complete6": (13, 6, None),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_pose_graph_against_reference(ctx, name):
    seed, K, extra = CASES[name]
    gt, edges, T, L, unc = graph(seed, K, extra or [], complete=extra is None)
    want = ref.optimize(K, edges, T, L, R_CORR, unc)
    got = ctx.optimize_pose_graph(K, edges, T, L, R_CORR, uncertain=unc)
    assert (got["iterations"], got["inner_iterations"]) == (want["iterations"], want["inner_iterations"])
    assert np.array_equal(got["mask"], want["mask"])
    np.testing.assert_allclose(got["poses"], want["poses"], rtol=0, atol=1e-8)
    np.testing.assert_allclose(got["weights"], want["weights"], rtol=0, atol=1e-8)
    np.testing.assert_allclose(got["residuals"], want["residuals"], rtol=1e-6, atol=1e-12)
    assert abs(got["cost"] - want["cost"]) <= 1e-8 * max(1.0, want["cost"])


def test_wrong_closure_rejected(ctx):
    K = 16
    gt, edges, T, L, unc = graph(21, K, [(15, 0), (8, 0), (12, 4)], wrong=[(10, 2), (14, 6)], noise=0.004)
    got = ctx.optimize_pose_graph(K, edges, T, L, R_CORR, uncertain=unc)
    want = ref.optimize(K, edges, T, L, R_CORR, unc)
    assert np.array_equal(got["mask"], want["mask"])
    assert not got["mask"][-2:].any() and got["mask"][:-2].all()
    odo = ref.bfs(K, edges, T, [d == s + 1 for s, d in edges], [0] * len(edges), 0)  # odometry composition alone
    err_odo = max(np.linalg.norm(p[:3, 3] - g[:3, 3]) for p, g in zip(odo, gt))
    err_opt = max(np.linalg.norm(p[:3, 3] - g[:3, 3]) for p, g in zip(got["poses"], gt))
    assert err_opt < err_odo


def test_all_certain_runs_no_gnc_step(ctx):
    gt, edges, T, L, unc = graph(31, 8, [(7, 0)])
    got = ctx.optimize_pose_graph(8, edges, T, L, R_CORR, uncertain=None)
    assert got["iterations"] == 1 and (got["weights"] == 1).all() and got["mask"].all()
    want = ref.optimize(8, edges, T, L, R_CORR, None)
    assert got["inner_iterations"] == want["inner_iterations"]


def test_explicit_initial_poses_equal_the_default(ctx):
    gt, edges, T, L, unc = graph(41, 10, [(9, 0), (6, 1)])
    base = ctx.optimize_pose_graph(10, edges, T, L, R_CORR, uncertain=unc)
    init = ref.bfs(10, edges, T, [True] * len(edges), unc, 0)
    again = ctx.optimize_pose_graph(10, edges, T, L, R_CORR, uncertain=unc, initial_poses=init)
    for k in base:
        assert np.array_equal(base[k], again[k]), k
    # another reference node: the same minimum up to a rigid motion, to within the inner solve's stopping rule (its
    # damping and stopping point are not gauge-invariant; 1.4e-7 was the largest difference seen)
    moved = ctx.optimize_pose_graph(10, edges, T, L, R_CORR, uncertain=unc, reference_node=3)
    G = moved["poses"][3] @ ref.inv(base["poses"][3])
    np.testing.assert_allclose(moved["poses"], np.stack([G @ p for p in base["poses"]]), atol=1e-6)


def test_pose_graph_errors(ctx):
    gt, edges, T, L, unc = graph(51, 5, [])
    with pytest.raises(capi.TzrError, match="INVALID|invalid"):
        ctx.optimize_pose_graph(6, edges, T, L, R_CORR)  # node 5 has no edge
    with pytest.raises(capi.TzrError):
        ctx.optimize_pose_graph(1025, edges, T, L, R_CORR)
    bad = [t.copy() for t in T]
    bad[2][:3, :3] *= 1.001
    with pytest.raises(capi.TzrError):
        ctx.optimize_pose_graph(5, edges, bad, L, R_CORR)
    bad = [t.copy() for t in T]
    bad[1][0, 3] = np.nan
    with pytest.raises(capi.TzrError):
        ctx.optimize_pose_graph(5, edges, bad, L, R_CORR)


def test_launch_count(ctx):
    gt, edges, T, L, unc = graph(61, 7, [(6, 0)])
    l0 = ctx.kernel_launches()
    got = ctx.optimize_pose_graph(7, edges, T, L, R_CORR, uncertain=unc, max_inner_iterations=6)
    assert ctx.kernel_launches() - l0 == got["iterations"] * (3 + 4 * 6)


# ---- the chained entry ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stray", [False, True])
def test_multiway_equals_the_chain_of_public_calls(ctx, stray):
    clouds = _sequence([600, 900, 700, 800, 650], seed=7)
    pairs = [(0, 1), (1, 2), (2, 3), (3, 4), (4, 0), (3, 1)]
    if stray:  # a two-point cloud: its pair is not solved, so its node is not connected
        clouds.append(clouds[2][:2].copy())
        pairs.append((5, 2))
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=0, rotation_cost_threshold=1e-12)
    plain = ctx.register_cloud_pairs(clouds, pairs, prm, **PAIR_FLAGS)
    S = int((plain[2] >= 0).sum())
    ret_plain = _retained(ctx, S)
    got = ctx.register_multiway(clouds, pairs, prm, R_CORR, **PAIR_FLAGS)
    assert _retained(ctx, S) == ret_plain
    chain = ctx.register_cloud_pairs_icp(clouds, pairs, prm, R_CORR, method="point_to_plane", **PAIR_FLAGS)
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


def test_multiway_rejects_estimated_scale(ctx):
    clouds = _sequence([600, 900], seed=8)
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=1)
    with pytest.raises(capi.TzrError):
        ctx.register_multiway(clouds, [(0, 1)], prm, R_CORR, **PAIR_FLAGS)


def test_singular_node_block_does_not_stop_the_graph(ctx):
    rng = np.random.default_rng(8)
    gt, edges, T, L, unc = graph(71, 7, [(6, 0)])
    Lsing = np.zeros((6, 6))
    Lsing[5, 5] = 100.0
    edges2 = np.vstack([edges, [[7, 3]]]).astype(np.int32)
    T2, L2, unc2 = T + [ref.inv(gt[3]) @ rigid(rng)], L + [Lsing], unc + [1]
    got = ctx.optimize_pose_graph(8, edges2, T2, L2, R_CORR, uncertain=unc2)
    want = ref.optimize(8, edges2, T2, L2, R_CORR, unc2)
    base = ctx.optimize_pose_graph(7, edges, T, L, R_CORR, uncertain=unc)
    assert (got["iterations"], got["inner_iterations"]) == (want["iterations"], want["inner_iterations"])
    np.testing.assert_allclose(got["poses"], want["poses"], rtol=0, atol=1e-8)
    np.testing.assert_allclose(got["poses"][:7], base["poses"], rtol=0, atol=1e-8)


def test_argument_checks_with_a_context(ctx):
    gt, edges, T, L, unc = graph(81, 4, [])
    for kw, match in [(dict(reference_node=9), "reference_node"), (dict(gnc_factor=1.0), "invalid")]:
        with pytest.raises(capi.TzrError, match=match):
            ctx.optimize_pose_graph(4, edges, T, L, R_CORR, **kw)
    bad = [x.copy() for x in L]
    bad[0][5, 5] = -1.0
    with pytest.raises(capi.TzrError, match="Lambda"):
        ctx.optimize_pose_graph(4, edges, T, bad, R_CORR)
    bad[0][5, 5] = np.inf
    with pytest.raises(capi.TzrError, match="non-finite"):
        ctx.optimize_pose_graph(4, edges, T, bad, R_CORR)
    init = [np.eye(4)] * 4
    init[2] = 2 * np.eye(4)
    with pytest.raises(capi.TzrError, match="initial pose"):
        ctx.optimize_pose_graph(4, edges, T, L, R_CORR, initial_poses=init)
    clouds = _sequence([600, 900], seed=8)
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=0)
    with pytest.raises(capi.TzrError):  # one uncertain flag per pair
        ctx.register_multiway(clouds, [(0, 1)], prm, R_CORR, uncertain=[0, 1], **PAIR_FLAGS)
    with pytest.raises(capi.TzrError):  # pose-graph parameters out of range
        ctx.register_multiway(clouds, [(0, 1)], prm, R_CORR, pose_graph=capi.pose_graph_params(R_CORR, max_iterations=0),
                              **PAIR_FLAGS)


# ---- façades ----------------------------------------------------------------------------------------------------------
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "teaser-plusplus_b200", "host")
CSRC = os.path.join(ROOT, "teaser-plusplus_b200", "csrc")


def test_cpp_facade_equals_the_c_abi(tmp_path):
    """informationMatrix(Batch), PoseGraph::optimize and solveMultiway against the C-ABI (tests/cpp/pose_graph_test.cc)."""
    subprocess.check_call(["make", "-s", "-C", HOST])
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    exe = str(tmp_path / "pose_graph_test")
    subprocess.check_call([cxx, "-std=c++17", "-O1", "-I", os.path.join(HOST, "include"), "-I",
                           os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "pose_graph_test.cc"),
                           "-L", HOST, "-lteaser_registration", "-L", CSRC, "-lteaser_b200",
                           f"-Wl,-rpath,{HOST}:{CSRC}", "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr


def test_pybind_multiway(ctx):
    subprocess.check_call(["make", "-s", "-C", HOST])
    sys.path.insert(0, os.path.join(HOST, "python"))
    import teaserpp_python as tpp
    src, dst, R, t = scan_pair(3, 900, 1000)
    T = tpp.RegistrationSolution()
    T.scale = 1.0
    T.rotation = np.asarray(R, dtype=np.float64)
    T.translation = np.asarray(t, dtype=np.float64)
    L, n = tpp.information_matrix(src, dst, T, R_CORR)
    want, wn = ctx.information_matrix(src, dst, sim(R, t), R_CORR)
    assert n == wn and np.array_equal(L, want)
    LB, nb = tpp.information_matrix_batch([src, src], [dst, dst], [T, T], R_CORR)
    assert nb == [n, n] and all(np.array_equal(x, want) for x in LB)
    gt, edges, Te, Le, unc = graph(12, 12, [(11, 0), (8, 0), (9, 3), (7, 2)])
    g = tpp.PoseGraph(R_CORR).optimize(12, [tuple(e) for e in edges.tolist()], Te, Le, [bool(u) for u in unc])
    c = ctx.optimize_pose_graph(12, edges, Te, Le, R_CORR, uncertain=unc)
    assert np.array_equal(np.stack(g["poses"]), c["poses"]) and np.array_equal(g["weights"], c["weights"])
    assert (g["iterations"], g["inner_iterations"], g["cost"]) == (c["iterations"], c["inner_iterations"], c["cost"])
    clouds = _sequence([600, 900, 700, 800], seed=7)
    pairs = [(0, 1), (1, 2), (2, 3), (3, 0)]
    solver = tpp.RobustRegistrationSolver(noise_bound=0.01, estimate_scaling=False, rotation_cost_threshold=1e-12)
    res = solver.solve_multiway(clouds, pairs, R_CORR, normal_search_radius=PAIR_FLAGS["normal_search_radius"],
                                fpfh_search_radius=PAIR_FLAGS["fpfh_search_radius"],
                                use_absolute_scale=PAIR_FLAGS["use_absolute_scale"],
                                use_crosscheck=PAIR_FLAGS["use_crosscheck"], use_tuple_test=PAIR_FLAGS["use_tuple_test"])
    assert res["pose_graph_status"] == 0
    mw = ctx.register_multiway(clouds, pairs, capi.default_params(noise_bound=0.01, estimate_scaling=0,
                                                                  rotation_cost_threshold=1e-12), R_CORR,
                               tuple_seeds=[0x7ea5e2 + 0x9E3779B97F4A7C15 * p & (2 ** 64 - 1) for p in range(4)],
                               **PAIR_FLAGS)[7]
    assert np.array_equal(np.stack(res["poses"]), mw["poses"])
    assert np.array_equal(np.asarray(res["edge_weights"]), mw["weights"])
    assert np.array_equal(np.stack(res["information"]), mw["information"])
