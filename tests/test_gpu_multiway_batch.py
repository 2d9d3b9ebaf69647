"""Many scan sequences in one multiway call (tzr_register_cloud_pairs_multiway(_line_process)_batch, DESIGN.md §3.25):
the batch against the chain of public calls (register_cloud_pairs_icp -> information_matrix_batch ->
optimize_pose_graph_batch / global_optimization_batch -> voxel_downsample_batch of the host-built concatenation),
byte for byte; each sequence against a batch of one, reordered sequences and interleaved pairs; the routes against the
single register_multiway; per-graph refusals; launch counts; the fused map against ground truth; the retained solve;
the call-level refusals with a context; the C++ and pybind façades against the C ABI."""
import importlib
import os
import subprocess
import sys

import numpy as np
import pytest
from scipy.spatial import cKDTree

from multiway_map_reference import transform_concat
from test_gpu_icp import PAIR_FLAGS, _retained, _sequence
import test_multiway_batch_cpu as cpu

capi = importlib.import_module("teaser-plusplus_b200.capi")
pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R_CORR = 0.05
VOX = 0.02
PRM = dict(noise_bound=0.01, estimate_scaling=0, rotation_cost_threshold=1e-12)
LP_KEYS = ("iterations", "trials", "stop_reason", "pruned", "mu")


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


def colours_of(clouds, seed):
    rng = np.random.default_rng(seed)
    return [rng.uniform(0, 1, size=(len(c), 3)).astype(np.float32) for c in clouds]


def sequences(seed=11, sizes=((600, 900, 700, 800), (500, 650, 700), (700, 600, 800, 550, 650))):
    seqs = [_sequence(list(s), seed + k) for k, s in enumerate(sizes)]
    pairs = [[(k, k + 1) for k in range(len(s) - 1)] + [(len(s) - 1, 0)] for s in seqs]
    return seqs, pairs


def pair_bytes(res):
    """Every per-pair output of one sequence's result, the solutions without their stage timings"""
    sols, status, index, corr, clq, gs, icp, d = res
    stage = capi.SOLUTION_DTYPE.fields["stage_ms"][1]
    keys = [k for k in ("information", "counts", "weights", "mask", "confidence", "kept") if k in d]
    return ([s.tobytes()[:stage] for s in sols], status.tobytes(), index.tobytes(), [c.tobytes() for c in corr],
            [c.tobytes() for c in clq], gs, icp.tobytes(), [np.ascontiguousarray(d[k]).tobytes() for k in keys])


def graph_bytes(d):
    return {k: (np.ascontiguousarray(v).tobytes() if isinstance(v, np.ndarray) else v) for k, v in d.items()
            if k not in ("information", "counts", "weights", "mask", "confidence", "kept")}


def as_bytes(res):
    return pair_bytes(res), graph_bytes(res[7])


def batch(ctx, seqs, pairs, optimizer="gnc_tls", colors=None, **kw):
    return ctx.register_multiway_batch(seqs, pairs, capi.default_params(**PRM), R_CORR, optimizer=optimizer,
                                       colors=colors, **kw, **PAIR_FLAGS)


def transforms_of(icp, refined):
    return [dict(scale=float(icp[p]["transform"]["scale"]), rotation=icp[p]["transform"]["rotation"],
                 translation=icp[p]["transform"]["translation"]) for p in refined]


# ---- the chain of public calls ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("colored", [False, True])
@pytest.mark.parametrize("optimizer", ["gnc_tls", "line_process"])
def test_batch_equals_the_chain_of_public_calls(ctx, optimizer, colored):
    seqs, pairs = sequences()
    cols = [colours_of(s, 40 + k) for k, s in enumerate(seqs)] if colored else None
    got = batch(ctx, seqs, pairs, optimizer, cols, map_voxel_size=VOX)
    flat = capi.multiway_batch_table(seqs, pairs, colors=cols)
    prm = capi.default_params(**PRM)
    chain = ctx.register_cloud_pairs_icp(flat["clouds"], flat["pairs"], prm, R_CORR,
                                         method="colored" if colored else "point_to_plane", colors=flat["colors"],
                                         **PAIR_FLAGS)
    stage = capi.SOLUTION_DTYPE.fields["stage_ms"][1]
    icp = chain[6]
    graphs = []
    for g, (a, b) in enumerate(zip(flat["pair_offsets"][:-1], flat["pair_offsets"][1:])):
        res = got[g]
        assert [s.tobytes()[:stage] for s in res[0]] == [s.tobytes()[:stage] for s in chain[0][a:b]]
        assert res[1].tobytes() == chain[1][a:b].tobytes() and res[6].tobytes() == icp[a:b].tobytes()
        assert all(np.array_equal(x, y) for x, y in zip(res[3], chain[3][a:b])) and res[5] == chain[5][a:b]
        refined = [p for p in range(a, b) if icp[p]["transform"]["scale"] > 0]
        assert len(refined) >= 2
        o = flat["offsets"][g]
        trs = transforms_of(icp, refined)
        L, n = ctx.information_matrix_batch([flat["clouds"][flat["pairs"][p][0]] for p in refined],
                                            [flat["clouds"][flat["pairs"][p][1]] for p in refined], trs, R_CORR)
        d = res[7]
        for j, p in enumerate(refined):
            assert d["information"][p - a].tobytes() == L[j].tobytes() and d["counts"][p - a] == n[j]
        graphs.append(dict(K=len(seqs[g]), edges=[tuple(flat["pairs"][p] - o) for p in refined], transforms=trs,
                           information=L, uncertain=[int(flat["uncertain"][p]) for p in refined], refined=refined))
    args = [{k: v for k, v in x.items() if k != "refined"} for x in graphs]
    pg = ctx.global_optimization_batch(args, R_CORR) if optimizer == "line_process" else \
        ctx.optimize_pose_graph_batch(args, R_CORR)
    w, m = ("confidence", "kept") if optimizer == "line_process" else ("weights", "mask")
    for g, x in enumerate(graphs):
        d, want = got[g][7], pg[g]
        a = flat["pair_offsets"][g]
        local = [p - a for p in x["refined"]]
        assert d["status"] == want["status"] == 0
        assert d["poses"].tobytes() == want["poses"].tobytes()
        assert d[w][local].tobytes() == want[w].tobytes() and np.array_equal(d[m][local], want[m])
        keys = LP_KEYS + ("residual",) if optimizer == "line_process" else ("iterations", "inner_iterations", "cost")
        assert all(d[k] == want[k] for k in keys)
        # the fused map: voxel_downsample(_colors)_batch of the host-built concatenation, bit for bit
        cat = transform_concat(seqs[g], d["poses"])
        if colored:
            vp, vc = ctx.voxel_downsample(cat, VOX, colors=np.concatenate(cols[g]))[:2]
            assert d["map_colors"].tobytes() == vc.tobytes()
        else:
            vp = ctx.voxel_downsample(cat, VOX)
            vp = vp[0] if isinstance(vp, tuple) else vp
        assert len(d["map"]) > 0 and d["map"].tobytes() == np.ascontiguousarray(vp, dtype=np.float32).tobytes()


# ---- independence -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("optimizer", ["gnc_tls", "line_process"])
def test_each_sequence_equals_a_batch_of_one_and_any_order(ctx, optimizer):
    seqs, pairs = sequences(seed=21)
    seeds = [[(0x9E3779B97F4A7C15 * (17 * g + p + 1)) & (2 ** 64 - 1) for p in range(len(pr))]
             for g, pr in enumerate(pairs)]
    got = batch(ctx, seqs, pairs, optimizer, tuple_seeds=seeds, map_voxel_size=VOX)
    assert all(r[7]["status"] == 0 for r in got)
    for g in range(len(seqs)):
        one = batch(ctx, [seqs[g]], [pairs[g]], optimizer, tuple_seeds=[seeds[g]], map_voxel_size=VOX)[0]
        assert as_bytes(one) == as_bytes(got[g]), g
    order = [2, 0, 1]
    rev = batch(ctx, [seqs[g] for g in order], [pairs[g] for g in order], optimizer,
                tuple_seeds=[seeds[g] for g in order], map_voxel_size=VOX)
    for j, g in enumerate(order):
        assert as_bytes(rev[j]) == as_bytes(got[g])
    # the pairs interleaved in the flat table: every per-pair output moves with its pair, every graph output stays
    flat = capi.multiway_batch_table(seqs, pairs, tuple_seeds=seeds)
    P = len(flat["pairs"])
    perm = np.argsort([(k - a) * 10 + g for g, (a, b) in enumerate(zip(flat["pair_offsets"][:-1],
                                                                         flat["pair_offsets"][1:]))
                       for k in range(a, b)], kind="stable")
    assert list(perm) != list(range(P))
    opt = capi.line_process_params(R_CORR) if optimizer == "line_process" else capi.pose_graph_params(R_CORR)
    out = ctx._register_pairs(flat["clouds"], flat["pairs"][perm], capi.default_params(**PRM),
                              PAIR_FLAGS["normal_search_radius"], PAIR_FLAGS["fpfh_search_radius"],
                              PAIR_FLAGS["use_absolute_scale"], PAIR_FLAGS["use_crosscheck"],
                              PAIR_FLAGS["use_tuple_test"], 0.0, [flat["tuple_seeds"][p] for p in perm],
                              capi.icp_params(R_CORR, max_iteration=30), plane=True,
                              multiway=(flat["uncertain"][perm], opt, flat["offsets"], VOX))
    inv = np.argsort(perm)
    stage = capi.SOLUTION_DTYPE.fields["stage_ms"][1]
    mw = out[7]
    for g, (a, b) in enumerate(zip(flat["pair_offsets"][:-1], flat["pair_offsets"][1:])):
        rows = inv[a:b]
        d = got[g][7]
        assert [out[0][r].tobytes()[:stage] for r in rows] == [s.tobytes()[:stage] for s in got[g][0]]
        assert out[6][rows].tobytes() == got[g][6].tobytes()
        for k in ("information", "counts", "weights", "mask", "confidence", "kept"):
            if k in d:
                assert mw[k][rows].tobytes() == np.ascontiguousarray(d[k]).tobytes()
        gd = dict(mw["graphs"][g])
        gd["poses"] = mw["poses"][flat["offsets"][g]:flat["offsets"][g + 1]]
        assert graph_bytes(gd) == graph_bytes(d)


# ---- the routes against the single entry ------------------------------------------------------------------------------
@pytest.mark.parametrize("optimizer", ["gnc_tls", "line_process"])
def test_routes_against_the_single_entry(ctx, optimizer):
    big = _sequence([600, 700] * 65, seed=31)
    big_pairs = [(k, k + 1) for k in range(129)] + [(k + 8, k) for k in range(0, 120, 40)]
    seqs, pairs = sequences(seed=33, sizes=((600, 900, 700, 800),))
    got = batch(ctx, [big] + seqs, [big_pairs] + pairs, optimizer)
    prm = capi.default_params(**PRM)
    single = [ctx.register_multiway(s, p, prm, R_CORR, optimizer=optimizer, **PAIR_FLAGS)
              for s, p in zip([big] + seqs, [big_pairs] + pairs)]
    # K = 130: the single entry's route, byte for byte, poses included
    assert got[0][7]["status"] == single[0][7]["status"] == 0
    assert pair_bytes(got[0]) == pair_bytes(single[0])
    for k, v in single[0][7].items():
        assert np.ascontiguousarray(got[0][7][k]).tobytes() == np.ascontiguousarray(v).tobytes(), k
    # K <= 128: the same pairs and information matrices, and the same decisions
    d, s = got[1][7], single[1][7]
    assert pair_bytes(got[1]) == pair_bytes(single[1])
    assert d["status"] == s["status"] == 0
    if optimizer == "line_process":
        assert all(d[k] == s[k] for k in LP_KEYS) and np.array_equal(d["kept"], s["kept"])
    else:
        assert (d["iterations"], d["inner_iterations"]) == (s["iterations"], s["inner_iterations"])
        assert np.array_equal(d["mask"], s["mask"])
    assert np.allclose(d["poses"], s["poses"], atol=1e-9)


# ---- per-graph refusals -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("optimizer", ["gnc_tls", "line_process"])
def test_refused_graphs_leave_their_neighbours_solved(ctx, optimizer):
    seqs, pairs = sequences(seed=41, sizes=((600, 900, 700), (500, 650, 700, 800)))
    lone = _sequence([600, 700], seed=42)
    lone[1] = lone[1][:2].copy()  # two points: the only pair is not solved, so the graph has no edge
    split = _sequence([600, 900, 700, 800], seed=43)  # two pairs that share no cloud: a disconnected graph
    all_seqs = [seqs[0], lone, seqs[1], split]
    all_pairs = [pairs[0], [(0, 1)], pairs[1], [(0, 1), (2, 3)]]
    got = batch(ctx, all_seqs, all_pairs, optimizer, map_voxel_size=VOX)
    for g in (1, 3):
        d = got[g][7]
        assert d["status"] == capi.TZR_ERR_INVALID_ARG
        assert not d["poses"][:, :3].any() and len(d["map"]) == 0
        assert not (d["weights"] if optimizer == "gnc_tls" else d["confidence"]).any()
        assert not (d["mask"] if optimizer == "gnc_tls" else d["kept"]).any()
    assert not got[1][7]["information"].any()
    for g in (0, 2):
        assert got[g][7]["status"] == 0 and len(got[g][7]["map"]) > 0
        one = batch(ctx, [all_seqs[g]], [all_pairs[g]], optimizer, map_voxel_size=VOX)[0]
        assert as_bytes(one) == as_bytes(got[g])


# ---- launches ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("optimizer", ["gnc_tls", "line_process"])
def test_pose_graph_step_adds_one_or_two_launches(ctx, optimizer):
    seqs = [_sequence([600, 700, 650], seed=100 + g) for g in range(64)]
    pairs = [[(0, 1), (1, 2), (2, 0)]] * 64
    prm = capi.default_params(**PRM)
    flat = capi.multiway_batch_table(seqs, pairs)
    # the information step's own launches: the single chained entry minus its ICP chain and its pose graph
    l0 = ctx.kernel_launches()
    one = ctx.register_multiway(seqs[0], pairs[0], prm, R_CORR, optimizer=optimizer, **PAIR_FLAGS)
    l1 = ctx.kernel_launches()
    icp_one = ctx.register_cloud_pairs_icp(seqs[0], pairs[0], prm, R_CORR, method="point_to_plane", **PAIR_FLAGS)[6]
    l2 = ctx.kernel_launches()
    refined = [p for p in range(3) if icp_one[p]["transform"]["scale"] > 0]
    trs = transforms_of(icp_one, refined)
    L = one[7]["information"][refined]
    unc = [0 if b == a + 1 else 1 for a, b in pairs[0]]
    g0 = dict(K=3, edges=[pairs[0][p] for p in refined], transforms=trs, information=L,
              uncertain=[unc[p] for p in refined])
    single = ctx.global_optimization if optimizer == "line_process" else ctx.optimize_pose_graph
    l3 = ctx.kernel_launches()
    single(g0["K"], g0["edges"], g0["transforms"], g0["information"], R_CORR, uncertain=g0["uncertain"])
    info_launches = (l1 - l0) - (l2 - l1) - (ctx.kernel_launches() - l3)
    assert info_launches > 0
    l4 = ctx.kernel_launches()
    got = batch(ctx, seqs, pairs, optimizer)
    l5 = ctx.kernel_launches()
    ctx.register_cloud_pairs_icp(flat["clouds"], flat["pairs"], prm, R_CORR, method="point_to_plane", **PAIR_FLAGS)
    l6 = ctx.kernel_launches()
    assert all(r[7]["status"] == 0 for r in got)
    assert (l5 - l4) - (l6 - l5) - info_launches == (2 if optimizer == "line_process" else 1)
    # the map: one transform launch and the voxel pipeline's ten
    l7 = ctx.kernel_launches()
    batch(ctx, seqs, pairs, optimizer, map_voxel_size=VOX)
    assert ctx.kernel_launches() - l7 == (l5 - l4) + 11


# ---- the fused map against ground truth -------------------------------------------------------------------------------
def test_map_matches_the_ground_truth_fused_cloud(ctx):
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    probe = importlib.import_module("multiway_probe")
    clouds, truth = probe.sequence(800, 8, seed=5)
    pairs = [(k, k + 1) for k in range(7)] + [(k + 2, k) for k in range(0, 6, 3)]
    got = ctx.register_multiway_batch([clouds], [pairs], capi.default_params(**PRM), R_CORR, map_voxel_size=VOX,
                                      **probe.FLAGS)[0][7]
    assert got["status"] == 0
    fused = transform_concat(clouds, truth)
    dist, _ = cKDTree(fused.astype(np.float64)).query(got["map"].astype(np.float64))
    assert len(got["map"]) < len(fused) and dist.max() < R_CORR and np.median(dist) < VOX


# ---- the retained solve -----------------------------------------------------------------------------------------------
def test_retained_solve_is_the_registration(ctx):
    seqs, pairs = sequences(seed=51)
    flat = capi.multiway_batch_table(seqs, pairs)
    prm = capi.default_params(**PRM)
    plain = ctx.register_cloud_pairs(flat["clouds"], flat["pairs"], prm, **PAIR_FLAGS)
    S = int((plain[2] >= 0).sum())
    want = _retained(ctx, S)
    batch(ctx, seqs, pairs, "line_process", map_voxel_size=VOX)
    assert _retained(ctx, S) == want


# ---- call-level refusals with a context -------------------------------------------------------------------------------
@pytest.mark.parametrize("lp", [False, True])
@pytest.mark.parametrize("case", sorted(cpu.REFUSALS) + ["estimate_scaling", "negative voxel", "map without buffers"])
def test_call_level_refusals(ctx, case, lp):
    """Each refusal with a context: TZR_ERR_INVALID_ARG, nothing written, and (for the partition and map cases) the
    many-sequence check's own message, after another entry's refusal left a different one"""
    def last_error():
        return capi.lib().tzr_last_error(ctx._h).decode()

    def other_refusal():
        pg = capi.pose_graph_params(R_CORR)
        assert capi.lib().tzr_pose_graph_optimize_batch(ctx._h, cpu.C.byref(pg), 0, *([None] * 13)) == \
            capi.TZR_ERR_INVALID_ARG
        assert not last_error().startswith("multiway batch")

    if case in cpu.REFUSALS:
        offsets, pairs, G = cpu.REFUSALS[case]
        k = cpu.table(offsets, pairs, G)
        k["clouds"] += [k["clouds"][0]] * (4 - len(k["clouds"]))
        k["n"] = np.full(4, 8, dtype=np.int32)
        other_refusal()
        assert cpu.call(ctx._h, k, len(offsets) - 1 if G is None else G, lp=lp) == (capi.TZR_ERR_INVALID_ARG, False)
        assert last_error().startswith("multiway batch"), last_error()
        return
    if case == "estimate_scaling":
        seqs, pairs = sequences(seed=61, sizes=((600, 900),))
        with pytest.raises(capi.TzrError):
            ctx.register_multiway_batch(seqs, [[(0, 1)]], capi.default_params(noise_bound=0.01, estimate_scaling=1),
                                        R_CORR, optimizer="line_process" if lp else "gnc_tls", **PAIR_FLAGS)
        return
    k = cpu.table(map_voxel_size=-1.0 if case == "negative voxel" else VOX)
    if case == "map without buffers":
        k["maps"] = None
    other_refusal()
    assert cpu.call(ctx._h, k, 2, lp=lp) == (capi.TZR_ERR_INVALID_ARG, False)
    assert last_error().startswith("multiway batch"), last_error()


# ---- the façades ------------------------------------------------------------------------------------------------------
HOST = os.path.join(ROOT, "teaser-plusplus_b200", "host")
CSRC = os.path.join(ROOT, "teaser-plusplus_b200", "csrc")


def test_cpp_facade_equals_the_c_abi(tmp_path):
    """RobustRegistrationSolver::solveMultiwayBatch against the C ABI (tests/cpp/multiway_batch_test.cc)"""
    subprocess.check_call(["make", "-s", "-C", HOST])
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    exe = str(tmp_path / "multiway_batch_test")
    subprocess.check_call([cxx, "-std=c++17", "-O1", "-I", os.path.join(HOST, "include"), "-I",
                           os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "multiway_batch_test.cc"),
                           "-L", HOST, "-lteaser_registration", "-L", CSRC, "-lteaser_b200",
                           f"-Wl,-rpath,{HOST}:{CSRC}", "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr


@pytest.mark.parametrize("optimizer", ["gnc_tls", "line_process"])
def test_pybind_equals_ctypes(ctx, optimizer):
    """pybind's solve_multiway_batch against Context.register_multiway_batch: the same seeds (tuple_seed + golden j per
    sequence pair j), so every output byte for byte"""
    subprocess.check_call(["make", "-s", "-C", HOST])
    sys.path.insert(0, os.path.join(HOST, "python"))
    import teaserpp_python as tpp
    seqs, pairs = sequences(seed=71, sizes=((600, 900, 700), (500, 650, 700, 800)))
    cols = [colours_of(s, 80 + k) for k, s in enumerate(seqs)] if optimizer == "gnc_tls" else None
    seed0 = 0x7ea5e2
    seeds = [[(seed0 + 0x9E3779B97F4A7C15 * j) & (2 ** 64 - 1) for j in range(len(p))] for p in pairs]
    want = batch(ctx, seqs, pairs, optimizer, cols, tuple_seeds=seeds, map_voxel_size=VOX)
    prm = tpp.RobustRegistrationSolver.Params()
    prm.noise_bound, prm.estimate_scaling, prm.rotation_cost_threshold = 0.01, False, 1e-12
    kw = dict(global_optimization=tpp.GlobalOptimization(R_CORR)) if optimizer == "line_process" else {}
    got = tpp.RobustRegistrationSolver(prm).solve_multiway_batch(
        seqs, pairs, R_CORR, tuple_seed=seed0, colors=cols, map_voxel_size=VOX, **kw, **PAIR_FLAGS)
    assert len(got) == len(seqs)
    for g, r in enumerate(got):
        d = want[g][7]
        w, m = ("confidence", "kept") if optimizer == "line_process" else ("weights", "mask")
        assert r["pose_graph_status"] == d["status"] == 0
        assert np.stack(r["poses"]).tobytes() == d["poses"].tobytes()
        assert np.asarray(r["edge_weights"]).tobytes() == d[w].tobytes()
        assert np.array_equal(np.asarray(r["edge_inliers"]), d[m])
        assert np.stack(r["information"]).tobytes() == d["information"].tobytes()
        assert np.asarray(r["map"], dtype=np.float32).tobytes() == d["map"].tobytes() and len(d["map"]) > 0
        if cols is not None:
            assert np.asarray(r["map_colors"], dtype=np.float32).tobytes() == d["map_colors"].tobytes()
        if optimizer == "line_process":
            assert r["line_process"]["pruned"] == d["pruned"]
        else:
            assert (r["iterations"], r["inner_iterations"], r["cost"]) == (d["iterations"], d["inner_iterations"],
                                                                          d["cost"])
        icp = want[g][6]
        for j, q in enumerate(r["pairs"]):
            assert q["status"] == want[g][1][j] and q["refined"] == (icp[j]["transform"]["scale"] > 0)
