"""GPU tests of the round-2 additions (`pytest -m gpu`): the tensor-core graph kernel against the CUDA-core kernel and
the oracle, the retained-graph bookkeeping of a shared context (generation counter, inlier selection NONE), the
stage-timing log and the in-library multi-GPU batch call.  Everything goes through the C-ABI; the oracle is the checker."""
import importlib
import os
import subprocess
import sys

import numpy as np
import pytest

import oracle_lib as orc

capi = importlib.import_module("teaser-plusplus_b200.capi")
synth = importlib.import_module("teaser-plusplus_b200.synth")

pytestmark = pytest.mark.gpu
ROT_TOL = TRANS_TOL = 1e-4


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


# ------------------------------------------------------------------ tensor-core graph kernel
@pytest.mark.parametrize("cfg,n", [("C2", 1500), ("C2cube", 1100), ("C3", 2000), ("C4", 640), ("C5", 1700), ("C2", 130)])
def test_tc_kernel_is_used_and_bit_exact(ctx, cfg, n):
    """Tensor-core kernel (flag 1024; debug counter 7 counts the problems that took it): its bitset, degrees and edge
    count equal the oracle's and the default CUDA-core kernel's, and the on-device verification of every decided pair
    against the exact FP64 predicate (flag 2) finds no disagreement."""
    pr = synth.config_problem(cfg, 21, n=n)
    beta = 2 * pr["noise_bound"]
    obits, odeg, oe = orc.build_graph_bits(pr["src"], pr["dst"], pr["noise_bound"])
    ctx.set_flags(1024 | 2 | 4)
    bits, deg, ne = ctx.graph_build(pr["src"], pr["dst"], beta)
    cnt = ctx.debug_counters()
    ctx.set_flags(0)
    assert cnt["tc_problems"] == 1, "the problem did not take the tensor-core path"
    assert cnt["filter_mismatches"] == 0
    assert cnt["filter_rechecks"] < 0.01 * n * n + 64  # the exact path is the exception
    assert np.array_equal(bits, obits) and np.array_equal(deg, odeg) and ne == oe
    ctx.set_flags(4)
    bits2, deg2, ne2 = ctx.graph_build(pr["src"], pr["dst"], beta)
    cnt2 = ctx.debug_counters()
    ctx.set_flags(0)
    assert cnt2["tc_problems"] == 0
    assert np.array_equal(bits2, obits) and np.array_equal(deg2, odeg) and ne2 == oe


@pytest.mark.parametrize("cfg,n", [("C2", 1300), ("C2cube", 1000), ("C3", 1500), ("C5", 900), ("C2", 33)])
def test_v7_strip_kernel_bit_exact(ctx, cfg, n):
    """graph_strip3_kernel (flag 2048: one MUFU per pair, sign-bit column words, re-check queue + tc_patch_kernel):
    bit-identical to the oracle, every decided pair verified on the device, also with the exact-everything guard."""
    pr = synth.config_problem(cfg, 5, n=n)
    beta = 2 * pr["noise_bound"]
    obits, odeg, oe = orc.build_graph_bits(pr["src"], pr["dst"], pr["noise_bound"])
    for flags in (2048 | 2 | 4, 2048 | 4, 2048 | 1):
        ctx.set_flags(flags)
        bits, deg, ne = ctx.graph_build(pr["src"], pr["dst"], beta)
        cnt = ctx.debug_counters()
        ctx.set_flags(0)
        assert cnt["filter_mismatches"] == 0
        assert np.array_equal(bits, obits) and np.array_equal(deg, odeg) and ne == oe
        if not flags & 1:
            assert cnt["filter_rechecks"] < 0.01 * n * n + 64


def test_tc_kernel_falls_back_when_ill_conditioned(ctx):
    """A noise bound that is tiny against the extent of the clouds (C1-like: beta/D ~ 1e-4) makes the tensor-core
    filter's undecided band (E / (0.75 D) in |sqrt a - sqrt b|) wider than beta/64: prep_kernel routes the problem to the
    CUDA-core kernel; bits stay exact."""
    pr = synth.config_problem("C2", 4, n=400)
    src, dst = pr["src"].copy(), pr["dst"].copy()
    dst[::7] += 300.0
    nb = 1e-5
    obits, _, oe = orc.build_graph_bits(src, dst, nb)
    ctx.set_flags(1024 | 2 | 4)
    bits, _, ne = ctx.graph_build(src, dst, 2 * nb)
    cnt = ctx.debug_counters()
    ctx.set_flags(0)
    assert cnt["tc_problems"] == 0 and cnt["filter_mismatches"] == 0
    assert np.array_equal(bits, obits) and ne == oe


def test_tc_kernel_duplicates_coincident_points(ctx):
    """Zero-length TIMs (duplicate correspondences): a' = 0 +- error can come out negative, and with s = a + b <= beta^2
    the sign of the polynomial says nothing — those pairs must land in the exact path (the beta^4 floor of the band), not in
    a wrong bit."""
    pr = synth.config_problem("C2cube", 8, n=700)
    src, dst = pr["src"].copy(), pr["dst"].copy()
    for k in range(0, 60, 3):
        src[k + 1] = src[k]
    for k in range(100, 160, 3):
        dst[k + 1] = dst[k]
        src[k + 1] = src[k] + 1e-9
    obits, odeg, oe = orc.build_graph_bits(src, dst, pr["noise_bound"])
    ctx.set_flags(1024 | 2 | 4)
    bits, deg, ne = ctx.graph_build(src, dst, 2 * pr["noise_bound"])
    cnt = ctx.debug_counters()
    ctx.set_flags(0)
    assert cnt["tc_problems"] == 1 and cnt["filter_mismatches"] == 0
    assert np.array_equal(bits, obits) and np.array_equal(deg, odeg) and ne == oe


def test_tc_kernel_batch_mixed_with_fallback_problems(ctx):
    """One batch, some problems on the tensor-core path and some on the CUDA-core path: every problem equals its
    single-problem solve."""
    prs = [synth.config_problem("C4", 300 + b, n=520) for b in range(10)]
    for b in (2, 5, 9):  # blow up the extent of these: they fall back
        prs[b]["dst"][::11] += 5e3
    p = capi.default_params(**fixed_params(prs[0]["noise_bound"]))
    ctx.set_flags(1024 | 4)
    sols, cliques = ctx.solve_batch([q["src"] for q in prs], [q["dst"] for q in prs], p)
    cnt = ctx.debug_counters()
    ctx.set_flags(0)
    assert 1 <= cnt["tc_problems"] <= 9
    for b, q in enumerate(prs):
        o = orc.solve(q["src"], q["dst"], orc.default_params(**fixed_params(q["noise_bound"])))
        assert np.array_equal(cliques[b], o["clique"]) and int(sols[b]["n_edges"]) == o["sol"].n_edges


def test_tc_kernel_unknown_scale(ctx):
    """estimate_scaling=true: the operand tiles are built from the source cloud scaled by the TLS estimate."""
    pr = synth.config_problem("C4", 77, n=900)
    kw = fixed_params(pr["noise_bound"], estimate_scaling=1)
    src = pr["src"] * 1.7
    o = orc.solve(src, pr["dst"], orc.default_params(**kw))
    ctx.set_flags(1024 | 2 | 4)
    g = ctx.solve(src, pr["dst"], capi.default_params(**kw))
    cnt = ctx.debug_counters()
    ctx.set_flags(0)
    assert cnt["tc_problems"] == 1 and cnt["filter_mismatches"] == 0
    assert np.array_equal(g["clique"], o["clique"]) and g["n_edges"] == o["sol"].n_edges
    assert abs(g["scale"] - o["scale"]) < 1e-9


# ------------------------------------------------------------------ retained graph of a context
def test_last_graph_info_generation_and_none_mode(ctx):
    pr = synth.config_problem("C2", 1, n=300)
    p = capi.default_params(**fixed_params(pr["noise_bound"]))
    ctx.solve(pr["src"], pr["dst"], p)
    a = ctx.last_graph_info()
    assert a["B"] == 1 and a["n"] == 300 and a["has_graph"]
    ctx.solve(pr["src"][:200], pr["dst"][:200], p)
    b = ctx.last_graph_info()
    assert b["n"] == 200 and b["generation"] != a["generation"]
    # a stage call that re-uses the workspace invalidates the retained graph instead of leaving it dangling
    bits, _, _ = ctx.graph_build(pr["src"][:64], pr["dst"][:64], 2 * pr["noise_bound"])
    ctx.max_clique(bits, 64)
    c = ctx.last_graph_info()
    assert c["generation"] != b["generation"] and c["n"] == 0 and not c["has_graph"]
    # inlier selection NONE: the reference never populates the graph (registration.cc:607-650) -> empty adjacency
    ctx.solve(pr["src"], pr["dst"], capi.default_params(**fixed_params(pr["noise_bound"], inlier_selection_mode=3)))
    d = ctx.last_graph_info()
    assert d["n"] == 300 and not d["has_graph"]
    W = (300 + 63) // 64
    gb = np.full((300, W), 0xFFFFFFFFFFFFFFFF, dtype=np.uint64)
    gd = np.full(300, 7, dtype=np.int32)
    ctx._ck(capi.lib().tzr_last_graph(ctx._h, 0, capi._p(gb, capi.C.c_uint64), capi._p(gd, capi.C.c_int32)))
    assert not gb.any() and not gd.any()


def test_facade_getters_survive_another_solver_on_the_same_thread():
    """Two façade objects share the per-thread context: the lazy getInlierGraph() of the first one must not return the
    second one's graph (ADVICE r1: stale / overflowing tzr_last_graph)."""
    host = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "teaser-plusplus_b200", "host")
    subprocess.check_call(["make", "-s", "-C", host])
    sys.path.insert(0, os.path.join(host, "python"))
    import teaserpp_python as tp
    pa = synth.config_problem("C4", 31, n=400)
    pb = synth.config_problem("C4", 32, n=900)   # larger: would overflow a buffer sized for the first solver
    def mk(pr, mode=None):
        p = tp.RobustRegistrationSolver.Params()
        p.noise_bound = pr["noise_bound"]
        p.estimate_scaling = False
        p.rotation_cost_threshold = 1e-12
        if mode is not None:
            p.inlier_selection_mode = mode
        return tp.RobustRegistrationSolver(p)
    sa, sb = mk(pa), mk(pb)
    sa.solve(pa["src"].T, pa["dst"].T)
    sb.solve(pb["src"].T, pb["dst"].T)
    _, dega, ea = orc.build_graph_bits(pa["src"], pa["dst"], pa["noise_bound"])
    _, degb, eb = orc.build_graph_bits(pb["src"], pb["dst"], pb["noise_bound"])
    adj_a = sa.getInlierGraph()     # context now holds sb's graph -> re-solve, then the right graph
    assert [len(r) for r in adj_a] == dega.tolist()
    adj_b = sb.getInlierGraph()     # and sb's was overwritten by that re-solve
    assert [len(r) for r in adj_b] == degb.tolist()
    # NONE mode: empty graph like the reference
    sn = mk(pa, tp.RobustRegistrationSolver.INLIER_SELECTION_MODE.NONE)
    sn.solve(pa["src"][pa["inliers"]].T, pa["dst"][pa["inliers"]].T)
    assert sn.getInlierGraph() == []


# ------------------------------------------------------------------ stage log
def test_stage_log_accumulates_without_per_step_sync(ctx):
    import torch
    prs = [synth.config_problem("C4", 500 + b, n=512) for b in range(16)]
    src = torch.tensor(np.stack([q["src"] for q in prs]), device="cuda")
    dst = torch.tensor(np.stack([q["dst"] for q in prs]), device="cuda")
    sol = torch.zeros(16 * capi.SOLUTION_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    clq = torch.zeros((16, 512), dtype=torch.int32, device="cuda")
    p = capi.default_params(**fixed_params(prs[0]["noise_bound"]))
    ctx.stage_log(True)
    for _ in range(5):
        ctx.solve_batch_dev(p, 16, 512, src.data_ptr(), dst.data_ptr(), sol.data_ptr(), clq.data_ptr())
    sums, calls = ctx.stage_log_read()
    ctx.stage_log(False)
    assert calls == 5 and all(v > 0 for v in sums.values())
    ctx.solve_batch_dev(p, 16, 512, src.data_ptr(), dst.data_ptr(), sol.data_ptr(), clq.data_ptr())
    ctx.synchronize()
    one = ctx.last_stage_ms()
    assert 0.2 * sums["graph"] / 5 < one["graph"] < 5 * sums["graph"] / 5
    torch.cuda.synchronize()


# ------------------------------------------------------------------ multi-GPU batch inside the library
def test_solve_batch_multi_matches_single_device(ctx):
    """tzr_solve_batch_multi over every visible device (1 on a single-GPU machine, >= 2 on a multi-GPU one):
    ragged batch, results in caller order, identical to the single-context call."""
    import torch
    sizes = [400, 400, 650, 400, 300, 650, 400, 300, 500, 400, 400, 650]
    prs = [synth.config_problem("C4", 900 + b, n=n) for b, n in enumerate(sizes)]
    p = capi.default_params(**fixed_params(prs[0]["noise_bound"]))
    sols, cliques = capi.solve_batch_multi([q["src"] for q in prs], [q["dst"] for q in prs], p)
    sols1, cliques1 = ctx.solve_batch([q["src"] for q in prs], [q["dst"] for q in prs], p)
    for b in range(len(prs)):
        assert np.array_equal(cliques[b], cliques1[b]) and np.array_equal(cliques[b], prs[b]["inliers"])
        assert np.array_equal(sols[b]["rotation"], sols1[b]["rotation"])
        assert np.array_equal(sols[b]["translation"], sols1[b]["translation"])
    if torch.cuda.device_count() >= 2:
        sols2, cliques2 = capi.solve_batch_multi([q["src"] for q in prs], [q["dst"] for q in prs], p, devices=[1, 0])
        for b in range(len(prs)):
            assert np.array_equal(cliques2[b], cliques1[b])
            assert np.array_equal(sols2[b]["rotation"], sols1[b]["rotation"])


def test_facade_solve_batch():
    """RobustRegistrationSolver::solveBatch / teaserpp_python solve_batch: the drop-in surface reaches every GPU of the
    node from one call, no torchrun."""
    host = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "teaser-plusplus_b200", "host")
    subprocess.check_call(["make", "-s", "-C", host])
    sys.path.insert(0, os.path.join(host, "python"))
    import teaserpp_python as tp
    prs = [synth.config_problem("C4", 1200 + b, n=450) for b in range(9)]
    p = tp.RobustRegistrationSolver.Params()
    p.noise_bound = prs[0]["noise_bound"]
    p.estimate_scaling = False
    p.rotation_cost_threshold = 1e-12
    s = tp.RobustRegistrationSolver(p)
    sols, cliques = s.solve_batch([q["src"].T for q in prs], [q["dst"].T for q in prs])
    assert len(sols) == 9
    for b, q in enumerate(prs):
        one = tp.RobustRegistrationSolver(p)
        ref = one.solve(q["src"].T, q["dst"].T)
        assert sols[b].valid and cliques[b] == one.getInlierMaxClique() == q["inliers"].tolist()
        assert np.array_equal(sols[b].rotation, ref.rotation) and np.array_equal(sols[b].translation, ref.translation)
