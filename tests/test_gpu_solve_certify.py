"""Certifying batched solves on the device (run on an H100: `pytest -m gpu`).

tzr_last_inliers returns every problem's masks of the most recent solve, byte for byte what tzr_solve gives for that
problem alone, on every solve entry.  tzr_certify_last_solve certifies problems of that solve with inputs gathered on
the device; the host-built inputs it is held to come from tests/rotation_reference.py (chain_tims / complete_tims,
the device's TIM rule replayed from a clique and a scale).
"""
import importlib
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
import certifier_oracle as co  # noqa: E402
import rotation_reference as rr  # noqa: E402

capi = importlib.import_module("teaser-plusplus_b200.capi")
synth = importlib.import_module("teaser-plusplus_b200.synth")

pytestmark = pytest.mark.gpu

TOL = 1e-7
ONE_CLASS = 16777216
LOOP_EIG = 2097152
NB = synth.NOISE_BOUND_SIGMA_001


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


def problem(n, seed, outliers=0.9, scale=1.0):
    pr = synth.make_problem(n, outliers if n > 2 else 0.0, 9000 + seed, "ball")
    return pr["src"], np.ascontiguousarray(scale * pr["dst"])


def no_clique(n):
    # grid points 0.1 apart, target scaled by 3: no pair is consistent, the clique has one point, the solution is invalid
    g = np.stack(np.meshgrid(*[np.arange(8)] * 3, indexing="ij"), -1).reshape(-1, 3)[:n] * 0.1
    return np.ascontiguousarray(g, dtype=np.float64), np.ascontiguousarray(3.0 * g)


def _close(a, b, tol):
    return len(a) == len(b) and (len(a) == 0 or np.abs(a - b).max() <= tol * max(1.0, np.abs(b).max()))


def retained_masks(ctx, B):
    return [ctx.last_inliers(b) for b in range(B)]


def check_masks(ctx, probs, prm, got):
    """got (the retained masks of a batch) against tzr_solve on each problem alone."""
    for b, (s, d) in enumerate(probs):
        one = ctx.solve(s, d, prm)
        rot, trans = got[b]
        if not one["valid"]:
            assert rot.size == 0 and trans.size == 0, b
            continue
        assert np.array_equal(rot, one["rot_inliers"]) and np.array_equal(trans, one["trans_inliers"]), b
        # tzr_solve retains its own problem too
        r1, t1 = ctx.last_inliers(0)
        assert np.array_equal(r1, one["rot_inliers"]) and np.array_equal(t1, one["trans_inliers"]), b


def host_batch(ctx, probs, prm):
    ctx.set_flags(0)
    sols, _ = ctx.solve_batch([p[0] for p in probs], [p[1] for p in probs], prm)
    return sols


def ragged_dev(ctx, probs, prm):
    torch = pytest.importorskip("torch")
    sizes = [len(p[0]) for p in probs]
    src = torch.from_numpy(np.concatenate([p[0] for p in probs])).cuda()
    dst = torch.from_numpy(np.concatenate([p[1] for p in probs])).cuda()
    sol_t = torch.zeros(len(sizes) * capi.SOLUTION_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    ctx.solve_batch_ragged_dev(prm, sizes, src.data_ptr(), dst.data_ptr(), sol_t.data_ptr())
    return (src, dst, sol_t)  # no host synchronisation: the caller reads the masks right away


CASES = [
    ("chain_gnc", dict(), [300, 300, 300]),
    ("chain_fgr", dict(rotation_estimation_algorithm=1), [300, 250, 420]),
    ("chain_quatro", dict(rotation_estimation_algorithm=2), [300, 320]),
    ("complete_gnc", dict(rotation_tim_graph=1), [60, 60, 45]),
    ("complete_fgr", dict(rotation_tim_graph=1, rotation_estimation_algorithm=1), [60, 50]),
    ("scale_small", dict(estimate_scaling=1), [120, 200, 200]),
    ("scale_large", dict(estimate_scaling=1), [600, 1000, 1000]),
    ("kcore", dict(inlier_selection_mode=2), [400, 400, 700]),
    ("none", dict(inlier_selection_mode=3), [80, 80, 50]),
]


@pytest.mark.parametrize("name,kw,sizes", CASES, ids=[c[0] for c in CASES])
def test_masks_every_entry_point(ctx, name, kw, sizes):
    torch = pytest.importorskip("torch")
    prm = params(**kw)
    scale = 1.3 if kw.get("estimate_scaling") else 1.0
    probs = [problem(n, i, 0.5 if kw.get("rotation_tim_graph") else 0.9, scale) for i, n in enumerate(sizes)]
    probs.append(no_clique(min(sizes)))  # counts 0 and 0
    uniform = [problem(sizes[0], 40 + i, 0.5 if kw.get("rotation_tim_graph") else 0.9, scale) for i in range(3)]
    # tzr_solve_batch, uniform
    host_batch(ctx, uniform, prm)
    check_masks(ctx, uniform, prm, retained_masks(ctx, len(uniform)))
    # tzr_solve_batch, ragged, with and without one class
    for flags in (0, ONE_CLASS):
        ctx.set_flags(flags)
        ctx.solve_batch([p[0] for p in probs], [p[1] for p in probs], prm)
        got = retained_masks(ctx, len(probs))
        ctx.set_flags(0)
        check_masks(ctx, probs, prm, got)
    # tzr_solve_batch_dev, uniform, from torch tensors
    n = len(uniform[0][0])
    src = torch.from_numpy(np.stack([p[0] for p in uniform])).cuda()
    dst = torch.from_numpy(np.stack([p[1] for p in uniform])).cuda()
    sol_t = torch.zeros(len(uniform) * capi.SOLUTION_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    ctx.solve_batch_dev(prm, len(uniform), n, src.data_ptr(), dst.data_ptr(), sol_t.data_ptr())
    check_masks(ctx, uniform, prm, retained_masks(ctx, len(uniform)))
    # tzr_solve_batch_ragged_dev
    keep = ragged_dev(ctx, probs, prm)
    got = retained_masks(ctx, len(probs))
    del keep
    check_masks(ctx, probs, prm, got)


def test_masks_large_route_problem():
    c = capi.Context(0, max_n=65536)
    try:
        probs = [problem(500, 1, 0.97), problem(33000, 2, 0.97), problem(900, 3, 0.97)]
        prm = params()
        c.solve_batch([p[0] for p in probs], [p[1] for p in probs], prm)
        got = retained_masks(c, 3)
        assert got[1][0].size > 0
        check_masks(c, probs, prm, got)
    finally:
        c.close()


def test_retention(ctx):
    fresh = capi.Context(0)
    try:
        with pytest.raises(capi.TzrError):
            fresh.last_inliers(0)
        with pytest.raises(capi.TzrError):
            fresh.certify_last()
        s, d = problem(200, 5)
        prm = params()
        fresh.solve(s, d, prm)
        fresh.last_inliers(0)
        with pytest.raises(capi.TzrError):
            fresh.last_inliers(1)
        with pytest.raises(capi.TzrError):
            fresh.last_inliers(-1)
        with pytest.raises(capi.TzrError):
            fresh.certify_last(problems=[1])
        fresh.graph_build(s, d, 2 * NB)
        with pytest.raises(capi.TzrError):
            fresh.last_inliers(0)
        with pytest.raises(capi.TzrError):
            fresh.certify_last()
        fresh.solve(s, d, prm)
        bits, _ = fresh.last_graph(0, len(s))
        fresh.max_clique(bits, len(s))
        with pytest.raises(capi.TzrError):
            fresh.last_inliers(0)
    finally:
        fresh.close()


def certify_host(ctx, probs, sols, cliques, masks, complete, noise_bounds):
    """tzr_certify_batch on host-built inputs, one noise bound per call (a list of single calls when they differ)."""
    R, S, D, T = [], [], [], []
    for b, (s, d) in enumerate(probs):
        tims = (rr.complete_tims if complete else rr.chain_tims)(s, d, cliques[b], float(sols[b]["scale"]))
        R.append(capi.rotation_from_solution_record(sols[b]))
        S.append(tims.x.T)
        D.append(tims.y.T)
        T.append(masks[b])
    if len(set(noise_bounds)) == 1:
        return ctx.certify_batch(R, S, D, T, noise_bound=noise_bounds[0], cbar2=1.0)
    return [ctx.certify_batch([R[b]], [S[b]], [D[b]], [T[b]], noise_bound=noise_bounds[b], cbar2=1.0)[0]
            for b in range(len(probs))]


def same(a, b):
    return (a["is_optimal"] == b["is_optimal"] and a["best_suboptimality"] == b["best_suboptimality"] and
            np.array_equal(a["suboptimality_traj"], b["suboptimality_traj"]))


@pytest.mark.parametrize("flags", [0, LOOP_EIG])
@pytest.mark.parametrize("complete", [0, 1])
def test_certify_known_scale_equals_host_batch(ctx, flags, complete):
    sizes = [40, 40, 36, 44, 40, 30, 40, 38, 42] if complete else [300, 260, 300, 340, 300, 280, 320, 300, 310]
    probs = [problem(n, 100 + i, 0.5 if complete else 0.9) for i, n in enumerate(sizes)]
    prm = params(rotation_tim_graph=complete)
    ctx.set_flags(flags)
    sols, cliques = ctx.solve_batch([p[0] for p in probs], [p[1] for p in probs], prm)
    masks = [ctx.last_inliers(b)[0] for b in range(len(probs))]
    got = ctx.certify_last(noise_bound=2 * NB, cbar2=1.0)
    assert all(sols["valid"]) and all(g["status"] == 0 for g in got)
    if complete:
        assert max(len(c) for c in cliques) <= 24  # N <= 276
    want = certify_host(ctx, probs, sols, cliques, masks, complete, [2 * NB] * len(probs))
    ctx.set_flags(0)
    for b in range(len(probs)):
        assert same(got[b], want[b]), b


def test_certify_unknown_scale(ctx):
    scales = [0.7, 1.0, 1.4, 1.9, 0.8, 1.2, 1.6, 0.9, 1.1]
    probs = [problem(300, 200 + i, 0.9, s) for i, s in enumerate(scales)]
    prm = params(estimate_scaling=1)
    sols, cliques = ctx.solve_batch([p[0] for p in probs], [p[1] for p in probs], prm)
    masks = [ctx.last_inliers(b)[0] for b in range(len(probs))]
    full = ctx.certify_last(noise_bound=2 * NB, cbar2=1.0)
    singles = [ctx.certify_last(problems=[b], noise_bound=2 * NB, cbar2=1.0)[0] for b in range(len(probs))]
    nbs = [2 * NB / float(sols[b]["scale"]) for b in range(len(probs))]
    want = certify_host(ctx, probs, sols, cliques, masks, 0, nbs)
    assert len({float(s["scale"]) for s in sols}) > 1
    for b in range(len(probs)):
        assert same(singles[b], want[b]), b
        assert full[b]["status"] == 0 and full[b]["is_optimal"] == singles[b]["is_optimal"], b
        assert _close(full[b]["suboptimality_traj"], singles[b]["suboptimality_traj"], TOL), b


def test_status_of_bad_entries(ctx):
    good = [problem(300, 300 + i) for i in range(9)]
    s_nan, d_nan = problem(60, 320)
    s_nan = s_nan.copy()
    s_nan[7, 1] = np.inf
    prm = params()
    # CHAIN batch: the good ones, an invalid solution
    probs = good + [no_clique(100)]
    ctx.solve_batch([p[0] for p in probs], [p[1] for p in probs], prm)
    ref = ctx.certify_last(problems=list(range(9)), noise_bound=2 * NB, cbar2=1.0)
    got = ctx.certify_last(noise_bound=2 * NB, cbar2=1.0)
    assert got[9]["status"] == capi.TZR_ERR_INVALID_ARG and got[9]["suboptimality_traj"].size == 0
    assert not got[9]["is_optimal"] and got[9]["best_suboptimality"] == np.inf
    for b in range(9):
        assert got[b]["status"] == 0 and _close(got[b]["suboptimality_traj"], ref[b]["suboptimality_traj"], TOL), b
    # duplicates and reordered entries
    order = [3, 0, 3, 9, 1]
    dup = ctx.certify_last(problems=order, noise_bound=2 * NB, cbar2=1.0)
    for j, b in enumerate(order):
        assert dup[j]["status"] == got[b]["status"], j
        assert _close(dup[j]["suboptimality_traj"], got[b]["suboptimality_traj"], TOL), j
    # NONE mode with a non-finite row: the gather flags it, the others are certified
    prm_none = params(inlier_selection_mode=3)
    probs = [problem(60, 330 + i, 0.0) for i in range(8)] + [(s_nan, d_nan)]
    ctx.solve_batch([p[0] for p in probs], [p[1] for p in probs], prm_none)
    ref = ctx.certify_last(problems=list(range(8)), noise_bound=2 * NB, cbar2=1.0)
    got = ctx.certify_last(noise_bound=2 * NB, cbar2=1.0)
    assert got[8]["status"] == capi.TZR_ERR_INVALID_ARG and got[8]["suboptimality_traj"].size == 0
    assert got[8]["best_suboptimality"] == np.inf and not got[8]["is_optimal"]
    for b in range(8):
        assert got[b]["status"] == 0 and _close(got[b]["suboptimality_traj"], ref[b]["suboptimality_traj"], TOL), b
    # COMPLETE: a clique above 128 points is too large; the call returns TZR_ERR_TOO_LARGE exactly then
    prm_c = params(rotation_tim_graph=1)
    probs = [problem(40, 340 + i, 0.5) for i in range(8)] + [problem(300, 350, 0.4)]
    sols, _ = ctx.solve_batch([p[0] for p in probs], [p[1] for p in probs], prm_c)
    assert sols[8]["clique_size"] > 128
    ref = ctx.certify_last(problems=list(range(8)), noise_bound=2 * NB, cbar2=1.0)
    got = ctx.certify_last(noise_bound=2 * NB, cbar2=1.0)
    assert got[8]["status"] == capi.TZR_ERR_TOO_LARGE and got[8]["best_suboptimality"] == np.inf
    for b in range(8):
        assert got[b]["status"] == 0 and _close(got[b]["suboptimality_traj"], ref[b]["suboptimality_traj"], TOL), b
    import ctypes as C
    res = (capi.CertificationResult * 9)()
    p = ctx.certifier_params(noise_bound=2 * NB)
    assert capi.lib().tzr_certify_last_solve(ctx._h, C.byref(p), 9, None, res, None, None, None) == capi.TZR_ERR_TOO_LARGE
    assert capi.lib().tzr_certify_last_solve(ctx._h, C.byref(p), 8, capi._p(np.arange(8, dtype=np.int32), C.c_int32),
                                             res, None, None, None) == capi.TZR_OK


def test_launches(ctx):
    probs = [problem(300, 400 + i) for i in range(9)]
    prm = params()
    sols, cliques = ctx.solve_batch([p[0] for p in probs], [p[1] for p in probs], prm)
    masks = [ctx.last_inliers(b)[0] for b in range(len(probs))]
    l0 = ctx.kernel_launches()
    ctx.certify_last(noise_bound=2 * NB, cbar2=1.0)
    l1 = ctx.kernel_launches()
    certify_host(ctx, probs, sols, cliques, masks, 0, [2 * NB] * len(probs))
    l2 = ctx.kernel_launches()
    assert l1 - l0 == (l2 - l1) + 1  # one group: one gather launch


def test_front_end_to_certified_ragged_solve(ctx):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(21)
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
    nb = 0.01
    prm = params(noise_bound=nb)
    keep = ragged_dev(ctx, probs, prm)
    got = ctx.certify_last(noise_bound=2 * nb, cbar2=1.0)
    del keep
    for b in range(B):
        assert got[b]["status"] == 0 and got[b]["is_optimal"], b


def test_certified_ragged_solve_matches_oracle(ctx):
    """One problem of a device-pointer ragged solve, certified from the workspace, against oracle/certifier_oracle.py
    on the host-built chain TIMs (the geometry of test_gpu_certifier.py's solve-then-certify test)."""
    prs = [synth.config_problem("C2", 1 + i, n=n) for i, n in enumerate([600, 450, 800])]
    probs = [(p["src"], p["dst"]) for p in prs]
    nb = prs[0]["noise_bound"]
    prm = params(noise_bound=nb)
    keep = ragged_dev(ctx, probs, prm)
    got = ctx.certify_last(problems=[0], noise_bound=2 * nb, cbar2=1.0)[0]
    sol = np.frombuffer(keep[2].cpu().numpy().tobytes(), dtype=capi.SOLUTION_DTYPE)
    rot0, _ = ctx.last_inliers(0)
    one = ctx.solve(*probs[0], prm)
    assert np.array_equal(one["rot_inliers"], rot0)
    tims = rr.chain_tims(probs[0][0], probs[0][1], one["clique"], float(sol[0]["scale"]))
    o = co.certify(one["R"], tims.x.T, tims.y.T, one["rot_inliers"], 2 * nb, 1.0)
    t = got["suboptimality_traj"]
    assert got["status"] == 0 and got["is_optimal"] == o["is_optimal"]
    assert len(t) == len(o["suboptimality_traj"])
    assert np.abs(t - o["suboptimality_traj"]).max() < 1e-6 * max(1.0, o["suboptimality_traj"].max())


def test_pybind_solve_and_certify_batch(ctx):
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    host = os.path.join(root, "teaser-plusplus_b200", "host")
    subprocess.check_call(["make", "-s", "-C", host])
    sys.path.insert(0, os.path.join(host, "python"))
    import teaserpp_python as tpp
    probs = [problem(n, 500 + i) for i, n in enumerate([300, 420, 300, 260])] + [no_clique(100)]
    solver = tpp.RobustRegistrationSolver(noise_bound=NB, estimate_scaling=False, rotation_cost_threshold=1e-12)
    cp = tpp.DRSCertifier.Params()
    cp.noise_bound = 2 * NB
    cp.cbar2 = 1.0
    out = solver.solve_and_certify_batch([p[0].T for p in probs], [p[1].T for p in probs], cp)
    prm = params()
    sols, cliques = ctx.solve_batch([p[0] for p in probs], [p[1] for p in probs], prm)
    masks = retained_masks(ctx, len(probs))
    want = ctx.certify_last(noise_bound=2 * NB, cbar2=1.0)
    for b, r in enumerate(out):
        assert r["solution"].valid == bool(sols[b]["valid"]), b
        assert np.array_equal(np.asarray(r["solution"].rotation), capi.rotation_from_solution_record(sols[b])), b
        assert np.array_equal(np.asarray(r["max_clique"]), cliques[b]), b
        assert np.array_equal(np.asarray(r["rotation_inliers_mask"]), masks[b][0]), b
        assert np.array_equal(np.asarray(r["translation_inliers_mask"]), masks[b][1]), b
        assert r["certified"] == (want[b]["status"] == 0), b
        c = r["certification"]
        assert c.is_optimal == want[b]["is_optimal"] and c.best_suboptimality == want[b]["best_suboptimality"], b
        assert np.array_equal(np.asarray(c.suboptimality_traj), want[b]["suboptimality_traj"]), b
