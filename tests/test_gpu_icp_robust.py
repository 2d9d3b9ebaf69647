"""Robust kernels for point-to-plane and generalized ICP on the device (run on an H100: `pytest -m gpu`).

Every kernel type against the numpy restatement (tests/icp_robust_reference.py) for both methods and both search
routes, with s != 1, NaN and zero-length normals; L2 and a large-k Huber against the unweighted entries bit for bit; a
ragged batch against each problem alone; normal signs; L1 at exact recovery; Tukey with every residual beyond k; the
clutter fixture; the launch count and the retained solve; the chained entry against the chain of public calls; the C++
and pybind façades.
"""
import importlib
import os
import subprocess
import sys

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import icp_robust_reference as ref
from test_gpu_icp import PAIR_FLAGS, RN as PAIR_RN, _retained, _sequence, perturbed, scan_pair
from test_gpu_icp_plane import _grid_surface, as_bytes, with_flags

capi = importlib.import_module("teaser-plusplus_b200.capi")

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "teaser-plusplus_b200", "host")
CSRC = os.path.join(ROOT, "teaser-plusplus_b200", "csrc")
BRUTE, GRID = capi.FLAG_ICP_BRUTE_FORCE, capi.FLAG_ICP_GRID
R_CORR = 0.05
RN = 0.15  # normal radius on the test scans (about 25 neighbours)
EPS = 1e-3
L = ref.LOSSES
# k per method: point-to-plane residuals are distances; generalized ones are whitened (about 1 / sqrt(2 epsilon) ~ 22
# times a distance along the normals, about 0.7 times one across them)
KERNELS = {
    "plane": [("l2", 1.0), ("l1", 0.0), ("huber", 0.01), ("cauchy", 0.01), ("gm", 1e-4), ("tukey", 0.03)],
    "gicp": [("l2", 1.0), ("l1", 0.0), ("huber", 0.2), ("cauchy", 0.2), ("gm", 0.04), ("tukey", 0.6)],
}


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.set_flags(0)
    c.close()


def _normals(ctx, *clouds):
    return [ctx.estimate_normals(c, RN) for c in clouds]


def _run(ctx, method, src, dst, sn, dn, init, kernel, **kw):
    if method == "plane":
        return ctx.icp_point_to_plane(src, dst, dn, R_CORR, init=init, kernel=kernel, **kw)
    return ctx.icp_generalized(src, dst, sn, dn, R_CORR, init=init, kernel=kernel, epsilon=kw.pop("epsilon", EPS), **kw)


def _run_ref(method, src, dst, sn, dn, init, name, k, **kw):
    common = dict(s=init["scale"], R=np.asarray(init["rotation"]), t=init["translation"], trace=True)
    if method == "plane":
        return ref.icp_plane(src, dst, dn, R_CORR, L[name], k, **common, **kw)
    return ref.icp_gicp(src, dst, sn, dn, R_CORR, L[name], k, epsilon=kw.pop("epsilon", EPS), **common, **kw)


def _check_against_reference(ctx, method, src, dst, sn, dn, init, name, k, atol=1e-8, **kw):
    want = _run_ref(method, src, dst, sn, dn, init, name, k, **dict(kw))
    for m in want["margins"]:
        assert m["tie"] > 1e-9 and m["bound"] > 1e-9, m
    got, corr = _run(ctx, method, src, dst, sn, dn, init, (name, k), **dict(kw))
    assert want["iterations"] > 1
    assert (got["iterations"], got["converged"], got["n_correspondences"]) == \
        (want["iterations"], want["converged"], want["n_correspondences"])
    assert got["fitness"] == want["fitness"] and got["scale"] == init["scale"]
    assert np.array_equal(corr, want["corr"])
    np.testing.assert_allclose(got["R"], want["R"], rtol=0, atol=atol)
    np.testing.assert_allclose(got["t"], want["t"], rtol=0, atol=atol)
    assert abs(got["inlier_rmse"] - want["inlier_rmse"]) <= 1e-9 * want["inlier_rmse"]
    return got


def _case(ctx, seed, ns, nd, nan_share=0.0, zero_share=0.0):
    src, dst, R, t = scan_pair(seed, ns, nd)
    sn, dn = _normals(ctx, src, dst)
    rng = np.random.default_rng(seed)
    if nan_share:
        sn[rng.random(ns) < nan_share, :3] = np.nan
        dn[rng.random(nd) < nan_share, :3] = np.nan
    if zero_share:
        sn[rng.random(ns) < zero_share, :3] = 0.0
        dn[rng.random(nd) < zero_share, :3] = 0.0
    return src, dst, sn, dn, perturbed(R, t, seed, deg=1.0, shift=0.3 * R_CORR)


# ---- against the reference --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("method", ["plane", "gicp"])
@pytest.mark.parametrize("kk", range(6), ids=[n for n, _ in KERNELS["plane"]])
def test_every_kernel_against_reference(ctx, method, kk):
    name, k = KERNELS[method][kk]
    src, dst, sn, dn, init = _case(ctx, 11 + kk, 1500, 1800, nan_share=0.05, zero_share=0.03)
    got = _check_against_reference(ctx, method, src, dst, sn, dn, init, name, k)
    # both search routes give the same bits
    run = lambda: _run(ctx, method, src, dst, sn, dn, init, (name, k))  # noqa: E731
    (ra, ca), (rb, cb) = with_flags(ctx, BRUTE, run), with_flags(ctx, GRID, run)
    assert all(np.array_equal(ra[f], rb[f]) and np.array_equal(ra[f], got[f]) for f in got)
    assert np.array_equal(ca, cb)


@pytest.mark.parametrize("method,name", [("plane", "tukey"), ("gicp", "tukey"), ("gicp", "cauchy")])
def test_fixed_scale_against_reference(ctx, method, name):
    """s = 0.8: the target shrunk about the scans' centre."""
    src, dst, R, t = scan_pair(61, 1500, 1500)
    s = 0.8
    c = np.array([0.5, -0.2, 2.0])
    dst_s = (s * (dst.astype(np.float64) - c) + c).astype(np.float32)
    sn, dn = _normals(ctx, src, dst_s)
    init = dict(scale=s, rotation=Rotation.from_rotvec([0.01, -0.02, 0.015]).as_matrix() @ R,
                translation=s * t + (1 - s) * c + [0.01, 0.0, -0.01])
    k = dict(KERNELS[method])[name]
    _check_against_reference(ctx, method, src, dst_s, sn, dn, init, name, k)


# ---- against the unweighted entries -----------------------------------------------------------------------------------
@pytest.mark.parametrize("method", ["plane", "gicp"])
def test_l2_bit_identical_to_the_unweighted_entries(ctx, method):
    src, dst, sn, dn, init = _case(ctx, 31, 3000, 2500, nan_share=0.05)
    kernels = [("l2", 0.0), capi.RobustKernel(0, 0, float("nan"))]  # k is not read for L2
    if method == "plane":
        kernels.append(("huber", 1e6))  # w = k / max(e, k) = 1 exactly: the same products
    plain = (ctx.icp_point_to_plane_batch([src], [dst], [dn], R_CORR, [init]) if method == "plane" else
             ctx.icp_generalized_batch([src], [dst], [sn], [dn], R_CORR, [init]))
    assert plain[0][0]["iterations"] > 1
    for kern in kernels:
        got = (ctx.icp_point_to_plane_batch([src], [dst], [dn], R_CORR, [init], kernel=kern) if method == "plane" else
               ctx.icp_generalized_batch([src], [dst], [sn], [dn], R_CORR, [init], kernel=kern))
        assert as_bytes(got[0]) == as_bytes(plain[0]) and np.array_equal(got[1][0], plain[1][0]), kern


@pytest.mark.parametrize("method", ["plane", "gicp"])
def test_batch_equals_single_forward_and_reverse(ctx, method):
    name, k = ("tukey", dict(KERNELS[method])["tukey"])
    probs = []
    for j, (ns, nd) in enumerate([(300, 1000), (1000, 1023), (1500, 1024), (5000, 1200), (20001, 20000)]):
        src, dst, R, t = scan_pair(80 + j, ns, nd)
        probs.append((src, dst, *_normals(ctx, src, dst), perturbed(R, t, 80 + j, deg=1.0, shift=0.3 * R_CORR)))
    src, dst, R, t = scan_pair(90, 600, 600)
    probs.append((src, dst, np.full((600, 4), np.nan, dtype=np.float32), _normals(ctx, dst)[0], perturbed(R, t, 90)))
    far_src, far_dst, _, _ = scan_pair(91, 300, 300)
    probs.append((far_src, far_dst + np.float32(50), *_normals(ctx, far_src, far_dst), None))

    def call(ps):
        inits = [p[4] for p in ps]
        if method == "plane":
            return ctx.icp_point_to_plane_batch([p[0] for p in ps], [p[1] for p in ps], [p[3] for p in ps], R_CORR,
                                                inits, kernel=(name, k))
        return ctx.icp_generalized_batch([p[0] for p in ps], [p[1] for p in ps], [p[2] for p in ps],
                                         [p[3] for p in ps], R_CORR, inits, kernel=(name, k))

    singles = [call([p]) for p in probs]
    for order in (list(range(len(probs))), list(reversed(range(len(probs))))):
        res, corr = call([probs[j] for j in order])
        for i, j in enumerate(order):
            assert as_bytes(res[i:i + 1]) == as_bytes(singles[j][0]), j
            assert np.array_equal(corr[i], singles[j][1][0]), j
    assert singles[4][0][0]["n_correspondences"] > 10000 and singles[4][0][0]["iterations"] > 1
    far = singles[-1][0][0]
    assert (far["n_correspondences"], far["iterations"], far["converged"]) == (0, 1, 1)


# ---- normals and edge rules -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("method,name", [("plane", "cauchy"), ("gicp", "tukey"), ("gicp", "l1")])
def test_normal_signs_do_not_matter(ctx, method, name):
    src, dst, sn, dn, init = _case(ctx, 23, 2000, 2000)
    rng = np.random.default_rng(23)
    sf, df = sn.copy(), dn.copy()
    sf[rng.random(len(sf)) < 0.5, :3] *= -1
    df[rng.random(len(df)) < 0.5, :3] *= -1
    sf[:, 3], df[:, 3] = 7.0, -3.0  # the fourth float is ignored
    kern = (name, dict(KERNELS[method])[name])
    a = _run(ctx, method, src, dst, sn, dn, init, kern)
    b = _run(ctx, method, src, dst, sf, df, init, kern)
    assert all(np.array_equal(a[0][f], b[0][f]) for f in a[0]) and np.array_equal(a[1], b[1])
    assert a[0]["iterations"] > 1


@pytest.mark.parametrize("method", ["plane", "gicp"])
def test_l1_at_exact_recovery_stays_finite(ctx, method):
    """The loop reaches zero residuals, where L1's weight is infinite: those correspondences leave the system and every
    output stays finite."""
    src, dst, nrm, R, t = _grid_surface((0.0, 0.0, 0.0))
    src_n = np.concatenate([nrm[:, :3].astype(np.float64) @ R, np.zeros((len(nrm), 1))], axis=1).astype(np.float32)
    init = perturbed(R, t, 7, deg=0.5, shift=0.2 * R_CORR, center=(0.0, 0.0, 0.0))
    got, _ = _run(ctx, method, src, dst, src_n, nrm, init, "l1", max_iteration=60, relative_fitness=0, relative_rmse=0)
    assert np.isfinite(got["R"]).all() and np.isfinite(got["t"]).all() and np.isfinite(got["inlier_rmse"])
    np.testing.assert_allclose(got["R"], R, rtol=0, atol=1e-6)
    np.testing.assert_allclose(got["t"], t, rtol=0, atol=1e-6)
    assert got["n_correspondences"] == len(src) and got["inlier_rmse"] < 1e-6


@pytest.mark.parametrize("method", ["plane", "gicp"])
def test_tukey_with_every_residual_beyond_k_gives_identity_updates(ctx, method):
    src, dst, sn, dn, init = _case(ctx, 92, 800, 800)
    got, _ = _run(ctx, method, src, dst, sn, dn, init, ("tukey", 1e-12))
    want = ref.evaluate(src, dst, 1.0, np.asarray(init["rotation"]), np.asarray(init["translation"]), R_CORR ** 2)
    assert got["n_correspondences"] == want["count"] > 100 and got["fitness"] == want["fitness"]
    assert got["iterations"] == 1 and got["converged"]
    assert np.array_equal(got["R"], np.asarray(init["rotation"])) and np.array_equal(got["t"], init["translation"])


@pytest.mark.parametrize("method", ["plane", "gicp"])
def test_clutter_fixture(ctx, method):
    """A parallel sheet 0.04 off the surface replaces a third of the overlap: Tukey lands at least 10x closer to the
    truth than L2 (tests/test_icp_robust_reference_cpu.py establishes the same on the reference)."""
    f = ref.clutter_pair(0)
    init = dict(scale=1.0, rotation=f["R0"], translation=f["t0"])
    k = f["k_plane"] if method == "plane" else f["k_gicp"]
    if method == "plane":
        l2, _ = ctx.icp_point_to_plane(f["src"], f["dst"], f["dst_normals"], f["r"], init=init)
        tk, _ = ctx.icp_point_to_plane(f["src"], f["dst"], f["dst_normals"], f["r"], init=init, kernel=("tukey", k))
    else:
        l2, _ = ctx.icp_generalized(f["src"], f["dst"], f["src_normals"], f["dst_normals"], f["r"], init=init)
        tk, _ = ctx.icp_generalized(f["src"], f["dst"], f["src_normals"], f["dst_normals"], f["r"], init=init,
                                    kernel=("tukey", k))
    e_l2 = ref.pose_error(l2["R"], l2["t"], f["R"], f["t"])
    e_tk = ref.pose_error(tk["R"], tk["t"], f["R"], f["t"])
    print(f"{method}: L2 {e_l2:.3e}, Tukey {e_tk:.3e}")
    assert e_tk * 10 <= e_l2


def test_launch_count_does_not_depend_on_B(ctx):
    src, dst, sn, dn, init = _case(ctx, 99, 2000, 2000)
    for method in ("plane", "gicp"):
        counts = []
        for B in (1, 5):
            l0 = ctx.kernel_launches()
            if method == "plane":
                ctx.icp_point_to_plane_batch([src] * B, [dst] * B, [dn] * B, R_CORR, [init] * B, max_iteration=7,
                                             kernel=("tukey", 0.03))
            else:
                ctx.icp_generalized_batch([src] * B, [dst] * B, [sn] * B, [dn] * B, R_CORR, [init] * B,
                                          max_iteration=7, kernel=("tukey", 0.6))
            counts.append(ctx.kernel_launches() - l0)
        assert counts == [4 + 2 + 4 * 7] * 2, method


def test_retained_solve_survives_a_robust_call(ctx):
    rng = np.random.default_rng(3)
    src = rng.uniform(-1, 1, (120, 3))
    R = Rotation.from_rotvec([0.1, 0.2, -0.1]).as_matrix()
    dst = src @ R.T + [0.1, 0.0, 0.2]
    dst[:30] = rng.uniform(-1, 1, (30, 3))
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=0, rotation_cost_threshold=1e-12)
    ctx.solve(src, dst, prm)
    before = ctx.last_inliers(0)
    cert_before = ctx.certify_last(noise_bound=0.02)
    s, d, sn, dn, init = _case(ctx, 97, 1500, 1500)
    ctx.icp_point_to_plane(s, d, dn, R_CORR, init=init, kernel=("huber", 0.01))
    ctx.icp_generalized(s, d, sn, dn, R_CORR, init=init, kernel=("tukey", 0.6))
    after = ctx.last_inliers(0)
    assert all(np.array_equal(a, b) for a, b in zip(before, after))
    cert_after = ctx.certify_last(noise_bound=0.02)
    assert cert_before[0]["best_suboptimality"] == cert_after[0]["best_suboptimality"]


@pytest.mark.parametrize("kernel", [capi.RobustKernel(9, 0, 1.0), capi.RobustKernel(5, 0, 0.0),
                                    capi.RobustKernel(3, 0, float("nan"))])
def test_bad_kernels_with_a_context_launch_nothing(ctx, kernel):
    src, dst, sn, dn, init = _case(ctx, 98, 500, 500)
    l0 = ctx.kernel_launches()
    with pytest.raises(capi.TzrError):
        ctx.icp_point_to_plane(src, dst, dn, R_CORR, init=init, kernel=kernel)
    with pytest.raises(capi.TzrError):
        ctx.icp_generalized(src, dst, sn, dn, R_CORR, init=init, kernel=kernel)
    assert ctx.kernel_launches() == l0


# ---- the chained entry ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("method,name,k", [("point_to_plane", "tukey", 0.03), ("generalized", "cauchy", 0.2)])
def test_chained_entry_equals_the_chain(ctx, method, name, k):
    clouds = _sequence([600, 1500, 500, 700], seed=5)
    clouds.append((clouds[0] + np.float32(40.0)).astype(np.float32))
    clouds.append(clouds[2][:2].copy())
    pairs = [(0, 1), (1, 2), (2, 3), (3, 1), (1, 0), (0, 4), (5, 2)]
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=0, rotation_cost_threshold=1e-12)
    l0 = ctx.kernel_launches()
    plain = ctx.register_cloud_pairs(clouds, pairs, prm, **PAIR_FLAGS)
    l1 = ctx.kernel_launches()
    S = int((plain[2] >= 0).sum())
    ret_plain = _retained(ctx, S)
    l2 = ctx.kernel_launches()
    chained = ctx.register_cloud_pairs_icp(clouds, pairs, prm, R_CORR, max_iteration=40, method=method, epsilon=EPS,
                                           kernel=(name, k), **PAIR_FLAGS)
    l3 = ctx.kernel_launches()
    stage = capi.SOLUTION_DTYPE.fields["stage_ms"][1]
    for a, b in zip(plain[0], chained[0]):
        assert a.tobytes()[:stage] == b.tobytes()[:stage]
    assert np.array_equal(plain[1], chained[1]) and np.array_equal(plain[2], chained[2])
    assert _retained(ctx, S) == ret_plain
    icp_res = chained[6]
    refined = [p for p in range(len(pairs)) if plain[1][p] == 0 and plain[0][p]["valid"]]
    assert len(refined) >= 3
    for p in range(len(pairs)):
        if p not in refined:
            assert not icp_res[p].tobytes().strip(b"\0"), p
    normals = ctx.estimate_normals_batch(clouds, PAIR_RN)
    seeds = [dict(scale=plain[0][p]["scale"], rotation=plain[0][p]["rotation"], translation=plain[0][p]["translation"])
             for p in refined]
    S_, D_ = [clouds[pairs[p][0]] for p in refined], [clouds[pairs[p][1]] for p in refined]
    DN = [normals[pairs[p][1]] for p in refined]
    if method == "point_to_plane":
        want, _ = ctx.icp_point_to_plane_batch(S_, D_, DN, R_CORR, seeds, max_iteration=40, kernel=(name, k))
    else:
        want, _ = ctx.icp_generalized_batch(S_, D_, [normals[pairs[p][0]] for p in refined], DN, R_CORR, seeds,
                                            epsilon=EPS, max_iteration=40, kernel=(name, k))
    for j, p in enumerate(refined):
        assert icp_res[p].tobytes() == want[j].tobytes(), p
        assert icp_res[p]["iterations"] >= 1 and icp_res[p]["n_correspondences"] > 0
    # with L2 the chained robust entry is the unweighted chained entry
    unweighted = ctx.register_cloud_pairs_icp(clouds, pairs, prm, R_CORR, max_iteration=40, method=method,
                                              epsilon=EPS, **PAIR_FLAGS)[6]
    l2k = ctx.register_cloud_pairs_icp(clouds, pairs, prm, R_CORR, max_iteration=40, method=method, epsilon=EPS,
                                       kernel="l2", **PAIR_FLAGS)[6]
    assert unweighted.tobytes() == l2k.tobytes()
    assert any(unweighted[p].tobytes() != icp_res[p].tobytes() for p in refined)
    assert (l3 - l2) - (l1 - l0) == 1 + 4 + 2 + 4 * 40


# ---- façades ----------------------------------------------------------------------------------------------------------
def test_cpp_facade_equals_the_c_abi(tmp_path):
    """PointToPlaneICP / GeneralizedICP with a RobustKernel and the robust solveCloudPairs overloads against the C-ABI
    (tests/cpp/icp_robust_test.cc)."""
    subprocess.check_call(["make", "-s", "-C", HOST])
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    exe = str(tmp_path / "icp_robust_test")
    subprocess.check_call([cxx, "-std=c++17", "-O1", "-I", os.path.join(HOST, "include"), "-I",
                           os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "icp_robust_test.cc"),
                           "-L", HOST, "-lteaser_registration", "-L", CSRC, "-lteaser_b200",
                           f"-Wl,-rpath,{HOST}:{CSRC}", "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr


def test_pybind_robust(ctx):
    subprocess.check_call(["make", "-s", "-C", HOST])
    sys.path.insert(0, os.path.join(HOST, "python"))
    import teaserpp_python as tpp
    src, dst, R, t = scan_pair(101, 1500, 1200)
    sn, dn = tpp.estimate_normals(src, RN), tpp.estimate_normals(dst, RN)
    init = perturbed(R, t, 101, deg=1.0, shift=0.3 * R_CORR)
    seed = tpp.RegistrationSolution()
    seed.scale = 1.0
    seed.rotation = np.asarray(init["rotation"], dtype=np.float64)
    seed.translation = np.asarray(init["translation"], dtype=np.float64)
    kt = tpp.RobustKernel("tukey", 0.03)
    assert kt.type == tpp.RobustKernel.Type.TUKEY and kt.k == 0.03
    pl = tpp.PointToPlaneICP(R_CORR, max_iteration=30, kernel=kt)
    got = pl.refine(src, dst, dn, seed)
    want, corr = ctx.icp_point_to_plane(src, dst, dn, R_CORR, init=init, kernel=("tukey", 0.03))
    assert np.array_equal(np.asarray(got["solution"].rotation), want["R"])
    assert np.array_equal(np.asarray(got["solution"].translation).ravel(), want["t"])
    assert (got["fitness"], got["inlier_rmse"], got["iterations"]) == \
        (want["fitness"], want["inlier_rmse"], want["iterations"])
    assert np.array_equal(np.array(got["correspondences"], dtype=np.int32).reshape(-1, 2), corr)
    gi = tpp.GeneralizedICP(R_CORR, max_iteration=30, epsilon=0.01,
                            kernel=tpp.RobustKernel(tpp.RobustKernel.Type.CAUCHY, 0.2))
    got = gi.refine(src, dst, sn, dn, seed)
    want, _ = ctx.icp_generalized(src, dst, sn, dn, R_CORR, init=init, epsilon=0.01, kernel=("cauchy", 0.2))
    assert np.array_equal(np.asarray(got["solution"].rotation), want["R"]) and got["iterations"] == want["iterations"]
    clouds = _sequence([600, 700, 500], seed=9)
    pairs = [(0, 1), (1, 2)]
    solver = tpp.RobustRegistrationSolver(noise_bound=0.01, estimate_scaling=False, rotation_cost_threshold=1e-12)
    res = solver.solve_cloud_pairs_icp(clouds, pairs, R_CORR, normal_search_radius=PAIR_FLAGS["normal_search_radius"],
                                       fpfh_search_radius=PAIR_FLAGS["fpfh_search_radius"], use_absolute_scale=False,
                                       use_tuple_test=False, tuple_seed=0, method="generalized", epsilon=0.01,
                                       kernel=tpp.RobustKernel("tukey", 0.6))
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=0, rotation_cost_threshold=1e-12)
    c = ctx.register_cloud_pairs_icp(clouds, pairs, prm, R_CORR, method="generalized", epsilon=0.01,
                                     kernel=("tukey", 0.6), **PAIR_FLAGS)
    assert any(r["refined"] for r in res)
    for p, r in enumerate(res):
        if r["refined"]:
            d = capi.icp_result_dict(c[6][p])
            assert np.array_equal(np.asarray(r["icp"]["solution"].rotation), d["R"])
            assert r["icp"]["iterations"] == d["iterations"] and r["icp"]["fitness"] == d["fitness"]
    with pytest.raises(ValueError):
        solver.solve_cloud_pairs_icp(clouds, pairs, R_CORR, method="point_to_point", kernel=tpp.RobustKernel("l1"))
