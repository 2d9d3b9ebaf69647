"""Generalized ICP on the device (run on an H100: `pytest -m gpu`).

Against the numpy restatement (tests/icp_generalized_reference.py) on scans with device normals, with NaN normals and
with a fixed scale other than 1; both nearest-neighbour routes bit for bit; a ragged batch against each problem alone;
the normals' sign and finiteness rules; a flat target, exact recovery and a far offset; the edge rules, the launch
count and the retained solve; the chained entry against the chain of public calls; the C++ and pybind façades; the
tutorial from raw scans refined by generalized ICP.
"""
import importlib
import os
import subprocess
import sys

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import icp_generalized_reference as ref
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


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.set_flags(0)
    c.close()


def _normals(ctx, *clouds):
    return [ctx.estimate_normals(c, RN) for c in clouds]


def run_ref(src, dst, sn, dn, init, **kw):
    return ref.icp(src, dst, sn, dn, R_CORR, s=init["scale"], R=np.asarray(init["rotation"]), t=init["translation"],
                   epsilon=kw.pop("epsilon", EPS), trace=True, **kw)


def _check_against_reference(ctx, src, dst, sn, dn, init, atol=1e-8, **kw):
    want = run_ref(src, dst, sn, dn, init, **kw)
    for m in want["margins"]:
        assert m["tie"] > 1e-9 and m["bound"] > 1e-9, m
    got, corr = ctx.icp_generalized(src, dst, sn, dn, R_CORR, init=init, epsilon=kw.get("epsilon", EPS))
    assert want["iterations"] > 1
    assert (got["iterations"], got["converged"], got["n_correspondences"]) == \
        (want["iterations"], want["converged"], want["n_correspondences"])
    assert got["fitness"] == want["fitness"] and got["scale"] == init["scale"]
    assert np.array_equal(corr, want["corr"])
    np.testing.assert_allclose(got["R"], want["R"], rtol=0, atol=atol)
    np.testing.assert_allclose(got["t"], want["t"], rtol=0, atol=atol)
    assert abs(got["inlier_rmse"] - want["inlier_rmse"]) <= 1e-9 * want["inlier_rmse"]
    return got


# ---- against the reference --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed,ns,nd,nan_share,epsilon", [(11, 1500, 1800, 0.0, EPS), (12, 3000, 2500, 0.1, EPS),
                                                          (13, 700, 900, 0.0, 0.05)])
def test_against_reference(ctx, seed, ns, nd, nan_share, epsilon):
    src, dst, R, t = scan_pair(seed, ns, nd)
    sn, dn = _normals(ctx, src, dst)
    if nan_share:
        rng = np.random.default_rng(seed)
        sn[rng.random(ns) < nan_share, :3] = np.nan
        dn[rng.random(nd) < nan_share, :3] = np.nan
    init = perturbed(R, t, seed)
    got = _check_against_reference(ctx, src, dst, sn, dn, init, epsilon=epsilon)
    # (n,3) normals are the same input
    got3, _ = ctx.icp_generalized(src, dst, sn[:, :3], dn[:, :3], R_CORR, init=init, epsilon=epsilon)
    assert all(np.array_equal(got[k], got3[k]) for k in got)


def test_fixed_scale_against_reference(ctx):
    """s = 0.8: the target shrunk about the scans' centre, so the source covariances enter as s^2 C(R m)."""
    src, dst, R, t = scan_pair(61, 1500, 1500)
    s = 0.8
    c = np.array([0.5, -0.2, 2.0])
    dst_s = (s * (dst.astype(np.float64) - c) + c).astype(np.float32)
    sn, dn = _normals(ctx, src, dst_s)
    init = dict(scale=s, rotation=Rotation.from_rotvec([0.01, -0.02, 0.015]).as_matrix() @ R,
                translation=s * t + (1 - s) * c + [0.01, 0.0, -0.01])
    _check_against_reference(ctx, src, dst_s, sn, dn, init)


def test_routes_bit_identical(ctx):
    src, dst, R, t = scan_pair(21, 3000, 3000)
    sn, dn = _normals(ctx, src, dst)
    init = perturbed(R, t, 21)
    run = lambda: ctx.icp_generalized_batch([src], [dst], [sn], [dn], R_CORR, [init])
    (ra, ca), (rb, cb) = with_flags(ctx, BRUTE, run), with_flags(ctx, GRID, run)
    assert as_bytes(ra) == as_bytes(rb) and np.array_equal(ca[0], cb[0])
    auto, _ = run()
    assert as_bytes(auto) == as_bytes(ra)
    assert ra[0]["iterations"] > 1 and ra[0]["n_correspondences"] > 1000


def test_batch_equals_single_forward_and_reverse(ctx):
    probs = []
    for k, (ns, nd) in enumerate([(300, 1000), (1000, 1023), (1500, 1024), (5000, 1200), (20001, 20000)]):
        src, dst, R, t = scan_pair(80 + k, ns, nd)
        probs.append((src, dst, *_normals(ctx, src, dst), perturbed(R, t, 80 + k, deg=2.0, shift=R_CORR)))
    src, dst, R, t = scan_pair(90, 600, 600)
    probs.append((src, dst, np.full((600, 4), np.nan, dtype=np.float32), _normals(ctx, dst)[0], perturbed(R, t, 90)))
    far_src, far_dst, _, _ = scan_pair(91, 300, 300)
    probs.append((far_src, far_dst + np.float32(50), *_normals(ctx, far_src, far_dst), None))
    singles = [ctx.icp_generalized_batch([s], [d], [a], [b], R_CORR, None if i is None else [i])
               for s, d, a, b, i in probs]
    for order in (list(range(len(probs))), list(reversed(range(len(probs))))):
        res, corr = ctx.icp_generalized_batch(*[[probs[k][f] for k in order] for f in range(4)], R_CORR,
                                              [probs[k][4] for k in order])
        for j, k in enumerate(order):
            assert as_bytes(res[j:j + 1]) == as_bytes(singles[k][0]), k
            assert np.array_equal(corr[j], singles[k][1][0]), k
    assert singles[4][0][0]["n_correspondences"] > 10000
    far = singles[-1][0][0]
    assert (far["n_correspondences"], far["iterations"], far["converged"]) == (0, 1, 1)


# ---- normals ----------------------------------------------------------------------------------------------------------
def test_normal_signs_do_not_matter(ctx):
    src, dst, R, t = scan_pair(23, 2000, 2000)
    sn, dn = _normals(ctx, src, dst)
    init = perturbed(R, t, 23)
    rng = np.random.default_rng(23)
    sf, df = sn.copy(), dn.copy()
    sf[rng.random(len(sf)) < 0.5, :3] *= -1
    df[rng.random(len(df)) < 0.5, :3] *= -1
    sf[:, 3], df[:, 3] = 7.0, -3.0  # the fourth float is ignored
    a = ctx.icp_generalized_batch([src], [dst], [sn], [dn], R_CORR, [init])
    b = ctx.icp_generalized_batch([src], [dst], [sf], [df], R_CORR, [init])
    assert as_bytes(a[0]) == as_bytes(b[0]) and np.array_equal(a[1][0], b[1][0])
    assert a[0][0]["iterations"] > 1
    # normals are used up to length: twice as long on one side is the same system up to rounding
    c, _ = ctx.icp_generalized(src, dst, sn, (dn.astype(np.float64) * 2).astype(np.float32), R_CORR, init=init)
    assert c["iterations"] == a[0][0]["iterations"]
    np.testing.assert_allclose(c["t"], a[0][0]["transform"]["translation"], atol=1e-9)


@pytest.mark.parametrize("side", ["source", "target"])
def test_nan_normals_count_but_do_not_move(ctx, side):
    """Every normal of one cloud NaN: its correspondences count for fitness and rmse, and every update is the identity,
    so the seed comes back after one iteration."""
    src, dst, R, t = scan_pair(92, 800, 800)
    sn, dn = _normals(ctx, src, dst)
    if side == "source":
        sn[:] = np.nan
    else:
        dn[:, :3] = 0.0  # zero length drops out as NaN does
        dn[::2, 0] = np.nan
    init = perturbed(R, t, 92, shift=0.3 * R_CORR)
    got, _ = ctx.icp_generalized(src, dst, sn, dn, R_CORR, init=init)
    want = ref.evaluate(src, dst, 1.0, np.asarray(init["rotation"]), np.asarray(init["translation"]), R_CORR ** 2)
    assert got["n_correspondences"] == want["count"] > 100 and got["fitness"] == want["fitness"]
    assert abs(got["inlier_rmse"] - want["rmse"]) <= 1e-12 * want["rmse"]
    assert got["iterations"] == 1 and got["converged"]
    assert np.array_equal(got["R"], np.asarray(init["rotation"])) and np.array_equal(got["t"], init["translation"])


# ---- geometry ---------------------------------------------------------------------------------------------------------
def test_flat_target_removes_both_offsets(ctx):
    """A flat grid target, the source offset in the plane and along its normal: generalized ICP removes both offsets,
    point-to-plane only the one along the normal."""
    g = np.arange(-1.0, 1.0, 0.02)
    X, Y = np.meshgrid(g, g)
    dst = np.stack([X.ravel(), Y.ravel(), np.zeros(X.size)], axis=1).astype(np.float32)
    nrm = np.tile(np.array([0, 0, 1, 0], dtype=np.float32), (len(dst), 1))
    src = (dst.astype(np.float64) + [0.003, 0.002, 0.01]).astype(np.float32)
    off = (src.astype(np.float64) - dst.astype(np.float64)).mean(axis=0)
    got, _ = ctx.icp_generalized(src, dst, nrm, nrm, R_CORR, max_iteration=10)
    assert got["n_correspondences"] == len(src) and got["converged"]
    np.testing.assert_allclose(got["t"], -off, rtol=0, atol=1e-7)
    np.testing.assert_allclose(got["R"], np.eye(3), rtol=0, atol=1e-7)
    pl, _ = ctx.icp_point_to_plane(src, dst, nrm, R_CORR, max_iteration=10)
    assert abs(pl["t"][2] + off[2]) < 1e-12
    assert abs(pl["t"][0]) < 1e-12 and abs(pl["t"][1]) < 1e-12  # the in-plane offset stays


def test_exact_recovery_at_the_origin(ctx):
    src, dst, nrm, R, t = _grid_surface((0.0, 0.0, 0.0))
    src_n = np.concatenate([nrm[:, :3].astype(np.float64) @ R, np.zeros((len(nrm), 1))], axis=1).astype(np.float32)
    init = perturbed(R, t, 7, deg=1.0, shift=0.4 * R_CORR, center=(0.0, 0.0, 0.0))
    got, _ = ctx.icp_generalized(src, dst, src_n, nrm, R_CORR, init=init, max_iteration=60, relative_fitness=0,
                                 relative_rmse=0)
    np.testing.assert_allclose(got["R"], R, rtol=0, atol=1e-9)
    np.testing.assert_allclose(got["t"], t, rtol=0, atol=1e-9)
    assert got["n_correspondences"] == len(src)


def test_large_offset_as_accurate_as_at_the_origin(ctx):
    """The ground-truth error at 1e5 is no worse than twice the error at the origin (or 0.05 degrees and 1e-3,
    whichever is larger).  Both runs use the device normals of the scans at the origin (the same surfaces, so the same
    normals): at 1e5 the float coordinates are rounded to 2^-7 ~ 0.008, and normals estimated there are that much
    noisier, which would measure the normal estimator rather than the step's arithmetic.  Measured on an H100 with
    normals estimated at 1e5 instead: 0.14 degrees against 0.03 at the origin."""
    errs = []
    src0, dst0, _, _ = scan_pair(71, 3000, 3000, offset=(0.0, 0.0, 0.0))
    sn, dn = _normals(ctx, src0, dst0)
    for off in ((0.0, 0.0, 0.0), (1e5, -1e5, 5e4)):
        src, dst, R, t = scan_pair(71, 3000, 3000, offset=off)
        init = perturbed(R, t, 71, deg=2.0, shift=R_CORR, center=off)
        got, _ = ctx.icp_generalized(src, dst, sn, dn, R_CORR, init=init)
        ang = np.degrees(Rotation.from_matrix(got["R"] @ R.T).magnitude())
        c = np.asarray(off)
        errs.append((ang, np.linalg.norm((got["R"] @ c + got["t"]) - (R @ c + t)), got["n_correspondences"]))
    (a0, t0, n0), (a1, t1, n1) = errs
    print(f"origin: {a0:.2e} deg {t0:.2e}; offset 1e5: {a1:.2e} deg {t1:.2e}")
    assert n0 > 1000 and n1 > 1000
    assert a1 <= max(2 * a0, 0.05) and t1 <= max(2 * t0, 1e-3), errs


# ---- edge rules -------------------------------------------------------------------------------------------------------
def test_max_iteration_zero_returns_the_seed(ctx):
    src, dst, R, t = scan_pair(51, 800, 800)
    sn, dn = _normals(ctx, src, dst)
    init = perturbed(R, t, 51, shift=0.2 * R_CORR)
    got, corr = ctx.icp_generalized(src, dst, sn, dn, R_CORR, init=init, max_iteration=0)
    p2p, corr2 = ctx.icp(src, dst, R_CORR, init=init, max_iteration=0)
    assert got["iterations"] == 0 and not got["converged"]
    assert np.array_equal(got["R"], np.asarray(init["rotation"])) and np.array_equal(got["t"], init["translation"])
    assert all(np.array_equal(got[k], p2p[k]) for k in got) and np.array_equal(corr, corr2) and len(corr) > 0


def test_launch_count_does_not_depend_on_B(ctx):
    src, dst, R, t = scan_pair(99, 2000, 2000)
    sn, dn = _normals(ctx, src, dst)
    counts = []
    for B in (1, 5):
        l0 = ctx.kernel_launches()
        ctx.icp_generalized_batch([src] * B, [dst] * B, [sn] * B, [dn] * B, R_CORR, [perturbed(R, t, 99)] * B,
                                  max_iteration=7)
        counts.append(ctx.kernel_launches() - l0)
    assert counts == [4 + 2 + 4 * 7] * 2
    l0 = ctx.kernel_launches()  # targets below 1024 points: no grid build
    ctx.icp_generalized_batch([src[:500]] * 3, [dst[:500]] * 3, [sn[:500]] * 3, [dn[:500]] * 3, R_CORR,
                              max_iteration=5)
    assert ctx.kernel_launches() - l0 == 2 + 4 * 5


def test_retained_solve_survives_a_generalized_call(ctx):
    rng = np.random.default_rng(3)
    src = rng.uniform(-1, 1, (120, 3))
    R = Rotation.from_rotvec([0.1, 0.2, -0.1]).as_matrix()
    dst = src @ R.T + [0.1, 0.0, 0.2]
    dst[:30] = rng.uniform(-1, 1, (30, 3))
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=0, rotation_cost_threshold=1e-12)
    ctx.solve(src, dst, prm)
    before = ctx.last_inliers(0)
    cert_before = ctx.certify_last(noise_bound=0.02)
    s, d, Rg, tg = scan_pair(97, 1500, 1500)
    sn, dn = ctx.estimate_normals_batch([s, d], RN)
    ctx.icp_generalized(s, d, sn, dn, R_CORR, init=perturbed(Rg, tg, 97))
    after = ctx.last_inliers(0)
    assert all(np.array_equal(a, b) for a, b in zip(before, after))
    cert_after = ctx.certify_last(noise_bound=0.02)
    assert cert_before[0]["best_suboptimality"] == cert_after[0]["best_suboptimality"]
    assert np.array_equal(cert_before[0]["suboptimality_traj"], cert_after[0]["suboptimality_traj"])


@pytest.mark.parametrize("case", ["null_src_normals", "null_dst_entry", "epsilon_zero", "epsilon_nan"])
def test_argument_checks_with_a_context(ctx, case):
    import test_icp_generalized_cpu as cpu
    p = capi.icp_params(0.1)
    kw = {"null_src_normals": dict(src_normals="null"), "null_dst_entry": dict(dst_normals="null_entry"),
          "epsilon_zero": dict(epsilon=0.0), "epsilon_nan": dict(epsilon=float("nan"))}[case]
    assert cpu._icp_batch(ctx._h, p, **kw) == capi.TZR_ERR_INVALID_ARG
    assert cpu._icp_batch(ctx._h, p) == 0


# ---- the chained entry ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("estimate_scaling", [0, 1])
def test_chained_entry_equals_the_chain(ctx, estimate_scaling):
    clouds = _sequence([600, 1500, 500, 700], seed=5)
    clouds.append((clouds[0] + np.float32(40.0)).astype(np.float32))
    clouds.append(clouds[2][:2].copy())
    pairs = [(0, 1), (1, 2), (2, 3), (3, 1), (1, 0), (0, 4), (5, 2)]
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=estimate_scaling, rotation_cost_threshold=1e-12)
    l0 = ctx.kernel_launches()
    plain = ctx.register_cloud_pairs(clouds, pairs, prm, **PAIR_FLAGS)
    l1 = ctx.kernel_launches()
    S = int((plain[2] >= 0).sum())
    ret_plain = _retained(ctx, S)
    l2 = ctx.kernel_launches()
    chained = ctx.register_cloud_pairs_icp(clouds, pairs, prm, R_CORR, max_iteration=40, method="generalized",
                                           epsilon=EPS, **PAIR_FLAGS)
    l3 = ctx.kernel_launches()
    stage = capi.SOLUTION_DTYPE.fields["stage_ms"][1]
    for a, b in zip(plain[0], chained[0]):
        assert a.tobytes()[:stage] == b.tobytes()[:stage]
    assert np.array_equal(plain[1], chained[1]) and np.array_equal(plain[2], chained[2])
    assert all(np.array_equal(a, b) for a, b in zip(plain[3], chained[3]))
    assert plain[5] == chained[5]
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
    want, _ = ctx.icp_generalized_batch([clouds[pairs[p][0]] for p in refined], [clouds[pairs[p][1]] for p in refined],
                                        [normals[pairs[p][0]] for p in refined], [normals[pairs[p][1]] for p in refined],
                                        R_CORR, seeds, epsilon=EPS, max_iteration=40)
    for k, p in enumerate(refined):
        assert icp_res[p].tobytes() == want[k].tobytes(), p
        assert icp_res[p]["iterations"] >= 1 and icp_res[p]["n_correspondences"] > 0
    # point-to-plane's chained entry refines the same pairs, differently
    pl = ctx.register_cloud_pairs_icp(clouds, pairs, prm, R_CORR, max_iteration=40, method="point_to_plane",
                                      **PAIR_FLAGS)[6]
    assert any(pl[p].tobytes() != icp_res[p].tobytes() for p in refined)
    assert (l3 - l2) - (l1 - l0) == 1 + 4 + 2 + 4 * 40
    with pytest.raises(capi.TzrError):
        ctx.register_cloud_pairs_icp(clouds, pairs, prm, R_CORR, method="generalized", epsilon=0.0, **PAIR_FLAGS)


# ---- façades ----------------------------------------------------------------------------------------------------------
def test_cpp_facade_equals_the_c_abi(tmp_path):
    """GeneralizedICP::refine / refineBatch and solveCloudPairsGeneralizedICP against the C-ABI
    (tests/cpp/icp_generalized_test.cc)."""
    subprocess.check_call(["make", "-s", "-C", HOST])
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    exe = str(tmp_path / "icp_generalized_test")
    subprocess.check_call([cxx, "-std=c++17", "-O1", "-I", os.path.join(HOST, "include"), "-I",
                           os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "icp_generalized_test.cc"),
                           "-L", HOST, "-lteaser_registration", "-L", CSRC, "-lteaser_b200",
                           f"-Wl,-rpath,{HOST}:{CSRC}", "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr


def test_pybind_generalized(ctx):
    subprocess.check_call(["make", "-s", "-C", HOST])
    sys.path.insert(0, os.path.join(HOST, "python"))
    import teaserpp_python as tpp
    src, dst, R, t = scan_pair(101, 1500, 1200)
    sn, dn = tpp.estimate_normals(src, RN), tpp.estimate_normals(dst, RN)
    init = perturbed(R, t, 101)
    seed = tpp.RegistrationSolution()
    seed.scale = 1.0
    seed.rotation = np.asarray(init["rotation"], dtype=np.float64)
    seed.translation = np.asarray(init["translation"], dtype=np.float64)
    icp = tpp.GeneralizedICP(R_CORR, max_iteration=30, epsilon=0.01)
    got = icp.refine(src, dst, sn, dn, seed)
    want, corr = ctx.icp_generalized(src, dst, sn, dn, R_CORR, init=init, epsilon=0.01)
    assert np.array_equal(np.asarray(got["solution"].rotation), want["R"])
    assert np.array_equal(np.asarray(got["solution"].translation).ravel(), want["t"])
    assert (got["fitness"], got["inlier_rmse"], got["iterations"], got["converged"]) == \
        (want["fitness"], want["inlier_rmse"], want["iterations"], want["converged"])
    assert np.array_equal(np.array(got["correspondences"], dtype=np.int32).reshape(-1, 2), corr)
    batch = icp.refine_batch([src, src], [dst, dst], [sn, sn[:, :3]], [dn, dn], [seed, seed])
    assert all(b["iterations"] == got["iterations"] and b["fitness"] == got["fitness"] for b in batch)
    clouds = _sequence([600, 700, 500], seed=9)
    pairs = [(0, 1), (1, 2)]
    solver = tpp.RobustRegistrationSolver(noise_bound=0.01, estimate_scaling=False, rotation_cost_threshold=1e-12)
    res = solver.solve_cloud_pairs_icp(clouds, pairs, R_CORR, normal_search_radius=PAIR_FLAGS["normal_search_radius"],
                                       fpfh_search_radius=PAIR_FLAGS["fpfh_search_radius"], use_absolute_scale=False,
                                       use_tuple_test=False, tuple_seed=0, method="generalized", epsilon=0.01)
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=0, rotation_cost_threshold=1e-12)
    c = ctx.register_cloud_pairs_icp(clouds, pairs, prm, R_CORR, method="generalized", epsilon=0.01, **PAIR_FLAGS)
    assert any(r["refined"] for r in res)
    for p, r in enumerate(res):
        assert r["refined"] == bool(c[1][p] == 0 and c[0][p]["valid"])
        if r["refined"]:
            d = capi.icp_result_dict(c[6][p])
            assert np.array_equal(np.asarray(r["icp"]["solution"].rotation), d["R"])
            assert r["icp"]["iterations"] == d["iterations"] and r["icp"]["fitness"] == d["fitness"]
    with pytest.raises(ValueError):
        solver.solve_cloud_pairs_icp(clouds, pairs, R_CORR, method="gicp")


# ---- the tutorial from raw scans, refined by generalized ICP -----------------------------------------------------------
def test_tutorial_from_raw_scans_generalized(ctx):
    from test_gpu_voxel import V, raw_pair
    pairs_gt = [raw_pair(20), raw_pair(21)]
    raw = [c for s, d, _, _ in pairs_gt for c in (s, d)]
    down = ctx.voxel_downsample_batch(raw, V)
    prm = capi.default_params(noise_bound=V, estimate_scaling=0, rotation_cost_threshold=1e-12)
    res = ctx.register_cloud_pairs_icp(down, [(0, 1), (2, 3)], prm, V, normal_search_radius=2 * V,
                                       fpfh_search_radius=5 * V, use_absolute_scale=False, use_crosscheck=True,
                                       use_tuple_test=False, method="generalized")
    sols, status, icp_res = res[0], res[1], res[6]
    for p, (src, _, R, t) in enumerate(pairs_gt):
        assert status[p] == 0 and sols[p]["valid"], p
        d = capi.icp_result_dict(icp_res[p])
        moved = src.astype(np.float64) @ d["R"].T + d["t"]
        truth = src.astype(np.float64) @ R.T + t
        err = np.linalg.norm(moved - truth, axis=1)
        rot_err = np.degrees(Rotation.from_matrix(d["R"] @ R.T).magnitude())
        print(f"pair {p}: mean displacement error {err.mean():.4f}, max {err.max():.4f}, rotation {rot_err:.3f} deg, "
              f"{d['iterations']} iterations")
        assert err.mean() < 0.004 and rot_err < 0.1, p
