"""tzr_estimate_normals(_batch) and point-to-plane ICP on the device (run on an H100: `pytest -m gpu`).

Normals against compute_fpfh's, bit for bit, on every route; point-to-plane ICP against the numpy restatement
(tests/icp_plane_reference.py) on scans with device normals; both nearest-neighbour routes bit for bit; a ragged batch
against each problem alone; the normals' sign and finiteness rules; a flat target, exact recovery and a far offset; the
edge rules, the launch count and the retained solve; the chained entry against the chain of public calls; the C++ and
pybind façades; the tutorial from raw scans with point-to-plane refinement.
"""
import importlib
import os
import subprocess
import sys

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import icp_plane_reference as ref
from test_gpu_icp import PAIR_FLAGS, RN as PAIR_RN, _retained, _sequence, perturbed, scan_pair, surface

capi = importlib.import_module("teaser-plusplus_b200.capi")

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "teaser-plusplus_b200", "host")
CSRC = os.path.join(ROOT, "teaser-plusplus_b200", "csrc")
BRUTE, GRID = capi.FLAG_ICP_BRUTE_FORCE, capi.FLAG_ICP_GRID
R_CORR = 0.05
RN = 0.15  # normal radius on the test scans (about 25 neighbours)


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.set_flags(0)
    c.close()


def as_bytes(res):
    return np.ascontiguousarray(res).tobytes()


def with_flags(ctx, flags, fn):
    ctx.set_flags(flags)
    try:
        return fn()
    finally:
        ctx.set_flags(0)


# ---- normals ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [700, 6000])
def test_normals_equal_compute_fpfh_on_every_route(ctx, n):
    pts = surface(np.random.default_rng(n), n).astype(np.float32)
    want = None
    for flags in (0, capi.FLAG_FPFH_BRUTE_FORCE, capi.FLAG_FPFH_GRID):
        _, nf = with_flags(ctx, flags, lambda: ctx.compute_fpfh(pts, RN, 2 * RN, return_normals=True))
        got = with_flags(ctx, flags, lambda: ctx.estimate_normals(pts, RN))
        assert got.tobytes() == nf.tobytes(), flags
        want = got if want is None else want
        assert got.tobytes() == want.tobytes(), flags  # and every route the same bits
    assert np.isfinite(want).all(axis=1).mean() > 0.95  # a few isolated points have fewer than 3 neighbours


def test_normals_batch_equals_single_and_overflow_fails_alone(ctx):
    rng = np.random.default_rng(3)
    clouds = [surface(rng, k).astype(np.float32) for k in (50, 1500, 5000, 2)]
    dense = np.zeros((4200, 3), dtype=np.float32)  # 4200 coincident points: 4199 neighbours each
    singles = [ctx.estimate_normals(c, RN) for c in clouds]
    for order in ([0, 1, 2, 3], [3, 2, 1, 0]):
        got = ctx.estimate_normals_batch([clouds[k] for k in order], RN)
        for j, k in enumerate(order):
            assert got[j].tobytes() == singles[k].tobytes(), k
    assert np.isnan(singles[3]).all()  # fewer than 3 neighbours
    with pytest.raises(capi.TzrError) as e:
        ctx.estimate_normals_batch([clouds[1], dense, clouds[0]], RN)
    assert e.value.status.tolist() == [0, capi.TZR_ERR_TOO_LARGE, 0]
    assert e.value.result[0].tobytes() == singles[1].tobytes()
    assert e.value.result[2].tobytes() == singles[0].tobytes()
    with pytest.raises(capi.TzrError):
        ctx.estimate_normals(dense, RN)
    # the descriptor batch agrees
    _, nf = ctx.compute_fpfh_batch(clouds, RN, 2 * RN, return_normals=True)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(nf, singles))


# ---- point-to-plane ICP against the reference -------------------------------------------------------------------------
def run_ref(src, dst, nrm, init, **kw):
    return ref.icp(src, dst, nrm, R_CORR, s=init["scale"], R=np.asarray(init["rotation"]), t=init["translation"],
                   trace=True, **kw)


@pytest.mark.parametrize("seed,ns,nd,nan_share", [(11, 1500, 1800, 0.0), (12, 3000, 2500, 0.1), (13, 700, 900, 0.0)])
def test_against_reference(ctx, seed, ns, nd, nan_share):
    src, dst, R, t = scan_pair(seed, ns, nd)
    nrm = ctx.estimate_normals(dst, RN)
    if nan_share:
        nrm[np.random.default_rng(seed).random(nd) < nan_share, :3] = np.nan
    init = perturbed(R, t, seed)
    want = run_ref(src, dst, nrm, init)
    for m in want["margins"]:
        assert m["tie"] > 1e-9 and m["bound"] > 1e-9, m
    got, corr = ctx.icp_point_to_plane(src, dst, nrm, R_CORR, init=init)
    assert want["iterations"] > 1
    assert (got["iterations"], got["converged"], got["n_correspondences"]) == \
        (want["iterations"], want["converged"], want["n_correspondences"])
    assert got["fitness"] == want["fitness"]
    assert np.array_equal(corr, want["corr"])
    np.testing.assert_allclose(got["R"], want["R"], rtol=0, atol=1e-8)
    np.testing.assert_allclose(got["t"], want["t"], rtol=0, atol=1e-8)
    assert abs(got["inlier_rmse"] - want["inlier_rmse"]) <= 1e-9 * want["inlier_rmse"]
    # (nd,3) normals are the same input
    got3, _ = ctx.icp_point_to_plane(src, dst, nrm[:, :3], R_CORR, init=init)
    assert all(np.array_equal(got[k], got3[k]) for k in got)


def test_routes_bit_identical(ctx):
    src, dst, R, t = scan_pair(21, 3000, 3000)
    nrm = ctx.estimate_normals(dst, RN)
    init = perturbed(R, t, 21)
    run = lambda: ctx.icp_point_to_plane_batch([src], [dst], [nrm], R_CORR, [init])
    (ra, ca), (rb, cb) = with_flags(ctx, BRUTE, run), with_flags(ctx, GRID, run)
    assert as_bytes(ra) == as_bytes(rb) and np.array_equal(ca[0], cb[0])
    auto, _ = run()
    assert as_bytes(auto) == as_bytes(ra)
    assert ra[0]["iterations"] > 1 and ra[0]["n_correspondences"] > 1000


def _ragged_problems(ctx):
    probs = []
    for k, (ns, nd) in enumerate([(300, 1000), (1000, 1023), (1500, 1024), (5000, 1200), (20001, 20000)]):
        src, dst, R, t = scan_pair(80 + k, ns, nd)
        probs.append((src, dst, ctx.estimate_normals(dst, RN), perturbed(R, t, 80 + k, deg=2.0, shift=R_CORR)))
    src, dst, R, t = scan_pair(90, 600, 600)
    probs.append((src, dst, np.full((600, 4), np.nan, dtype=np.float32), perturbed(R, t, 90)))
    far_src, far_dst, _, _ = scan_pair(91, 300, 300)
    probs.append((far_src, far_dst + np.float32(50), ctx.estimate_normals(far_dst, RN), None))
    return probs


def test_batch_equals_single_forward_and_reverse(ctx):
    probs = _ragged_problems(ctx)
    singles = [ctx.icp_point_to_plane_batch([s], [d], [n], R_CORR, None if i is None else [i]) for s, d, n, i in probs]
    for order in (list(range(len(probs))), list(reversed(range(len(probs))))):
        res, corr = ctx.icp_point_to_plane_batch([probs[k][0] for k in order], [probs[k][1] for k in order],
                                                 [probs[k][2] for k in order], R_CORR, [probs[k][3] for k in order])
        for j, k in enumerate(order):
            assert as_bytes(res[j:j + 1]) == as_bytes(singles[k][0]), k
            assert np.array_equal(corr[j], singles[k][1][0]), k
    assert singles[4][0][0]["n_correspondences"] > 10000
    far = singles[-1][0][0]
    assert (far["n_correspondences"], far["iterations"], far["converged"]) == (0, 1, 1)


def test_all_nan_normals_count_but_do_not_move(ctx):
    """A problem whose normals are all NaN: its correspondences count for fitness and rmse, and every update is the
    identity, so the seed comes back after one iteration."""
    src, dst, _, _, nrm, init = _nan_problem()
    got, corr = ctx.icp_point_to_plane(src, dst, nrm, R_CORR, init=init)
    want = ref.evaluate(src, dst, 1.0, np.asarray(init["rotation"]), np.asarray(init["translation"]), R_CORR ** 2)
    assert got["n_correspondences"] == want["count"] > 100 and got["fitness"] == want["fitness"]
    assert abs(got["inlier_rmse"] - want["rmse"]) <= 1e-12 * want["rmse"]
    assert got["iterations"] == 1 and got["converged"]
    assert np.array_equal(got["R"], np.asarray(init["rotation"])) and np.array_equal(got["t"], init["translation"])


def _nan_problem():
    src, dst, R, t = scan_pair(92, 800, 800)
    return src, dst, R, t, np.full((800, 4), np.nan, dtype=np.float32), perturbed(R, t, 92, shift=0.3 * R_CORR)


def test_normal_signs_do_not_matter(ctx):
    src, dst, R, t = scan_pair(23, 2000, 2000)
    nrm = ctx.estimate_normals(dst, RN)
    init = perturbed(R, t, 23)
    flipped = nrm.copy()
    flip = np.random.default_rng(23).random(len(nrm)) < 0.5
    flipped[flip, :3] *= -1
    flipped[~flip, 3] = 7.0  # the fourth float is ignored too
    a = ctx.icp_point_to_plane_batch([src], [dst], [nrm], R_CORR, [init])
    b = ctx.icp_point_to_plane_batch([src], [dst], [flipped], R_CORR, [init])
    assert as_bytes(a[0]) == as_bytes(b[0]) and np.array_equal(a[1][0], b[1][0])
    assert a[0][0]["iterations"] > 1


def test_partial_nan_normals_add_nothing(ctx):
    """A third of the normals NaN: the device agrees with the reference, which leaves those correspondences out of
    the system and keeps them in the evaluation."""
    src, dst, R, t = scan_pair(24, 1500, 1500)
    nrm = ctx.estimate_normals(dst, RN)
    nrm[::3, :3] = np.nan
    init = perturbed(R, t, 24)
    got, corr = ctx.icp_point_to_plane(src, dst, nrm, R_CORR, init=init)
    want = run_ref(src, dst, nrm, init)
    assert got["iterations"] == want["iterations"] and np.array_equal(corr, want["corr"])
    np.testing.assert_allclose(got["t"], want["t"], atol=1e-8)


# ---- geometry ---------------------------------------------------------------------------------------------------------
def test_flat_target_removes_the_normal_offset_only(ctx):
    g = np.arange(-1.0, 1.0, 0.02)
    X, Y = np.meshgrid(g, g)
    dst = np.stack([X.ravel(), Y.ravel(), np.zeros(X.size)], axis=1).astype(np.float32)
    nrm = np.tile(np.array([0, 0, 1, 0], dtype=np.float32), (len(dst), 1))
    src = (dst.astype(np.float64) + [0.003, 0.002, 0.01]).astype(np.float32)
    got, _ = ctx.icp_point_to_plane(src, dst, nrm, R_CORR, max_iteration=10)
    assert got["n_correspondences"] == len(src)
    off = (src.astype(np.float64) - dst.astype(np.float64)).mean(axis=0)  # the offset after the float rounding
    assert abs(got["t"][2] + off[2]) < 1e-12
    assert abs(got["t"][0]) < 1e-12 and abs(got["t"][1]) < 1e-12  # no drift in the plane
    np.testing.assert_allclose(got["R"], np.eye(3), rtol=0, atol=1e-12)


def _grid_surface(offset):
    """A smooth surface on a 2^-16 grid at `offset`, its analytic normals, and a motion (a quarter turn about z and a
    shift by whole float steps) that maps its float points onto floats exactly."""
    rng = np.random.default_rng(7)
    uv = rng.uniform(-1, 1, (3000, 2))
    z = 0.3 * np.sin(3 * uv[:, 0]) * np.cos(2 * uv[:, 1])
    n = np.stack([-0.9 * np.cos(3 * uv[:, 0]) * np.cos(2 * uv[:, 1]), 0.6 * np.sin(3 * uv[:, 0]) * np.sin(2 * uv[:, 1]),
                  np.ones(len(uv))], axis=1)
    P = np.round(np.stack([uv[:, 0], uv[:, 1], z], axis=1) * 2.0 ** 16) * 2.0 ** -16
    src = (P + np.asarray(offset)).astype(np.float32)
    R = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
    c = np.asarray(offset)
    t = c - R @ c + np.array([3.0, -2.0, 1.0]) * 2.0 ** -7
    dst = (src.astype(np.float64) @ R.T + t).astype(np.float32)
    nrm = np.concatenate([(n / np.linalg.norm(n, axis=1, keepdims=True)) @ R.T, np.zeros((len(n), 1))], axis=1)
    return src, dst, nrm.astype(np.float32), R, t


def test_exact_recovery_at_the_origin(ctx):
    src, dst, nrm, R, t = _grid_surface((0.0, 0.0, 0.0))
    assert np.array_equal(dst.astype(np.float64), src.astype(np.float64) @ R.T + t)  # the motion is exact in floats
    init = perturbed(R, t, 7, deg=1.0, shift=0.4 * R_CORR, center=(0.0, 0.0, 0.0))
    got, _ = ctx.icp_point_to_plane(src, dst, nrm, R_CORR, init=init, max_iteration=60, relative_fitness=0,
                                    relative_rmse=0)
    np.testing.assert_allclose(got["R"], R, rtol=0, atol=1e-9)
    np.testing.assert_allclose(got["t"], t, rtol=0, atol=1e-9)
    assert got["n_correspondences"] == len(src)


def test_large_offset_as_accurate_as_at_the_origin(ctx):
    """test_gpu_icp's check for point-to-point, here with device normals: the ground-truth error at 1e5 is no worse
    than twice the error at the origin (or 0.05 degrees and 1e-3, whichever is larger)."""
    errs = []
    for off in ((0.0, 0.0, 0.0), (1e5, -1e5, 5e4)):
        src, dst, R, t = scan_pair(71, 3000, 3000, offset=off)
        nrm = ctx.estimate_normals(dst, RN)
        init = perturbed(R, t, 71, deg=2.0, shift=R_CORR, center=off)
        got, _ = ctx.icp_point_to_plane(src, dst, nrm, R_CORR, init=init)
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
    nrm = ctx.estimate_normals(dst, RN)
    init = perturbed(R, t, 51, shift=0.2 * R_CORR)
    got, corr = ctx.icp_point_to_plane(src, dst, nrm, R_CORR, init=init, max_iteration=0)
    p2p, corr2 = ctx.icp(src, dst, R_CORR, init=init, max_iteration=0)
    assert got["iterations"] == 0 and not got["converged"]
    assert np.array_equal(got["R"], np.asarray(init["rotation"])) and np.array_equal(got["t"], init["translation"])
    assert all(np.array_equal(got[k], p2p[k]) for k in got) and np.array_equal(corr, corr2) and len(corr) > 0


def test_clouds_farther_apart_than_r(ctx):
    src, dst, _, _ = scan_pair(41, 500, 500)
    got, corr = ctx.icp_point_to_plane(src, dst + np.float32(10.0), ctx.estimate_normals(dst, RN), R_CORR)
    assert (got["iterations"], got["converged"], got["n_correspondences"]) == (1, True, 0)
    assert got["fitness"] == 0.0 and got["inlier_rmse"] == 0.0 and corr.shape == (0, 2)
    np.testing.assert_array_equal(got["R"], np.eye(3))
    np.testing.assert_array_equal(got["t"], np.zeros(3))


def test_launch_count_does_not_depend_on_B(ctx):
    src, dst, R, t = scan_pair(99, 2000, 2000)
    nrm = ctx.estimate_normals(dst, RN)
    counts = []
    for B in (1, 5):
        l0 = ctx.kernel_launches()
        ctx.icp_point_to_plane_batch([src] * B, [dst] * B, [nrm] * B, R_CORR, [perturbed(R, t, 99)] * B,
                                     max_iteration=7)
        counts.append(ctx.kernel_launches() - l0)
    assert counts == [4 + 2 + 4 * 7] * 2
    small = ctx.icp_point_to_plane_batch  # targets below 1024 points: no grid build
    l0 = ctx.kernel_launches()
    small([src[:500]] * 3, [dst[:500]] * 3, [nrm[:500]] * 3, R_CORR, max_iteration=5)
    assert ctx.kernel_launches() - l0 == 2 + 4 * 5


def test_retained_solve_survives_the_new_calls(ctx):
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
    nrm = ctx.estimate_normals_batch([d], RN)[0]
    ctx.estimate_normals(d, RN)
    ctx.icp_point_to_plane(s, d, nrm, R_CORR, init=perturbed(Rg, tg, 97))
    after = ctx.last_inliers(0)
    assert all(np.array_equal(a, b) for a, b in zip(before, after))
    cert_after = ctx.certify_last(noise_bound=0.02)
    assert cert_before[0]["best_suboptimality"] == cert_after[0]["best_suboptimality"]
    assert np.array_equal(cert_before[0]["suboptimality_traj"], cert_after[0]["suboptimality_traj"])


@pytest.mark.parametrize("case", ["null_normals", "null_entry", "r_zero", "nd_zero"])
def test_argument_checks_with_a_context(ctx, case):
    import test_icp_plane_cpu as cpu
    p = capi.icp_params(0.1)
    kw = {"null_normals": dict(normals="null"), "null_entry": dict(normals="null_entry"), "nd_zero": dict(nd=0)}.get(
        case, {})
    if case == "r_zero":
        p.max_correspondence_distance = 0.0
    assert cpu._icp_batch(ctx._h, p, **kw) == capi.TZR_ERR_INVALID_ARG
    assert cpu._icp_batch(ctx._h, capi.icp_params(0.1)) == 0


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
    chained = ctx.register_cloud_pairs_icp(clouds, pairs, prm, R_CORR, max_iteration=40, method="point_to_plane",
                                           **PAIR_FLAGS)
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
    want, _ = ctx.icp_point_to_plane_batch([clouds[pairs[p][0]] for p in refined], [clouds[pairs[p][1]] for p in refined],
                                           [normals[pairs[p][1]] for p in refined], R_CORR, seeds, max_iteration=40)
    for k, p in enumerate(refined):
        assert icp_res[p].tobytes() == want[k].tobytes(), p
        assert icp_res[p]["iterations"] >= 1 and icp_res[p]["n_correspondences"] > 0
    # point-to-point's chained entry refines the same pairs, differently
    p2p = ctx.register_cloud_pairs_icp(clouds, pairs, prm, R_CORR, max_iteration=40, **PAIR_FLAGS)[6]
    assert any(p2p[p].tobytes() != icp_res[p].tobytes() for p in refined)
    assert (l3 - l2) - (l1 - l0) == 1 + 4 + 2 + 4 * 40


# ---- façades ----------------------------------------------------------------------------------------------------------
def test_cpp_facade_equals_the_c_abi(tmp_path):
    """PointToPlaneICP::refine / refineBatch, estimateNormals(Batch) and solveCloudPairsPointToPlane against the C-ABI
    (tests/cpp/icp_plane_test.cc)."""
    subprocess.check_call(["make", "-s", "-C", HOST])
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    exe = str(tmp_path / "icp_plane_test")
    subprocess.check_call([cxx, "-std=c++17", "-O1", "-I", os.path.join(HOST, "include"), "-I",
                           os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "icp_plane_test.cc"),
                           "-L", HOST, "-lteaser_registration", "-L", CSRC, "-lteaser_b200",
                           f"-Wl,-rpath,{HOST}:{CSRC}", "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr


def test_pybind_point_to_plane(ctx):
    subprocess.check_call(["make", "-s", "-C", HOST])
    sys.path.insert(0, os.path.join(HOST, "python"))
    import teaserpp_python as tpp
    src, dst, R, t = scan_pair(101, 1500, 1200)
    nrm = tpp.estimate_normals(dst, RN)
    assert nrm.tobytes() == ctx.estimate_normals(dst, RN).tobytes()
    nb = tpp.estimate_normals_batch([src, dst], RN)
    assert nb[1].tobytes() == nrm.tobytes()
    init = perturbed(R, t, 101)
    seed = tpp.RegistrationSolution()
    seed.scale = 1.0
    seed.rotation = np.asarray(init["rotation"], dtype=np.float64)
    seed.translation = np.asarray(init["translation"], dtype=np.float64)
    icp = tpp.PointToPlaneICP(R_CORR, max_iteration=30)
    got = icp.refine(src, dst, nrm, seed)
    want, corr = ctx.icp_point_to_plane(src, dst, nrm, R_CORR, init=init)
    assert np.array_equal(np.asarray(got["solution"].rotation), want["R"])
    assert np.array_equal(np.asarray(got["solution"].translation).ravel(), want["t"])
    assert (got["fitness"], got["inlier_rmse"], got["iterations"], got["converged"]) == \
        (want["fitness"], want["inlier_rmse"], want["iterations"], want["converged"])
    assert np.array_equal(np.array(got["correspondences"], dtype=np.int32).reshape(-1, 2), corr)
    batch = icp.refine_batch([src, src], [dst, dst], [nrm, nrm[:, :3]], [seed, seed])
    assert all(b["iterations"] == got["iterations"] and b["fitness"] == got["fitness"] for b in batch)
    clouds = _sequence([600, 700, 500], seed=9)
    pairs = [(0, 1), (1, 2)]
    solver = tpp.RobustRegistrationSolver(noise_bound=0.01, estimate_scaling=False, rotation_cost_threshold=1e-12)
    res = solver.solve_cloud_pairs_icp(clouds, pairs, R_CORR, normal_search_radius=PAIR_FLAGS["normal_search_radius"],
                                       fpfh_search_radius=PAIR_FLAGS["fpfh_search_radius"], use_absolute_scale=False,
                                       use_tuple_test=False, tuple_seed=0, method="point_to_plane")
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=0, rotation_cost_threshold=1e-12)
    c = ctx.register_cloud_pairs_icp(clouds, pairs, prm, R_CORR, method="point_to_plane", **PAIR_FLAGS)
    assert any(r["refined"] for r in res)
    for p, r in enumerate(res):
        assert r["refined"] == bool(c[1][p] == 0 and c[0][p]["valid"])
        if r["refined"]:
            d = capi.icp_result_dict(c[6][p])
            assert np.array_equal(np.asarray(r["icp"]["solution"].rotation), d["R"])
            assert r["icp"]["iterations"] == d["iterations"] and r["icp"]["fitness"] == d["fitness"]
    with pytest.raises(ValueError):
        solver.solve_cloud_pairs_icp(clouds, pairs, R_CORR, method="plane")


# ---- the tutorial from raw scans, refined point-to-plane ---------------------------------------------------------------
def test_tutorial_from_raw_scans_point_to_plane(ctx):
    from test_gpu_voxel import V, raw_pair
    pairs_gt = [raw_pair(20), raw_pair(21)]
    raw = [c for s, d, _, _ in pairs_gt for c in (s, d)]
    down = ctx.voxel_downsample_batch(raw, V)
    prm = capi.default_params(noise_bound=V, estimate_scaling=0, rotation_cost_threshold=1e-12)
    res = ctx.register_cloud_pairs_icp(down, [(0, 1), (2, 3)], prm, V, normal_search_radius=2 * V,
                                       fpfh_search_radius=5 * V, use_absolute_scale=False, use_crosscheck=True,
                                       use_tuple_test=False, method="point_to_plane")
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
