"""Fast Global Registration on the device (run on an H100: `pytest -m gpu`).

The device against the restatement (tests/fgr_reference.py) over both scale modes, decrease_mu on and off, 0, 1 and 64
iterations, duplicated rows and K from the fallback's 9 to 100 000 (past the robust solve's 65536 cap); recovery at
95 % outliers; batches against each problem alone and permuted; the evaluation against tzr_icp_batch with
max_iteration = 0; the launch count; non-finite points; the chained entry against the public chain; and the C++
(tests/cpp/fgr_test.cc) and pybind façades against the C-ABI and ctypes.
"""
import importlib
import os
import subprocess
import sys

import numpy as np
import pytest

import fgr_reference as fr
from test_gpu_register_pairs import EXAMPLE, RF, RN, chain, params, sequence

capi = importlib.import_module("teaser-plusplus_b200.capi")

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "teaser-plusplus_b200", "host")
CSRC = os.path.join(ROOT, "teaser-plusplus_b200", "csrc")

# The restatement performs every sum and product of the device in the device's order (fgr_reference.block_sum), so
# the two differ only where sin / cos do: the host libm and CUDA's sincos agree to within 2 ulp, and the Gauss-Newton
# steps of these well-posed problems contract such differences instead of growing them.  1e-11 on R and on t / (1 +
# |t|) leaves a margin of about 1e4 over the few-ulp differences while catching any change of order or expression,
# which moves the result by far more on problems of hundreds of rows.
TOL = 1e-11


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


def problem(K, seed, outlier_rate=0.5, noise=1e-3, n=None, dup=0):
    """float32 clouds x (n points) and y = R x + t + noise, and K correspondences: a share of them random rows, dup of
    them duplicated.  Returns x, y, corr, R, t."""
    rng = np.random.default_rng(seed)
    n = max(64, K) if n is None else n
    x = rng.uniform(-1, 1, (n, 3)) + np.array([2.0, -1.0, 0.5])
    ax = rng.normal(size=3)
    ax /= np.linalg.norm(ax)
    Kx = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    a = rng.uniform(0.2, 0.8)
    R = np.eye(3) + np.sin(a) * Kx + (1 - np.cos(a)) * Kx @ Kx
    t = rng.uniform(-1, 1, 3)
    y = x @ R.T + t + rng.normal(scale=noise, size=x.shape)
    i = rng.integers(0, n, K)
    j = i.copy()
    bad = rng.random(K) < outlier_rate
    j[bad] = rng.integers(0, n, int(bad.sum()))
    corr = np.stack([i, j], axis=1).astype(np.int32)
    if dup:
        corr = np.concatenate([corr, corr[rng.integers(0, K, dup)]])[:K]
    return x.astype(np.float32), y.astype(np.float32), corr, R, t


def fgr_prm(**kw):
    return capi.fgr_params(**kw)


def close(res, ref):
    d = capi.icp_result_dict(res)
    assert d["iterations"] == ref["iterations"] and d["converged"] == bool(ref["converged"])
    assert d["scale"] == 1.0
    assert np.abs(d["R"] - ref["R"]).max() <= TOL, np.abs(d["R"] - ref["R"]).max()
    assert np.abs(d["t"] - ref["t"]).max() <= TOL * (1 + np.abs(ref["t"]).max()), np.abs(d["t"] - ref["t"]).max()


MODES = [dict(), dict(use_absolute_scale=1), dict(decrease_mu=0), dict(iteration_number=1), dict(iteration_number=0),
         dict(use_absolute_scale=1, decrease_mu=0, iteration_number=1)]
MIDS = ["default", "absolute", "fixed_mu", "one_step", "no_step", "absolute_fixed_one"]


@pytest.mark.parametrize("K", [9, 10, 255, 256, 257, 4096, 100000])
@pytest.mark.parametrize("mode", MODES, ids=MIDS)
def test_device_matches_the_restatement(ctx, K, mode):
    x, y, corr, _, _ = problem(K, seed=K, dup=K // 10)
    res, _ = ctx.fgr_batch([x], [y], [corr], fgr=fgr_prm(**mode))
    ref = fr.fgr(x, y, corr, **mode)
    if K < 10 or mode.get("iteration_number", 64) == 0:
        assert ref["converged"] == 0
    close(res[0], ref)


def test_recovers_the_ground_truth_at_95_percent_outliers(ctx):
    x, y, corr, R, t = problem(4000, seed=95, outlier_rate=0.95, noise=1e-3, n=4000)
    res, _ = ctx.fgr_batch([x], [y], [corr], fgr=fgr_prm(maximum_correspondence_distance=1e-4, iteration_number=128))
    d = capi.icp_result_dict(res[0])
    ang = np.degrees(np.arccos(np.clip((np.trace(d["R"].T @ R) - 1) / 2, -1, 1)))
    assert ang < 0.1 and np.linalg.norm(d["t"] - t) < 5e-3, (ang, d["t"] - t)
    close(res[0], fr.fgr(x, y, corr, maximum_correspondence_distance=1e-4, iteration_number=128))


def _batch(ctx, probs, fgr):
    res, ev = ctx.fgr_batch([p[0] for p in probs], [p[1] for p in probs], [p[2] for p in probs], fgr=fgr)
    return [res[k:k + 1].tobytes() for k in range(len(probs))], [e.tobytes() for e in ev]


def test_batch_equals_each_problem_alone_and_any_order(ctx):
    probs = [problem(K, seed=s, n=n)[:3] for K, s, n in ((300, 1, 500), (9, 2, 64), (5000, 3, 1500), (0, 4, 80),
                                                          (20000, 5, 3000), (257, 6, 2000))]
    fgr = fgr_prm()
    rec, ev = _batch(ctx, probs, fgr)
    for k, p in enumerate(probs):
        r1, e1 = _batch(ctx, [p], fgr)
        assert rec[k] == r1[0] and ev[k] == e1[0], k
        res1, e1 = ctx.fgr_batch([p[0]], [p[1]], [p[2]], fgr=fgr, single=True)  # the single-problem entry, tzr_fgr
        assert res1[0:1].tobytes() == rec[k] and e1[0].tobytes() == ev[k], k
    perm = [4, 0, 5, 2, 1, 3]
    rp, ep = _batch(ctx, [probs[k] for k in perm], fgr)
    for a, k in enumerate(perm):
        assert rp[a] == rec[k] and ep[a] == ev[k]


@pytest.mark.parametrize("K", [9, 600, 20000])
def test_evaluation_is_icp_with_no_iteration(ctx, K):
    x, y, corr, _, _ = problem(K, seed=7 + K, n=max(K, 1500))
    fgr = fgr_prm(maximum_correspondence_distance=0.05)
    res, ev = ctx.fgr_batch([x], [y], [corr], fgr=fgr)
    d = capi.icp_result_dict(res[0])
    init = dict(scale=1.0, rotation=d["R"], translation=d["t"])
    ires, icorr = ctx.icp_batch([x], [y], 0.05, inits=[init], max_iteration=0)
    for f in ("fitness", "inlier_rmse", "n_correspondences"):
        assert np.float64(res[0][f]).tobytes() == np.float64(ires[0][f]).tobytes(), f
    assert res[0]["transform"].tobytes() == ires[0]["transform"].tobytes()
    assert np.array_equal(ev[0], icorr[0])
    # and the record seeds ICP directly
    ctx.icp_batch([x], [y], 0.05, inits=[init], max_iteration=5)


def test_launch_count_does_not_depend_on_iterations_or_batch(ctx):
    x, y, corr, _, _ = problem(500, seed=9, n=600)
    counts = []
    for it, B in ((1, 1), (64, 1), (1, 256), (64, 256)):
        l0 = ctx.kernel_launches()
        ctx.fgr_batch([x] * B, [y] * B, [corr] * B, fgr=fgr_prm(iteration_number=it))
        counts.append(ctx.kernel_launches() - l0)
    assert counts == [4, 4, 4, 4], counts
    big = problem(500, seed=9, n=2000)
    l0 = ctx.kernel_launches()
    ctx.fgr_batch([big[0]], [big[1]], [big[2]])
    assert ctx.kernel_launches() - l0 == 8  # the evaluation's grid build for a 2000-point target


def test_non_finite_points(ctx):
    x, y, corr, _, _ = problem(800, seed=13, n=400)
    x[::7] = np.nan
    y[3::11, 1] = np.inf
    res, _ = ctx.fgr_batch([x], [y], [corr])
    ref = fr.fgr(x, y, corr)
    assert ref["info"]["K"] < 800 and ref["converged"] == 1
    close(res[0], ref)
    # no finite point in the source: every row is dropped, the identity
    xn = np.full_like(x, np.nan)
    res, _ = ctx.fgr_batch([xn], [y], [corr])
    d = capi.icp_result_dict(res[0])
    assert d["iterations"] == 0 and not d["converged"]
    assert np.array_equal(d["R"], np.eye(3)) and np.array_equal(d["t"], np.zeros(3))


def test_refusals_launch_nothing(ctx):
    x, y, corr, _, _ = problem(50, seed=1, n=64)
    l0 = ctx.kernel_launches()
    for bad in ([[0, 64]], [[-1, 0]], [[64, 0]], [[0, -3]]):
        with pytest.raises(capi.TzrError, match="invalid"):
            ctx.fgr_batch([x], [y], [np.array(bad)])
    for kw in (dict(division_factor=0.0), dict(division_factor=np.nan), dict(maximum_correspondence_distance=-1.0),
               dict(maximum_correspondence_distance=np.inf), dict(iteration_number=-1)):
        with pytest.raises(capi.TzrError, match="invalid"):
            ctx.fgr_batch([x], [y], [corr], fgr=fgr_prm(**kw))
    assert ctx.kernel_launches() == l0


# ---- the chained entry ---------------------------------------------------------------------------------------------
def three_calls(ctx, clouds, pairs, flags, seeds, fgr):
    """tzr_compute_fpfh_batch, tzr_match_correspondences_batch and tzr_fgr_batch on the matched rows."""
    want = chain(ctx, clouds, pairs, params(), flags, seeds, max_n=1 << 30)
    reg = [p for p in range(len(pairs)) if want["corr"][p] is not None and len(want["corr"][p]) > 0]
    res = {}
    if reg:
        r, _ = ctx.fgr_batch([clouds[pairs[p][0]] for p in reg], [clouds[pairs[p][1]] for p in reg],
                             [want["corr"][p] for p in reg], fgr=fgr)
        res = {p: r[k:k + 1].tobytes() for k, p in enumerate(reg)}
    return want, res


def check_chain(ctx, clouds, pairs, flags=EXAMPLE, fgr=None):
    fgr = fgr_prm() if fgr is None else fgr
    seeds = list(range(100, 100 + len(pairs)))
    status, corr, scales, res = ctx.register_cloud_pairs_fgr(clouds, pairs, RN, RF, *flags, tuple_seeds=seeds, fgr=fgr)
    want, wres = three_calls(ctx, clouds, pairs, flags, seeds, fgr)
    zero = bytes(res[0:1].nbytes)
    for p, (a, b) in enumerate(pairs):
        if want["ovf"][a] or want["ovf"][b]:
            assert status[p] == capi.TZR_ERR_TOO_LARGE and len(corr[p]) == 0 and res[p:p + 1].tobytes() == zero, p
            continue
        assert np.array_equal(corr[p], want["corr"][p]), p
        assert np.float32(scales[p]).tobytes() == np.float32(want["scales"][p]).tobytes(), p
        if len(corr[p]) == 0:
            assert status[p] == capi.TZR_ERR_INVALID_ARG and res[p:p + 1].tobytes() == zero, p
        else:
            assert status[p] == 0 and res[p:p + 1].tobytes() == wres[p], p
    return status, res


def test_chained_entry_equals_the_three_calls(ctx):
    clouds, pairs = sequence([600, 700, 650, 1500], seed=17)
    status, _ = check_chain(ctx, clouds, pairs + [(1, 0), (2, 2), (0, 3)])
    assert (status == 0).all()
    check_chain(ctx, clouds, pairs, fgr=fgr_prm(use_absolute_scale=1, iteration_number=7, decrease_mu=0))


def test_chained_entry_statuses(ctx):
    rng = np.random.default_rng(41)
    clouds, pairs = sequence([500, 600], seed=43)
    clouds.append(rng.uniform(0, 0.01, size=(5000, 3)).astype(np.float32))  # every point has 5000 neighbours
    clouds += [np.array([[0.1, 0.2, 0.3]], dtype=np.float32), np.array([[0.4, 0.1, 0.2]], dtype=np.float32)]
    pairs = [(0, 1), (2, 0), (3, 4), (1, 0)]
    status, _ = check_chain(ctx, clouds, pairs, flags=(False, True, True, 0.95))
    assert list(status) == [0, capi.TZR_ERR_TOO_LARGE, capi.TZR_ERR_INVALID_ARG, 0]


def test_chained_entry_keeps_a_retained_solve(ctx):
    rng = np.random.default_rng(11)
    src = rng.uniform(-1, 1, (200, 3))
    dst = src @ np.array([[0.0, -1, 0], [1, 0, 0], [0, 0, 1]]).T + 0.3
    dst[:40] = rng.uniform(-1, 1, (40, 3))
    ctx.solve(src, dst, capi.default_params(noise_bound=0.01))
    before = [m.tobytes() for m in ctx.last_inliers(0)]
    info0 = ctx.last_graph_info()
    clouds, pairs = sequence([500, 600], seed=3)
    ctx.register_cloud_pairs_fgr(clouds, pairs, RN, RF, *EXAMPLE)
    x, y, corr, _, _ = problem(300, seed=2)
    ctx.fgr_batch([x], [y], [corr])
    assert [m.tobytes() for m in ctx.last_inliers(0)] == before
    assert ctx.last_graph_info() == info0


def test_bunny_under_a_known_motion(ctx):
    synth = importlib.import_module("teaser-plusplus_b200.synth")
    pts = synth.read_ply_vertices(os.path.join(synth.GOLDEN_DIR, "bun_zipper_res3.ply")).astype(np.float64)
    pts = (pts - pts.mean(0)) / np.abs(pts - pts.mean(0)).max()  # about unit size
    a = 0.5
    R = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
    t = np.array([0.3, -0.2, 0.1])
    src = pts.astype(np.float32)
    dst = (pts @ R.T + t).astype(np.float32)
    status, corr, _, res = ctx.register_cloud_pairs_fgr([src, dst], [(0, 1)], 0.1, 0.25, False, True, True, 0.95,
                                                        fgr=fgr_prm(maximum_correspondence_distance=0.01))
    assert status[0] == 0 and len(corr[0]) >= 10
    d = capi.icp_result_dict(res[0])
    ang = np.degrees(np.arccos(np.clip((np.trace(d["R"].T @ R) - 1) / 2, -1, 1)))
    assert ang < 2.0 and np.linalg.norm(d["t"] - t) < 0.05, (ang, d["t"] - t)
    init = dict(scale=1.0, rotation=d["R"], translation=d["t"])
    ires, _ = ctx.icp_batch([src], [dst], 0.05, inits=[init], max_iteration=30)
    r = capi.icp_result_dict(ires[0])
    ang2 = np.degrees(np.arccos(np.clip((np.trace(r["R"].T @ R) - 1) / 2, -1, 1)))
    assert ang2 < 0.5 and r["fitness"] > 0.9, (ang2, r["fitness"])


# ---- façades ---------------------------------------------------------------------------------------------------------
def test_cpp_facade_equals_the_c_abi(tmp_path):
    """FastGlobalRegistration::registerPair / registerBatch / registerCloudPairs against tzr_fgr, tzr_fgr_batch and
    tzr_register_cloud_pairs_fgr (tests/cpp/fgr_test.cc)."""
    subprocess.check_call(["make", "-s", "-C", HOST])
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    exe = str(tmp_path / "fgr_test")
    subprocess.check_call([cxx, "-std=c++17", "-O1", "-I", os.path.join(HOST, "include"), "-I",
                           os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "fgr_test.cc"),
                           "-L", HOST, "-lteaser_registration", "-L", CSRC, "-lteaser_b200",
                           f"-Wl,-rpath,{HOST}:{CSRC}", "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr


def _same_record(d, rec, corr):
    """A pybind icp dict against a ctypes ICP_RESULT_DTYPE record and its evaluation rows, bit for bit."""
    want = capi.icp_result_dict(rec)
    assert np.asarray(d["solution"].rotation).tobytes() == want["R"].tobytes()
    assert np.asarray(d["solution"].translation).ravel().tobytes() == want["t"].tobytes()
    assert (d["fitness"], d["inlier_rmse"], d["iterations"], d["converged"]) == \
        (want["fitness"], want["inlier_rmse"], want["iterations"], want["converged"])
    if corr is not None:
        assert np.array_equal(np.array(d["correspondences"], dtype=np.int32).reshape(-1, 2), corr)


def test_pybind_equals_ctypes(ctx):
    subprocess.check_call(["make", "-s", "-C", HOST])
    sys.path.insert(0, os.path.join(HOST, "python"))
    import teaserpp_python as tpp
    probs = [problem(K, seed=s, n=n)[:3] for K, s, n in ((600, 21, 800), (9, 22, 64), (3000, 23, 1500))]
    kw = dict(maximum_correspondence_distance=0.05, iteration_number=40, use_absolute_scale=True)
    fgr = tpp.FastGlobalRegistration(**kw)
    res, ev = ctx.fgr_batch([p[0] for p in probs], [p[1] for p in probs], [p[2] for p in probs],
                            fgr=fgr_prm(**kw))
    got = fgr.register_batch([p[0] for p in probs], [p[1] for p in probs], [p[2] for p in probs])
    for k, p in enumerate(probs):
        _same_record(got[k], res[k], ev[k])
        _same_record(fgr.register(p[0], p[1], p[2]), res[k], ev[k])
    # the cloud table: the façade's seeds are solveCloudPairs' (tuple_seed + 0x9E3779B97F4A7C15 p)
    clouds, pairs = sequence([500, 600, 550], seed=29)
    pairs = pairs + [(1, 0)]
    seeds = [(0x7EA5E2 + 0x9E3779B97F4A7C15 * p) % 2 ** 64 for p in range(len(pairs))]
    status, corr, scales, rec = ctx.register_cloud_pairs_fgr(clouds, pairs, RN, RF, *EXAMPLE, tuple_seeds=seeds)
    flags = dict(zip(("use_absolute_scale", "use_crosscheck", "use_tuple_test", "tuple_scale"), EXAMPLE))
    for out in (tpp.register_cloud_pairs_fgr(clouds, pairs, RN, RF, **flags),
                tpp.FastGlobalRegistration().register_cloud_pairs(clouds, pairs, RN, RF, **flags)):
        for p in range(len(pairs)):
            assert out[p]["status"] == status[p] and out[p]["registered"] == (status[p] == 0)
            assert np.array_equal(np.array(out[p]["correspondences"], dtype=np.int32).reshape(-1, 2), corr[p])
            assert np.float32(out[p]["global_scale"]).tobytes() == np.float32(scales[p]).tobytes()
            if status[p] == 0:
                _same_record(out[p]["fgr"], rec[p], None)
