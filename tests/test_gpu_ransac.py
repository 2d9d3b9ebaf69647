"""Correspondence RANSAC on the device (run on an H100: `pytest -m gpu`).

The device against the restatement (tests/ransac_reference.py) bit for bit: the winner's transform, the loop summary
(drawn, passed, winner, inliers, rmse) and, through tzr_icp_batch with max_iteration = 0, the record and its
correspondences; across K' from ransac_n to tens of thousands, ransac_n 3, 4 and 8, each checker, confidence 0, 0.999
and 1 and max_iteration 0, 1 and 100000.  Batches against each problem alone and permuted, including a companion that
changes the round schedule; the launch count; non-finite points, the fallbacks and the refusals; recovery at 95 %
outliers and on the bunny; the chained entry against the public chain, its statuses and the retained solve.
"""
import importlib
import math
import os
import subprocess
import sys

import numpy as np
import pytest

import ransac_reference as rr
from test_gpu_fgr import problem
from test_gpu_register_pairs import EXAMPLE, RF, RN, chain, params, sequence

capi = importlib.import_module("teaser-plusplus_b200.capi")

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


def prm(r=0.01, **kw):
    return capi.ransac_params(r, **kw)


def ref_kw(p):
    """ransac_reference.ransac's keywords for a RansacParams."""
    return dict(ransac_n=p.ransac_n, max_iteration=p.max_iteration, confidence=p.confidence,
                edge=p.edge_length_similarity if p.check_edge_length else None,
                dist=p.distance_threshold if p.check_distance else None,
                normal_angle=p.normal_angle_threshold if p.check_normal else None)


def rot(rec):
    return np.asarray(rec["transform"]["rotation"]).reshape(3, 3).T


def check(ctx, x, y, corr, p, seed, xn=None, yn=None, exact_drawn=True):
    """One problem on the device against the restatement; the record against icp_batch(max_iteration=0) seeded with
    it.  Returns the reference's dict."""
    res, info, ev = ctx.ransac_batch([x], [y], [corr], p, seeds=[seed],
                                     src_normals=None if xn is None else [xn], dst_normals=None if yn is None else [yn])
    want = rr.ransac(x, y, corr, p.max_correspondence_distance, seed=seed, xn=xn, yn=yn, **ref_kw(p))
    i = info[0]
    if exact_drawn or want["margin"] > 1e-9:
        assert (i["drawn"], i["passed"], i["winner"]) == (want["drawn"], want["passed"], want["winner"]), (i, want)
        assert int(res[0]["iterations"]) == want["drawn"] and int(res[0]["converged"]) == want["converged"]
    assert i["usable"] == want["usable"] and i["inliers"] == want["inliers"]
    assert np.float64(i["rmse"]).tobytes() == np.float64(want["rmse"]).tobytes()
    assert rot(res[0]).tobytes() == np.asarray(want["R"], dtype=np.float64).tobytes()
    assert np.asarray(res[0]["transform"]["translation"]).tobytes() == np.asarray(want["t"]).tobytes()
    assert res[0]["transform"]["scale"] == 1.0
    # the record is icp_batch with no iteration, seeded with the winner
    init = dict(scale=1.0, rotation=rot(res[0]), translation=np.asarray(res[0]["transform"]["translation"]))
    ires, icorr = ctx.icp_batch([x], [y], p.max_correspondence_distance, inits=[init], max_iteration=0)
    for f in ("fitness", "inlier_rmse", "n_correspondences"):
        assert res[0][f] == ires[0][f], f
    assert np.array_equal(ev[0], icorr[0])
    return want


CASES = [  # K, outlier rate, ransac_n, params
    (3, 0.0, 3, {}),
    (40, 0.3, 3, {}),
    (600, 0.5, 3, dict(check_edge_length=1)),
    (600, 0.5, 4, dict(check_distance=1, distance_threshold=0.02)),
    (1500, 0.4, 8, dict(check_edge_length=1, edge_length_similarity=0.95)),
    (3000, 0.5, 3, dict(confidence=0.0)),
    (800, 0.6, 3, dict(confidence=1.0, max_iteration=400)),
    (800, 0.6, 3, dict(max_iteration=1)),
    (800, 0.6, 3, dict(max_iteration=0)),
    (20000, 0.4, 3, dict(check_edge_length=1, check_distance=1, distance_threshold=0.015)),
    (5000, 0.5, 4, dict(max_iteration=3000, confidence=0.99999)),
]


@pytest.mark.parametrize("K,out,n,kw", CASES)
def test_device_matches_the_restatement(ctx, K, out, n, kw):
    x, y, corr, _, _ = problem(K, seed=K + n, outlier_rate=out, noise=1e-3)
    check(ctx, x, y, corr, prm(0.01, ransac_n=n, **kw), seed=K * 7 + 1, exact_drawn=False)


def test_normal_checker(ctx):
    x, y, corr, R, _ = problem(700, seed=5, outlier_rate=0.5)
    rng = np.random.default_rng(5)
    xn = rng.normal(size=(len(x), 3))
    xn /= np.linalg.norm(xn, axis=1, keepdims=True)
    yn = xn @ R.T
    yn[::3] = -yn[::3]  # a third of the target normals flipped: hypotheses drawing them fail
    p = prm(0.01, check_normal=1, normal_angle_threshold=0.5)
    want = check(ctx, x.astype(np.float32), y, corr, p, seed=3, xn=xn.astype(np.float32), yn=yn.astype(np.float32))
    assert want["passed"] < want["drawn"]


def test_recovers_the_ground_truth_at_95_percent_outliers(ctx):
    x, y, corr, R, t = problem(4000, seed=77, outlier_rate=0.95, noise=0.0)
    res, info, _ = ctx.ransac_batch([x], [y], [corr], prm(0.005, check_edge_length=1), seeds=[9])
    d = capi.icp_result_dict(res[0])
    assert np.abs(d["R"] - R).max() < 1e-4 and np.abs(d["t"] - t).max() < 1e-4
    assert info[0]["winner"] >= 0 and info[0]["passed"] < info[0]["drawn"]


def test_batch_equals_each_problem_alone_and_any_order(ctx):
    probs = [problem(K, seed=s, outlier_rate=o)[:3] for K, s, o in ((300, 1, 0.5), (9, 2, 0.2), (2500, 3, 0.7),
                                                                   (2, 4, 0.0), (1200, 5, 0.6))]
    p = prm(0.01, check_edge_length=1)
    seeds = [11, 12, 13, 14, 2 ** 64 - 1]
    alone = []
    for (x, y, c), s in zip(probs, seeds):
        r, i, e = ctx.ransac_batch([x], [y], [c], p, seeds=[s])
        alone.append((r.tobytes(), i.tobytes(), e[0].tobytes()))
    r1, i1, e1 = ctx.ransac(*probs[0], p, seed=seeds[0])
    assert i1 == {k: np.frombuffer(alone[0][1], dtype=capi.RANSAC_INFO_DTYPE)[0][k].item()
                  for k in capi.RANSAC_INFO_DTYPE.names}
    for order in ([0, 1, 2, 3, 4], [4, 2, 0, 3, 1]):
        r, i, e = ctx.ransac_batch([probs[k][0] for k in order], [probs[k][1] for k in order],
                                   [probs[k][2] for k in order], p, seeds=[seeds[k] for k in order])
        for j, k in enumerate(order):
            assert (r[j:j + 1].tobytes(), i[j:j + 1].tobytes(), e[j].tobytes()) == alone[k], k
    # a large companion lowers the round cap (more, smaller rounds); the small problem's bits do not move
    x, y, c = probs[0]
    big = problem(40000, seed=8, outlier_rate=0.5)[:3]
    l0 = ctx.kernel_launches()
    ctx.ransac_batch([x], [y], [c], prm(0.01, max_iteration=5000), seeds=[1])
    l1 = ctx.kernel_launches()
    r, i, e = ctx.ransac_batch([x, big[0]], [y, big[1]], [c, big[2]], prm(0.01, max_iteration=5000), seeds=[1, 2])
    l2 = ctx.kernel_launches()
    solo, si, se = ctx.ransac_batch([x], [y], [c], prm(0.01, max_iteration=5000), seeds=[1])
    assert r[0:1].tobytes() == solo.tobytes() and i[0:1].tobytes() == si.tobytes() and e[0].tobytes() == se[0].tobytes()
    # the rounds did change: 4 + 3 rounds alone; the companion's 40000 rows cut the cap, and its target adds the
    # evaluation's grid build (4)
    assert rounds(5000, 300) < rounds(5000, 40000)
    assert (l1 - l0, l2 - l1) == (4 + 3 * rounds(5000, 300), 8 + 3 * rounds(5000, 40000)), (l1 - l0, l2 - l1)


def rounds(mi, k_max):
    """The header's round schedule: the number of rounds."""
    nseg = max(1, -(-k_max // 512))
    cap = 65536
    while cap > 256 and cap * nseg > 65536:
        cap //= 2
    n, start, r = 0, 0, 256
    while start < mi:
        start += min(r, cap)
        r = min(2 * r, cap)
        n += 1
    return n


def test_launch_count_does_not_depend_on_the_batch(ctx):
    x, y, c, _, _ = problem(500, seed=9, n=600)
    for mi in (0, 1, 1000, 100000):
        counts = []
        for B in (1, 7, 64):
            l0 = ctx.kernel_launches()
            ctx.ransac_batch([x] * B, [y] * B, [c] * B, prm(0.01, max_iteration=mi))
            counts.append(ctx.kernel_launches() - l0)
        assert counts == [4 + 3 * rounds(mi, 500)] * 3, (mi, counts)
    big = problem(500, seed=9, n=2000)
    l0 = ctx.kernel_launches()
    ctx.ransac_batch([big[0]], [big[1]], [big[2]], prm(0.01, max_iteration=10))
    assert ctx.kernel_launches() - l0 == 8 + 3  # the evaluation's grid build for a 2000-point target


def test_non_finite_points_and_fallbacks(ctx):
    x, y, c, _, _ = problem(800, seed=13, n=400)
    x[::7] = np.nan
    y[3::11, 1] = np.inf
    want = check(ctx, x, y, c, prm(0.01), seed=4)
    assert want["usable"] < 800
    for xx, cc, mi in ((np.full_like(x, np.nan), c, 100), (x, c[:0], 100), (x, c[:2], 100), (x, c, 0)):
        res, info, _ = ctx.ransac_batch([xx], [y], [cc], prm(0.01, max_iteration=mi))
        d = capi.icp_result_dict(res[0])
        assert info[0]["drawn"] == 0 and info[0]["winner"] == -1 and not d["converged"]
        assert np.array_equal(d["R"], np.eye(3)) and np.array_equal(d["t"], np.zeros(3))
    # no hypothesis with an inlier (random targets, a radius far below any fit's residual): the identity after every
    # hypothesis
    scatter = np.random.default_rng(3).uniform(-1, 1, y.shape).astype(np.float32)
    res, info, _ = ctx.ransac_batch([x], [scatter], [c], prm(1e-9, max_iteration=300, ransac_n=4))
    assert info[0]["winner"] == -1 and info[0]["drawn"] == 300 and res[0]["converged"] == 0


def test_refusals_launch_nothing(ctx):
    x, y, corr, _, _ = problem(50, seed=1, n=64)
    l0 = ctx.kernel_launches()
    for bad in ([[0, 64]], [[-1, 0]], [[64, 0]]):
        with pytest.raises(capi.TzrError, match="invalid"):
            ctx.ransac_batch([x], [y], [np.array(bad)], prm())
    for kw in (dict(max_correspondence_distance=0.0), dict(max_correspondence_distance=np.nan), dict(ransac_n=2),
               dict(ransac_n=17), dict(max_iteration=-1), dict(confidence=1.5), dict(confidence=-0.1),
               dict(check_edge_length=2), dict(check_distance=1, distance_threshold=np.inf),
               dict(check_normal=1)):  # the normal checker without normals
        p = prm()
        for k, v in kw.items():
            setattr(p, k, v)
        with pytest.raises(capi.TzrError, match="invalid"):
            ctx.ransac_batch([x], [y], [corr], p)
    assert ctx.kernel_launches() == l0


def test_both_search_routes(ctx):
    x, y, c, _, _ = problem(1500, seed=31, n=1500)
    for flag in (capi.FLAG_ICP_BRUTE_FORCE, capi.FLAG_ICP_GRID):
        ctx.set_flags(flag)
        try:
            check(ctx, x, y, c, prm(0.01, check_edge_length=1), seed=5)
        finally:
            ctx.set_flags(0)


# ---- the chained entry ---------------------------------------------------------------------------------------------
def check_chain(ctx, clouds, pairs, p, flags=EXAMPLE):
    seeds = list(range(100, 100 + len(pairs)))
    rseeds = [7 * k + 3 for k in range(len(pairs))]
    status, corr, scales, res, info = ctx.register_cloud_pairs_ransac(clouds, pairs, p, RN, RF, *flags,
                                                                      tuple_seeds=seeds, ransac_seeds=rseeds)
    want = chain(ctx, clouds, pairs, params(), flags, seeds, max_n=1 << 30)
    normals = None
    if p.check_normal:
        normals = [ctx.estimate_normals(c, RN) for c in clouds]
    zero = bytes(res[0:1].nbytes)
    for q, (a, b) in enumerate(pairs):
        if want["ovf"][a] or want["ovf"][b]:
            assert status[q] == capi.TZR_ERR_TOO_LARGE and res[q:q + 1].tobytes() == zero, q
            continue
        assert np.array_equal(corr[q], want["corr"][q]), q
        if len(corr[q]) == 0:
            assert status[q] == capi.TZR_ERR_INVALID_ARG and res[q:q + 1].tobytes() == zero, q
            continue
        r, i, _ = ctx.ransac_batch([clouds[a]], [clouds[b]], [corr[q]], p, seeds=[rseeds[q]],
                                   src_normals=None if normals is None else [normals[a]],
                                   dst_normals=None if normals is None else [normals[b]])
        assert status[q] == 0 and res[q:q + 1].tobytes() == r.tobytes() and info[q:q + 1].tobytes() == i.tobytes(), q
    return status


def test_chained_entry_equals_the_three_calls(ctx):
    clouds, pairs = sequence([600, 700, 650, 1500], seed=17)
    status = check_chain(ctx, clouds, pairs + [(1, 0), (2, 2), (0, 3)], prm(0.02, check_edge_length=1))
    assert (status == 0).all()
    check_chain(ctx, clouds, pairs, prm(0.02, check_normal=1, normal_angle_threshold=0.6, max_iteration=2000))


def test_chained_entry_statuses(ctx):
    rng = np.random.default_rng(41)
    clouds, pairs = sequence([500, 600], seed=43)
    clouds.append(rng.uniform(0, 0.01, size=(5000, 3)).astype(np.float32))  # every point has 5000 neighbours
    clouds += [np.array([[0.1, 0.2, 0.3]], dtype=np.float32), np.array([[0.4, 0.1, 0.2]], dtype=np.float32)]
    pairs = [(0, 1), (2, 0), (3, 4), (1, 0)]
    status = check_chain(ctx, clouds, pairs, prm(0.02), flags=(False, True, True, 0.95))
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
    ctx.register_cloud_pairs_ransac(clouds, pairs, prm(0.02), RN, RF, *EXAMPLE)
    x, y, corr, _, _ = problem(300, seed=2)
    ctx.ransac_batch([x], [y], [corr], prm())
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
    p = prm(0.02, check_edge_length=1, check_distance=1, distance_threshold=0.02)
    status, corr, _, res, info = ctx.register_cloud_pairs_ransac([src, dst], [(0, 1)], p, 0.1, 0.25, False, True, True,
                                                                 0.95)
    assert status[0] == 0 and len(corr[0]) >= 3 and info[0]["winner"] >= 0
    d = capi.icp_result_dict(res[0])
    ang = np.degrees(np.arccos(np.clip((np.trace(d["R"].T @ R) - 1) / 2, -1, 1)))
    assert ang < 2.0 and np.linalg.norm(d["t"] - t) < 0.05, (ang, d["t"] - t)
    init = dict(scale=1.0, rotation=d["R"], translation=d["t"])
    ires, _ = ctx.icp_batch([src], [dst], 0.05, inits=[init], max_iteration=30)
    r = capi.icp_result_dict(ires[0])
    ang2 = np.degrees(np.arccos(np.clip((np.trace(r["R"].T @ R) - 1) / 2, -1, 1)))
    assert ang2 < 0.5 and r["fitness"] > 0.9, (ang2, r["fitness"])
    # the winner's fitness is its inliers over the usable rows, recounted from the matched rows
    X, Y, _ = rr.usable(src, dst, corr[0])
    cnt, _, f, _ = rr.score(d["R"], d["t"], X, Y, 0.02 ** 2)
    assert cnt == info[0]["inliers"] and math.isclose(f, info[0]["inliers"] / info[0]["usable"])


# ---- every bound at equality, on the device ----------------------------------------------------------------------------
def first_hypothesis(x, y, c, seed, n=3):
    """Hypothesis 0's drawn rows and its (R, t), from the restatement (bit-exact with the device)."""
    X, Y, _ = rr.usable(x, y, c)
    rows = rr.draws(seed, n, 0, len(X))
    R, t = rr.kabsch(X[rows], Y[rows])
    return X, Y, rows, R, t


def test_score_counts_strictly_inside_at_the_device(ctx):
    x, y, c, _, _ = problem(3000, seed=61, outlier_rate=0.3, noise=2e-3)
    X, Y, _, R, t = first_hypothesis(x, y, c, seed=5)
    d2 = rr.d2_rows(R, t, X, Y)
    order = np.argsort(d2)
    r = None
    for k in order[len(order) // 4:]:  # a row whose d^2 is exactly some r * r
        cand = float(np.sqrt(d2[k]))
        if d2[k] > 0 and cand * cand == d2[k]:
            r = cand
            break
    assert r is not None
    assert int((d2 < r * r).sum()) < int((d2 <= r * r).sum())  # a row lies on the bound
    want = check(ctx, x, y, c, prm(r, max_iteration=1), seed=5)
    assert want["winner"] == 0 and want["inliers"] == int((d2 < r * r).sum())


def test_distance_checker_at_equality_on_the_device(ctx):
    x, y, c, _, _ = problem(500, seed=62, outlier_rate=0.2, noise=2e-3)
    X, Y, rows, R, t = first_hypothesis(x, y, c, seed=8)
    m = max(math.sqrt(v) for v in rr.d2_rows(R, t, X[rows], Y[rows]))
    assert m > 0
    for thr, passed in ((m, 1), (float(np.nextafter(m, 0.0)), 0)):
        want = check(ctx, x, y, c, prm(0.01, max_iteration=1, check_distance=1, distance_threshold=thr), seed=8)
        assert want["passed"] == passed, thr


def test_normal_checker_at_equality_on_the_device(ctx):
    x, y, c, _, _ = problem(500, seed=63, outlier_rate=0.2, noise=2e-3)
    X, Y, rows, R, _ = first_hypothesis(x, y, c, seed=4)
    rng = np.random.default_rng(63)
    for _ in range(50):  # normals whose smallest dot product is exactly the cosine of some angle
        xn = rng.normal(size=(len(x), 3)).astype(np.float32)
        yn = (xn.astype(np.float64) @ R.T + rng.normal(scale=0.3, size=xn.shape)).astype(np.float32)
        NX, NY = xn.astype(np.float64)[c[:, 0]], yn.astype(np.float64)[c[:, 1]]
        dots = []
        for k in rows:
            mm = [(R[q, 0] * NX[k, 0] + R[q, 1] * NX[k, 1]) + R[q, 2] * NX[k, 2] for q in range(3)]
            dots.append((NY[k, 0] * mm[0] + NY[k, 1] * mm[1]) + NY[k, 2] * mm[2])
        d = min(dots)
        if not -0.9 < d < 0.9:
            continue
        a = math.acos(d)
        hit = None
        for _ in range(64):
            if math.cos(a) == d:
                hit = a
                break
            a = float(np.nextafter(a, 0.0 if math.cos(a) < d else 4.0))
        if hit is None:
            continue
        below = hit
        while math.cos(below) <= d:  # a slightly smaller angle: cos above the dot product, the check fails
            below = float(np.nextafter(below, 0.0))
        for angle, passed in ((hit, 1), (below, 0)):
            want = check(ctx, x, y, c, prm(0.01, max_iteration=1, check_normal=1, normal_angle_threshold=angle),
                         seed=4, xn=xn, yn=yn)
            assert want["passed"] == passed, angle
        return
    pytest.fail("no angle whose cosine equals the smallest dot product")


def test_edge_checker_at_equality_on_the_device(ctx):
    K, seed = 200, 21
    rows = rr.draws(seed, 3, 0, K)
    assert len(set(rows)) == 3
    rng = np.random.default_rng(21)
    x = rng.uniform(-1, 1, (K, 3)).astype(np.float32)
    y = rng.uniform(-1, 1, (K, 3)).astype(np.float32)
    for k, p in zip(rows, ([0, 0, 0], [2, 0, 0], [0, 2, 0])):  # the sample's target edges are exactly half its source's
        x[k] = p
        y[k] = np.float32(0.5) * x[k]
    c = np.stack([np.arange(K), np.arange(K)], axis=1).astype(np.int32)
    for s, passed in ((0.5, 1), (float(np.nextafter(0.5, 1.0)), 0)):
        want = check(ctx, x, y, c, prm(0.01, max_iteration=1, check_edge_length=1, edge_length_similarity=s),
                     seed=seed)
        assert want["passed"] == passed, s


# ---- façades ---------------------------------------------------------------------------------------------------------
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "teaser-plusplus_b200", "host")
CSRC = os.path.join(ROOT, "teaser-plusplus_b200", "csrc")


def test_cpp_facade_equals_the_c_abi(tmp_path):
    """RANSACRegistration::registerPair / registerBatch / registerCloudPairs against tzr_ransac, tzr_ransac_batch and
    tzr_register_cloud_pairs_ransac (tests/cpp/ransac_test.cc)."""
    subprocess.check_call(["make", "-s", "-C", HOST])
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    exe = str(tmp_path / "ransac_test")
    subprocess.check_call([cxx, "-std=c++17", "-O1", "-I", os.path.join(HOST, "include"), "-I",
                           os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "ransac_test.cc"),
                           "-L", HOST, "-lteaser_registration", "-L", CSRC, "-lteaser_b200",
                           f"-Wl,-rpath,{HOST}:{CSRC}", "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr


def _same_record(d, rec, info, corr):
    """A pybind ransac dict against a ctypes ICP_RESULT_DTYPE record, its RANSAC_INFO_DTYPE summary and its
    evaluation rows, bit for bit."""
    want = capi.icp_result_dict(rec)
    assert np.asarray(d["solution"].rotation).tobytes() == want["R"].tobytes()
    assert np.asarray(d["solution"].translation).ravel().tobytes() == want["t"].tobytes()
    assert (d["fitness"], d["inlier_rmse"], d["iterations"], d["converged"]) == \
        (want["fitness"], want["inlier_rmse"], want["iterations"], want["converged"])
    assert d["info"] == {k: info[k].item() for k in ("drawn", "passed", "winner", "inliers", "usable", "rmse")}
    if corr is not None:
        assert np.array_equal(np.array(d["correspondences"], dtype=np.int32).reshape(-1, 2), corr)


def test_pybind_equals_ctypes(ctx):
    subprocess.check_call(["make", "-s", "-C", HOST])
    sys.path.insert(0, os.path.join(HOST, "python"))
    import teaserpp_python as tpp
    probs = [problem(K, seed=s, n=n)[:3] for K, s, n in ((600, 21, 800), (2, 22, 64), (3000, 23, 1500))]
    rng = np.random.default_rng(24)
    sn = [rng.normal(size=(len(q[0]), 3)).astype(np.float32) for q in probs]
    dn = [rng.normal(size=(len(q[1]), 3)).astype(np.float32) for q in probs]
    p = prm(0.01, check_edge_length=1, check_normal=1, normal_angle_threshold=1.2)
    rs = tpp.RANSACRegistration(0.01, check_edge_length=True, check_normal=True, normal_angle_threshold=1.2)
    seeds = [5, 6, 2 ** 64 - 1]
    res, info, ev = ctx.ransac_batch([q[0] for q in probs], [q[1] for q in probs], [q[2] for q in probs], p,
                                     seeds=seeds, src_normals=sn, dst_normals=dn)
    got = rs.register_batch([q[0] for q in probs], [q[1] for q in probs], [q[2] for q in probs], seeds, sn, dn)
    for b in range(3):
        _same_record(got[b], res[b], info[b], ev[b])
        one = rs.register(probs[b][0], probs[b][1], probs[b][2], seeds[b], sn[b], dn[b])
        _same_record(one, res[b], info[b], ev[b])
    clouds, pairs = sequence([500, 600, 550], seed=29)
    pr = tpp.register_cloud_pairs_ransac(clouds, pairs, 0.02, RN, RF, *EXAMPLE, tuple_seed=11, ransac_seeds=[3, 4],
                                         check_edge_length=True)
    tseeds = [(11 + 0x9E3779B97F4A7C15 * q) % (1 << 64) for q in range(len(pairs))]
    status, corr, scales, cres, cinfo = ctx.register_cloud_pairs_ransac(
        clouds, pairs, prm(0.02, check_edge_length=1), RN, RF, *EXAMPLE, tuple_seeds=tseeds, ransac_seeds=[3, 4])
    for q in range(len(pairs)):
        assert pr[q]["status"] == status[q] and pr[q]["registered"] == (status[q] == 0)
        assert np.array_equal(np.array(pr[q]["correspondences"], dtype=np.int32).reshape(-1, 2), corr[q])
        assert np.float32(pr[q]["global_scale"]) == np.float32(scales[q])
        if status[q] == 0:
            _same_record(pr[q]["ransac"], cres[q], cinfo[q], None)
