"""tzr_icp / tzr_icp_batch on the device (run on an H100: `pytest -m gpu`).

Against the numpy restatement (tests/icp_reference.py) on scans of a wavy surface whose decisions stay clear of ties;
the brute-force and grid nearest-neighbour routes bit for bit; the edge rules; a ragged batch against each problem alone,
bit for bit; the retained solve left intact; that refinement brings perturbed seeds closer to ground truth; the chained
entry tzr_register_cloud_pairs_icp against register_cloud_pairs followed by icp_batch; the C++ and pybind façades.
"""
import importlib

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import icp_reference as ref

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


def surface(rng, n, offset=(0.5, -0.2, 2.0)):
    uv = rng.uniform(-1, 1, size=(n, 2))
    pts = np.stack([uv[:, 0], uv[:, 1], 0.3 * np.sin(3 * uv[:, 0]) * np.cos(2 * uv[:, 1])], axis=1)
    return pts + rng.normal(scale=0.003, size=pts.shape) + np.asarray(offset)


def scan_pair(seed, ns, nd, offset=(0.5, -0.2, 2.0)):
    """Two scans of one surface: the source, and 2/3 of its points plus new samples moved by a ground-truth (R, t)."""
    rng = np.random.default_rng(seed)
    src = surface(rng, ns, offset)
    keep = min(ns, nd - nd // 3)
    pts = np.concatenate([src[:keep], surface(rng, nd - keep, offset)])[rng.permutation(nd)]
    R = Rotation.from_rotvec(rng.normal(size=3) * 0.03).as_matrix()
    c = np.asarray(offset)
    t = c - R @ c + rng.normal(size=3) * 0.02
    dst = pts @ R.T + t
    return src.astype(np.float32), dst.astype(np.float32), R, t


def perturbed(R, t, seed, deg=3.0, shift=2 * R_CORR, center=(0.5, -0.2, 2.0)):
    rng = np.random.default_rng(seed + 1000)
    a = rng.normal(size=3)
    dR = Rotation.from_rotvec(a / np.linalg.norm(a) * np.radians(deg)).as_matrix()
    d = rng.normal(size=3)
    # rotate about the image m of the source's centre, so that the seed's displacement there is the shift alone
    m = R @ np.asarray(center) + t
    return dict(scale=1.0, rotation=dR @ R, translation=dR @ (t - m) + m + d / np.linalg.norm(d) * shift)


def as_bytes(res):
    return np.ascontiguousarray(res).tobytes()


def run_ref(src, dst, init, **kw):
    return ref.icp(src, dst, R_CORR, s=init["scale"], R=np.asarray(init["rotation"]), t=init["translation"], trace=True,
                   **kw)


@pytest.mark.parametrize("seed,ns,nd", [(11, 1500, 1800), (12, 3000, 2500)])
def test_against_reference(ctx, seed, ns, nd):
    src, dst, R, t = scan_pair(seed, ns, nd)
    init = perturbed(R, t, seed)
    want = run_ref(src, dst, init)
    for m in want["margins"]:
        assert m["tie"] > 1e-9 and m["bound"] > 1e-9, m
    got, corr = ctx.icp(src, dst, R_CORR, init=init)
    assert want["iterations"] > 2
    assert (got["iterations"], got["converged"], got["n_correspondences"]) == \
        (want["iterations"], want["converged"], want["n_correspondences"])
    assert got["fitness"] == want["fitness"]
    assert np.array_equal(corr, want["corr"])
    np.testing.assert_allclose(got["R"], want["R"], rtol=0, atol=1e-10)
    np.testing.assert_allclose(got["t"], want["t"], rtol=0, atol=1e-10)
    assert abs(got["inlier_rmse"] - want["inlier_rmse"]) <= 1e-12 * want["inlier_rmse"]
    assert got["scale"] == 1.0


def _both_routes(ctx, srcs, dsts, inits, **kw):
    out = []
    for flag in (BRUTE, GRID):
        ctx.set_flags(flag)
        try:
            out.append(ctx.icp_batch(srcs, dsts, R_CORR, inits, **kw))
        finally:
            ctx.set_flags(0)
    (ra, ca), (rb, cb) = out
    assert as_bytes(ra) == as_bytes(rb)
    assert all(np.array_equal(a, b) for a, b in zip(ca, cb))
    return ra, ca


def test_routes_bit_identical_on_scans(ctx):
    src, dst, R, t = scan_pair(21, 3000, 3000)
    res, _ = _both_routes(ctx, [src], [dst], [perturbed(R, t, 21)])
    assert res[0]["iterations"] > 2 and res[0]["n_correspondences"] > 1000
    # the automatic route (grid above 1024 targets) gives the same bits
    auto, _ = ctx.icp_batch([src], [dst], R_CORR, [perturbed(R, t, 21)])
    assert as_bytes(auto) == as_bytes(res)


def test_routes_on_cell_edges_bounds_ties_and_non_finite(ctx):
    r_exact = 0.0625  # exactly representable: d^2 = r^2 exactly for axis-aligned offsets of r
    for rr in (R_CORR, r_exact):
        h = rr * (1 + 1e-5)       # the grid's cell edge
        o = np.float32(-2.0)      # the grid origin: the bounding-box minimum of the finite targets, (-2, -2, -2)
        tg = [[0, 0, 0], [r_exact, 0, 0], [0, 2 * r_exact, 0],           # (0,r,0) lies exactly r from targets 0 and 2
              [1.0, 1.0, 1.0], [1.0 + 0.03, 1.0, 1.0], [1.0 - 0.03, 1.0, 1.0],
              [np.nan, 0, 0], [np.inf, 1, 1], [o, o, o]]
        tg += [[o + m * h, 0.5, 0.5] for m in range(20, 61, 5)]           # targets on cell edges x = o + m h
        dst = np.array(tg, dtype=np.float32)
        qs = [[r_exact, 0, 0], [0, r_exact, 0], [1.0, 1.0, 1.0], [np.nan, 0, 0], [np.inf, 0, 0], [o, o, o + 0.01]]
        qs += [[o + m * h + d, 0.5 + e, 0.5] for m in range(20, 61, 5) for d in (0.0, 0.49 * h, -0.49 * h, 0.99 * h)
               for e in (0.0, 0.3 * h)]
        src = np.array(qs, dtype=np.float32)
        res = []
        for flag in (BRUTE, GRID):
            ctx.set_flags(flag)
            try:
                res.append(ctx.icp_batch([src], [dst], rr, max_iteration=0))
            finally:
                ctx.set_flags(0)
        assert as_bytes(res[0][0]) == as_bytes(res[1][0])
        assert np.array_equal(res[0][1][0], res[1][1][0])
        want = ref.icp(src, dst, rr, max_iteration=0)
        assert np.array_equal(res[0][1][0], want["corr"])
        corr = dict(map(tuple, want["corr"]))
        assert corr[0] == 1 and corr[2] == 3      # d = 0 to the coinciding target
        assert 3 not in corr and 4 not in corr    # non-finite queries
        if rr == r_exact:
            assert 1 not in corr                  # exactly r from its two nearest targets: strict bound, no match
        assert sum(1 for k in corr if k >= 6) > 20  # most edge queries match an edge target


def test_query_outside_the_grid_range_scans_its_targets(ctx):
    """A finite source point more than 2^32 cells from the grid's origin is searched by brute force over its
    problem's targets (the query-side guard), with the grid built for the rest of the cloud."""
    src, dst, R, t = scan_pair(33, 1500, 1500)
    src = np.concatenate([src, np.array([[1e12, 0, 0], [-1e12, 5, 5]], dtype=np.float32)])
    init = perturbed(R, t, 33)
    res, corr = _both_routes(ctx, [src], [dst], [init])
    want = run_ref(src, dst, init)
    assert res[0]["iterations"] == want["iterations"] and np.array_equal(corr[0], want["corr"])
    assert corr[0][-1, 0] < 1500  # the far points match nothing


def test_equidistant_targets_lowest_index(ctx):
    dst = np.array([[0.02, 0, 0], [-0.02, 0, 0], [0, 0.02, 0], [0, -0.02, 0]], dtype=np.float32)
    src = np.zeros((1, 3), dtype=np.float32)
    for flag in (BRUTE, GRID):
        ctx.set_flags(flag)
        try:
            _, corr = ctx.icp(src, dst[::-1].copy(), R_CORR, max_iteration=0)
            assert corr.tolist() == [[0, 0]]
        finally:
            ctx.set_flags(0)


def test_far_point_forces_grid_fallback(ctx):
    src, dst, R, t = scan_pair(31, 1500, 1500)
    dst = np.concatenate([dst, np.array([[1e9, 0, 0]], dtype=np.float32)])
    init = perturbed(R, t, 31)
    res, _ = _both_routes(ctx, [src], [dst], [init])
    want = run_ref(src, dst, init)
    assert res[0]["iterations"] == want["iterations"] and res[0]["n_correspondences"] == want["n_correspondences"]


def test_clouds_farther_apart_than_r(ctx):
    src, dst, _, _ = scan_pair(41, 500, 500)
    got, corr = ctx.icp(src, dst + np.float32(10.0), R_CORR)
    assert (got["iterations"], got["converged"], got["n_correspondences"]) == (1, True, 0)
    assert got["fitness"] == 0.0 and got["inlier_rmse"] == 0.0 and corr.shape == (0, 2)
    np.testing.assert_array_equal(got["R"], np.eye(3))
    np.testing.assert_array_equal(got["t"], np.zeros(3))


@pytest.mark.parametrize("k", [1, 2])
def test_one_or_two_correspondences_translate(ctx, k):
    dst = np.array([[0, 0, 0], [1, 0, 0], [5, 5, 5]], dtype=np.float32)
    src = (dst[:k] + np.array([0.01, -0.02, 0.005], dtype=np.float32)).astype(np.float32)
    src = np.concatenate([src, np.array([[9, 9, 9]], dtype=np.float32)])
    got, _ = ctx.icp(src, dst, R_CORR, max_iteration=1)
    want = ref.icp(src, dst, R_CORR, max_iteration=1)
    np.testing.assert_array_equal(got["R"], np.eye(3))
    np.testing.assert_allclose(got["t"], want["t"], rtol=0, atol=1e-15)
    assert got["n_correspondences"] == k and got["fitness"] == want["fitness"]


def test_max_iteration_zero_returns_the_seed(ctx):
    src, dst, R, t = scan_pair(51, 800, 800)
    init = perturbed(R, t, 51, shift=0.2 * R_CORR)
    got, corr = ctx.icp(src, dst, R_CORR, init=init, max_iteration=0)
    want = ref.icp(src, dst, R_CORR, R=init["rotation"], t=init["translation"], max_iteration=0)
    assert got["iterations"] == 0 and not got["converged"]
    assert np.array_equal(got["R"], np.asarray(init["rotation"])) and np.array_equal(got["t"], init["translation"])
    assert got["n_correspondences"] == want["n_correspondences"] > 0
    assert np.array_equal(corr, want["corr"]) and got["fitness"] == want["fitness"]


def test_fixed_scale(ctx):
    src, dst, R, t = scan_pair(61, 1500, 1500)
    s = 0.5
    c = np.array([0.5, -0.2, 2.0])
    dst_s = (s * (dst.astype(np.float64) - c) + c).astype(np.float32)  # the target shrunk about c by s
    init = dict(scale=s, rotation=R, translation=s * t + (1 - s) * c)
    got, _ = ctx.icp(src, dst_s, R_CORR, init=init)
    want = run_ref(src, dst_s, init)
    assert got["scale"] == s
    assert got["iterations"] == want["iterations"] and got["n_correspondences"] == want["n_correspondences"]
    np.testing.assert_allclose(got["R"], want["R"], atol=1e-10)
    np.testing.assert_allclose(got["t"], want["t"], atol=1e-10)


def test_large_offset_as_accurate_as_at_the_origin(ctx):
    """The same problem at the origin and at 1e5: the ground-truth error at 1e5 is no worse than twice the error at the
    origin (or 0.05 degrees and 1e-3, whichever is larger).  Measured on an H100: 1.8e-2 degrees and 1.7e-4 at the
    origin, 7.2e-3 degrees and 1.6e-4 at 1e5, although the float coordinates there are rounded to 2^-7 ~ 0.008."""
    errs = []
    for off in ((0.0, 0.0, 0.0), (1e5, -1e5, 5e4)):
        src, dst, R, t = scan_pair(71, 3000, 3000, offset=off)
        init = perturbed(R, t, 71, deg=2.0, shift=R_CORR, center=off)
        got, _ = ctx.icp(src, dst, R_CORR, init=init)
        ang = np.degrees(Rotation.from_matrix(got["R"] @ R.T).magnitude())
        c = np.asarray(off)
        errs.append((ang, np.linalg.norm((got["R"] @ c + got["t"]) - (R @ c + t)), got["n_correspondences"]))
    (a0, t0, n0), (a1, t1, n1) = errs
    print(f"origin: {a0:.2e} deg {t0:.2e}; offset 1e5: {a1:.2e} deg {t1:.2e}")
    assert n0 > 1000 and n1 > 1000
    assert a1 <= max(2 * a0, 0.05) and t1 <= max(2 * t0, 1e-3), errs


def _ragged_problems():
    probs = []
    for k, (ns, nd) in enumerate([(1, 1), (3, 3), (1000, 1000), (20000, 20000), (1000, 1200)]):
        if ns >= 500:
            src, dst, R, t = scan_pair(80 + k, ns, nd)
            init = perturbed(R, t, 80 + k, deg=2.0, shift=R_CORR)
        else:
            rng = np.random.default_rng(80 + k)
            src = rng.uniform(0, 0.03, (ns, 3)).astype(np.float32)
            dst = (src + rng.normal(scale=0.005, size=src.shape)).astype(np.float32)
            init = None
        probs.append((src, dst, init))
    nan_src, nan_dst, _, _ = scan_pair(90, 600, 600)
    nan_src[::7] = np.nan
    nan_dst[::5, 1] = np.inf
    probs.append((nan_src, nan_dst, None))
    far_src, far_dst, _, _ = scan_pair(91, 300, 300)
    probs.append((far_src, far_dst + np.float32(50), None))
    return probs


def test_batch_equals_single_forward_and_reverse(ctx):
    probs = _ragged_problems()
    singles = [ctx.icp_batch([s], [d], R_CORR, None if i is None else [i]) for s, d, i in probs]
    for order in (list(range(len(probs))), list(reversed(range(len(probs))))):
        S = [probs[k][0] for k in order]
        D = [probs[k][1] for k in order]
        I = [probs[k][2] for k in order]
        res, corr = ctx.icp_batch(S, D, R_CORR, I)
        for j, k in enumerate(order):
            assert as_bytes(res[j:j + 1]) == as_bytes(singles[k][0]), k
            assert np.array_equal(corr[j], singles[k][1][0]), k
    # the far pair and the large one behave as documented
    assert singles[-1][0][0]["n_correspondences"] == 0 and singles[-1][0][0]["iterations"] == 1
    assert singles[3][0][0]["n_correspondences"] > 10000


def test_single_call_equals_batch_of_one(ctx):
    src, dst, R, t = scan_pair(95, 2000, 2000)
    init = perturbed(R, t, 95)
    got, corr = ctx.icp(src, dst, R_CORR, init=init)
    res, corrs = ctx.icp_batch([src], [dst], R_CORR, [init])
    one = capi.icp_result_dict(res[0])
    assert all(np.array_equal(got[k], one[k]) for k in one) and np.array_equal(corr, corrs[0])


def test_retained_solve_survives_icp(ctx):
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
    ctx.icp(s, d, R_CORR, init=perturbed(Rg, tg, 97))
    after = ctx.last_inliers(0)
    assert all(np.array_equal(a, b) for a, b in zip(before, after))
    cert_after = ctx.certify_last(noise_bound=0.02)
    assert cert_before[0]["best_suboptimality"] == cert_after[0]["best_suboptimality"]
    assert np.array_equal(cert_before[0]["suboptimality_traj"], cert_after[0]["suboptimality_traj"])


def test_launch_count_does_not_depend_on_B(ctx):
    src, dst, R, t = scan_pair(99, 2000, 2000)
    counts = []
    for B in (1, 5):
        l0 = ctx.kernel_launches()
        ctx.icp_batch([src] * B, [dst] * B, R_CORR, [perturbed(R, t, 99)] * B, max_iteration=7)
        counts.append(ctx.kernel_launches() - l0)
    assert counts == [4 + 2 + 4 * 7] * 2


def test_refinement_improves_perturbed_seeds(ctx):
    better, total = 0, 0
    for k in range(8):
        src, dst, R, t = scan_pair(200 + k, 2500, 2500)
        init = perturbed(R, t, 200 + k, deg=4.0, shift=2 * R_CORR)
        got, _ = ctx.icp(src, dst, R_CORR, init=init, max_iteration=100)
        c = np.array([0.5, -0.2, 2.0])
        e0 = np.degrees(Rotation.from_matrix(np.asarray(init["rotation"]) @ R.T).magnitude())
        e1 = np.degrees(Rotation.from_matrix(got["R"] @ R.T).magnitude())
        d0 = np.linalg.norm(np.asarray(init["rotation"]) @ c + init["translation"] - (R @ c + t))
        d1 = np.linalg.norm(got["R"] @ c + got["t"] - (R @ c + t))
        better += (e1 < e0) and (d1 < d0)
        total += 1
    print(f"refinement lowered both errors for {better} of {total} pairs")
    assert better >= total // 2 + 1


@pytest.mark.parametrize("case", ["r_zero", "r_negative", "r_nan", "r_inf", "iter_negative", "B_zero", "ns_zero",
                                  "nd_zero", "scale_zero", "rotation_nan"])
def test_argument_checks_with_a_context(ctx, case):
    """Each malformed call is refused by its own check (a real context here, so no earlier check can answer)."""
    import ctypes as C
    L = capi.lib()
    p = capi.icp_params(0.1)
    B, ns, nd = 2, 4, 4
    init = (capi.Similarity * 2)(capi.similarity(None), capi.similarity(None))
    if case == "r_zero":
        p.max_correspondence_distance = 0.0
    elif case == "r_negative":
        p.max_correspondence_distance = -1.0
    elif case == "r_nan":
        p.max_correspondence_distance = float("nan")
    elif case == "r_inf":
        p.max_correspondence_distance = float("inf")
    elif case == "iter_negative":
        p.max_iteration = -1
    elif case == "B_zero":
        B = 0
    elif case == "ns_zero":
        ns = 0
    elif case == "nd_zero":
        nd = 0
    elif case == "scale_zero":
        init[1].scale = 0.0
    elif case == "rotation_nan":
        init[1].rotation[4] = float("nan")
    x = np.zeros((4, 3), dtype=np.float32)
    fp, i32p = C.POINTER(C.c_float), C.POINTER(C.c_int32)
    n_s = np.array([4, ns], dtype=np.int32)
    n_d = np.array([nd, 4], dtype=np.int32)
    res = (capi.IcpResult * 2)()
    pts = (fp * 2)(x.ctypes.data_as(fp), x.ctypes.data_as(fp))
    assert L.tzr_icp_batch(ctx._h, C.byref(p), B, n_s.ctypes.data_as(i32p), pts, n_d.ctypes.data_as(i32p), pts, init,
                           res, None) == capi.TZR_ERR_INVALID_ARG
    # the well-formed call runs
    good = capi.icp_params(0.1)
    ok_init = (capi.Similarity * 2)(capi.similarity(None), capi.similarity(None))
    four = np.array([4, 4], dtype=np.int32)
    assert L.tzr_icp_batch(ctx._h, C.byref(good), 2, four.ctypes.data_as(i32p), pts, four.ctypes.data_as(i32p), pts,
                           ok_init, res, None) == 0


# ---- the chained entry: register_cloud_pairs, then ICP of every valid solved pair, in one call ----------------------
RN, RF = 0.1, 0.15
PAIR_FLAGS = dict(normal_search_radius=RN, fpfh_search_radius=RF, use_absolute_scale=False, use_crosscheck=True,
                  use_tuple_test=False)


def _sequence(sizes, seed):
    rng = np.random.default_rng(seed)
    clouds = [surface(rng, sizes[0]).astype(np.float32)]
    for n in sizes[1:]:
        prev = clouds[-1].astype(np.float64)
        keep = min(len(prev), n - n // 3)
        pts = np.concatenate([prev[:keep], surface(rng, n - keep)])[rng.permutation(n)]
        R = Rotation.from_rotvec(rng.normal(size=3) * 0.03).as_matrix()
        clouds.append((pts @ R.T + [0.04, 0.0, 0.0]).astype(np.float32))
    return clouds


def _retained(ctx, S):
    masks = [tuple(m.tobytes() for m in ctx.last_inliers(k)) for k in range(S)]
    cert = ctx.certify_last(noise_bound=0.02, max_iterations=5)
    return masks, [(c["status"], c["best_suboptimality"], c["suboptimality_traj"].tobytes()) for c in cert]


@pytest.mark.parametrize("estimate_scaling", [0, 1])
def test_chained_entry_equals_the_chain(ctx, estimate_scaling):
    clouds = _sequence([600, 1500, 500, 700], seed=5)
    clouds.append((clouds[0] + np.float32(40.0)).astype(np.float32))  # a far copy: refined from a far seed
    clouds.append(clouds[2][:2].copy())  # two points: no normals, so at best a degenerate, unrefined pair
    pairs = [(0, 1), (1, 2), (2, 3), (3, 1), (1, 0), (0, 4), (5, 2)]
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=estimate_scaling, rotation_cost_threshold=1e-12)
    l0 = ctx.kernel_launches()
    plain = ctx.register_cloud_pairs(clouds, pairs, prm, **PAIR_FLAGS)
    l1 = ctx.kernel_launches()
    S = int((plain[2] >= 0).sum())
    ret_plain = _retained(ctx, S)
    l2 = ctx.kernel_launches()
    chained = ctx.register_cloud_pairs_icp(clouds, pairs, prm, R_CORR, max_iteration=40, **PAIR_FLAGS)
    l3 = ctx.kernel_launches()
    sols_a, sols_b = plain[0], chained[0]
    stage = capi.SOLUTION_DTYPE.fields["stage_ms"][1]
    for a, b in zip(sols_a, sols_b):
        assert a.tobytes()[:stage] == b.tobytes()[:stage]
    assert np.array_equal(plain[1], chained[1]) and np.array_equal(plain[2], chained[2])
    assert all(np.array_equal(a, b) for a, b in zip(plain[3], chained[3]))
    assert all(np.array_equal(a, b) for a, b in zip(plain[4], chained[4]))
    assert plain[5] == chained[5]
    assert _retained(ctx, S) == ret_plain
    icp_res = chained[6]
    refined = [p for p in range(len(pairs)) if plain[1][p] == 0 and sols_a[p]["valid"]]
    assert len(refined) >= 3
    for p in range(len(pairs)):
        if p not in refined:
            assert not icp_res[p].tobytes().strip(b"\0"), p
    print(f"refined {len(refined)} of {len(pairs)} pairs")
    seeds = [dict(scale=sols_a[p]["scale"], rotation=sols_a[p]["rotation"], translation=sols_a[p]["translation"])
             for p in refined]
    want, _ = ctx.icp_batch([clouds[pairs[p][0]] for p in refined], [clouds[pairs[p][1]] for p in refined], R_CORR,
                            seeds, max_iteration=40)
    for k, p in enumerate(refined):
        assert icp_res[p].tobytes() == want[k].tobytes(), p
        assert icp_res[p]["transform"]["scale"] == sols_a[p]["scale"]
        assert icp_res[p]["iterations"] >= 1 and icp_res[p]["n_correspondences"] > 0
    # the same launches as register_cloud_pairs, plus the seed launch and the refinement's (clouds of 1024 points and
    # more: the grid build)
    assert (l3 - l2) - (l1 - l0) == 1 + 4 + 2 + 4 * 40


def test_cpp_facade_equals_the_c_abi(tmp_path):
    """PointToPointICP::refine / refineBatch against tzr_icp, and solveCloudPairs(..., PointToPointICP::Params)
    against solveCloudPairs + refineBatch (tests/cpp/icp_test.cc)."""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    host = os.path.join(root, "teaser-plusplus_b200", "host")
    csrc = os.path.join(root, "teaser-plusplus_b200", "csrc")
    subprocess.check_call(["make", "-s", "-C", host])
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    exe = str(tmp_path / "icp_test")
    subprocess.check_call([cxx, "-std=c++17", "-O1", "-I", os.path.join(host, "include"), "-I",
                           os.path.join(root, "include"), os.path.join(root, "tests", "cpp", "icp_test.cc"),
                           "-L", host, "-lteaser_registration", "-L", csrc, "-lteaser_b200",
                           f"-Wl,-rpath,{host}:{csrc}", "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr


def test_pybind_point_to_point_icp(ctx):
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    host = os.path.join(root, "teaser-plusplus_b200", "host")
    subprocess.check_call(["make", "-s", "-C", host])
    sys.path.insert(0, os.path.join(host, "python"))
    import teaserpp_python as tpp
    src, dst, R, t = scan_pair(101, 1500, 1200)
    init = perturbed(R, t, 101)
    seed = tpp.RegistrationSolution()
    seed.scale = 1.0
    seed.rotation = np.asarray(init["rotation"], dtype=np.float64)
    seed.translation = np.asarray(init["translation"], dtype=np.float64)
    icp = tpp.PointToPointICP(R_CORR, max_iteration=30)
    got = icp.refine(src, dst, seed)
    want, corr = ctx.icp(src, dst, R_CORR, init=init)
    assert np.array_equal(np.asarray(got["solution"].rotation), want["R"])
    assert np.array_equal(np.asarray(got["solution"].translation).ravel(), want["t"])
    assert (got["fitness"], got["inlier_rmse"], got["iterations"], got["converged"]) == \
        (want["fitness"], want["inlier_rmse"], want["iterations"], want["converged"])
    assert np.array_equal(np.array(got["correspondences"], dtype=np.int32).reshape(-1, 2), corr)
    batch = icp.refine_batch([src, dst], [dst, src], [seed, seed])
    assert batch[0]["iterations"] == got["iterations"] and batch[0]["fitness"] == got["fitness"]
    # solve_cloud_pairs_icp against the C-ABI's chained entry
    clouds = _sequence([600, 700, 500], seed=9)
    pairs = [(0, 1), (1, 2)]
    solver = tpp.RobustRegistrationSolver(noise_bound=0.01, estimate_scaling=False, rotation_cost_threshold=1e-12)
    res = solver.solve_cloud_pairs_icp(clouds, pairs, R_CORR, normal_search_radius=RN, fpfh_search_radius=RF,
                                       use_absolute_scale=False, use_tuple_test=False, tuple_seed=0)
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=0, rotation_cost_threshold=1e-12)
    c = ctx.register_cloud_pairs_icp(clouds, pairs, prm, R_CORR, **PAIR_FLAGS)
    for p, r in enumerate(res):
        assert r["refined"] == bool(c[1][p] == 0 and c[0][p]["valid"])
        if r["refined"]:
            d = capi.icp_result_dict(c[6][p])
            assert np.array_equal(np.asarray(r["icp"]["solution"].rotation), d["R"])
            assert r["icp"]["iterations"] == d["iterations"] and r["icp"]["fitness"] == d["fitness"]
