"""Multi-scale ICP on the device (run on an H100: `pytest -m gpu`).

tzr_icp_multiscale_batch against the chain of public calls it is defined by (voxel_downsample(_colors)_batch,
estimate_normals_batch, the method's ICP batch entry, seeded scale after scale), byte for byte: every method, with and
without a robust kernel, lambda 0.968 and 1, on a scene with a target shared by two pairs, a cloud no pair uses, clouds
whose downsampled sizes cross the 1024-point ICP route and the 4096-point normals route between scales, and a seed with
scale != 1.  Then the schedule's edges (one scale, a dense scale, max_iteration 0, an all-NaN cloud, a voxel grid that
fails Open3D's INT_MAX check, normals that overflow), the information matrices, the launch count, every refusal and the
retained solve.
"""
import ctypes as C
import importlib
import os
import subprocess
import sys

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from test_gpu_icp import PAIR_FLAGS, _sequence, surface

capi = importlib.import_module("teaser-plusplus_b200.capi")

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "teaser-plusplus_b200", "host")
CSRC = os.path.join(ROOT, "teaser-plusplus_b200", "csrc")

CENTER = (0.5, -0.2, 2.0)
# the tutorial's shape: three voxel sizes, distance 1.5 v, normals at 2 v, fewer iterations at the finer scales
SCHEDULE = [dict(voxel_size=v, max_correspondence_distance=1.5 * v, max_iteration=it)
            for v, it in ((0.08, 8), (0.04, 5), (0.02, 3))]
METHODS = ["point_to_point", "point_to_plane", "generalized", "colored"]
HUBER = ("huber", 0.02)


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.set_flags(0)
    c.close()


def texture(p):
    return np.stack([0.5 + 0.4 * np.sin(4 * p[:, 0]), 0.5 + 0.4 * np.cos(3 * p[:, 1]),
                     0.5 + 0.3 * np.sin(2 * (p[:, 0] + p[:, 1]))], axis=1)


def moved(pts, seed, deg=2.0):
    rng = np.random.default_rng(seed)
    R = Rotation.from_rotvec(rng.normal(size=3) * np.radians(deg) / np.sqrt(3)).as_matrix()
    c = np.asarray(CENTER)
    t = c - R @ c + rng.normal(size=3) * 0.01
    return (pts @ R.T + t), R, t


def scene():
    """c0 (3000 points: crosses 1024 at v = 0.04), c1 (12000: crosses 4096 at v = 0.02, the target of two pairs), c2 (a
    moved resample of c0's surface), c3 (no pair uses it); colours from a texture on the unmoved surface."""
    rng = np.random.default_rng(7)
    base = [surface(rng, 3000), surface(rng, 12000), surface(rng, 3000), surface(rng, 2000)]
    cols = [(texture(p) + 0.01 * rng.standard_normal((len(p), 3))).astype(np.float32) for p in base]
    c1, R1, t1 = moved(base[1], 1)
    c2, R2, t2 = moved(base[2], 2)
    clouds = [base[0].astype(np.float32), c1.astype(np.float32), c2.astype(np.float32), base[3].astype(np.float32)]
    pairs = [(0, 1), (2, 1), (1, 2)]
    # near-truth seeds, one with scale 1.02; (1, 2) maps c1 to c2: T2 T1^-1
    inits = [dict(scale=1.0, rotation=R1 @ Rotation.from_rotvec([0.01, -0.02, 0.01]).as_matrix(), translation=t1 + 0.01),
             dict(scale=1.02, rotation=R1 @ R2.T, translation=t1 - R1 @ R2.T @ t2 - 0.005),
             dict(scale=1.0, rotation=R2 @ R1.T, translation=t2 - R2 @ R1.T @ t1)]
    return clouds, cols, pairs, inits


def scale_list(schedule):
    return [capi.icp_scale(s) for s in schedule]


def carry(pose):
    r = np.zeros(1, dtype=capi.ICP_RESULT_DTYPE)[0]
    s = capi.similarity(pose)
    r["transform"]["scale"] = s.scale
    r["transform"]["rotation"] = s.rotation[:]
    r["transform"]["translation"] = s.translation[:]
    return r


def chain(ctx, method, schedule, clouds, pairs, inits, colors=None, kernel=None, lam=0.968, eps=1e-3, info=False):
    """The public calls, scale by scale.  Returns (records (P,S), n_down (K,S), status (K,S), information, counts,
    launches without the information call).  A cloud with no points at a scale sits out its normals; a pair using one
    carries its pose; a cloud whose normals overflow keeps the normals the batch wrote."""
    P, K, S = len(pairs), len(clouds), len(schedule)
    rec = np.zeros((P, S), dtype=capi.ICP_RESULT_DTYPE)
    n_down, status = np.zeros((K, S), np.int32), np.zeros((K, S), np.int32)
    poses = list(inits)
    launches = 0
    down_pts = None
    for s, sc in enumerate(scale_list(schedule)):
        l0 = ctx.kernel_launches()
        if sc.voxel_size > 0:
            out = ctx.voxel_downsample_batch(clouds, sc.voxel_size, colors=colors)
            down_pts, down_col = (out if colors is not None else (out, None))
        else:
            down_pts, down_col = list(clouds), colors
        n_down[:, s] = [len(p) for p in down_pts]
        live = [c for c in range(K) if len(down_pts[c]) > 0]
        nrm = {}
        if method != "point_to_point":
            try:
                got = ctx.estimate_normals_batch([down_pts[c] for c in live], sc.normal_search_radius)
            except capi.TzrError as e:
                got = e.result
                for k, c in enumerate(live):
                    status[c, s] = e.status[k]
            nrm = dict(zip(live, got))
        act = [p for p, (a, b) in enumerate(pairs) if len(down_pts[a]) and len(down_pts[b])]
        kw = dict(max_iteration=sc.max_iteration, relative_fitness=sc.relative_fitness, relative_rmse=sc.relative_rmse)
        if act:
            src = [down_pts[pairs[p][0]] for p in act]
            dst = [down_pts[pairs[p][1]] for p in act]
            ini = [poses[p] for p in act]
            r = sc.max_correspondence_distance
            if method == "point_to_point":
                res, _ = ctx.icp_batch(src, dst, r, ini, **kw)
            elif method == "point_to_plane":
                res, _ = ctx.icp_point_to_plane_batch(src, dst, [nrm[pairs[p][1]] for p in act], r, ini, kernel=kernel,
                                                      **kw)
            elif method == "generalized":
                res, _ = ctx.icp_generalized_batch(src, dst, [nrm[pairs[p][0]] for p in act],
                                                   [nrm[pairs[p][1]] for p in act], r, ini, epsilon=eps, kernel=kernel,
                                                   **kw)
            else:
                res, _ = ctx.icp_colored_batch(src, dst, [nrm[pairs[p][1]] for p in act],
                                               [down_col[pairs[p][0]] for p in act], [down_col[pairs[p][1]] for p in act],
                                               r, ini, lambda_geometric=lam, kernel=kernel, **kw)
            for k, p in enumerate(act):
                rec[p, s] = res[k]
        for p in range(P):
            if p not in act:
                rec[p, s] = carry(poses[p])
            poses[p] = rec[p, s]["transform"]
        launches += ctx.kernel_launches() - l0
    info_m, counts = np.zeros((P, 6, 6)), np.zeros(P, np.int32)
    if info:
        act = [p for p, (a, b) in enumerate(pairs) if len(down_pts[a]) and len(down_pts[b])]
        if act:
            L, cnt = ctx.information_matrix_batch([down_pts[pairs[p][0]] for p in act],
                                                  [down_pts[pairs[p][1]] for p in act],
                                                  [rec[p, S - 1]["transform"] for p in act],
                                                  scale_list(schedule)[-1].max_correspondence_distance)
            info_m[act], counts[act] = L, cnt
    return rec, n_down, status, info_m, counts, launches


def expected_launches(method, schedule, n_down, pairs, info):
    """The header's count: per scale 10 (voxel), the normals pass, 1 store, and with a refined pair 1 load and ICP."""
    total = 0
    S = len(schedule)
    for s, sc in enumerate(scale_list(schedule)):
        nd = n_down[:, s]
        total += 10 if sc.voxel_size > 0 else 0
        if method != "point_to_point" and nd.sum() > 0:
            total += 1 + (4 if nd.max() >= 4096 else 0)
        total += 1
        if any(nd[a] > 0 and nd[b] > 0 for a, b in pairs):
            total += 1 + 2 + 4 * sc.max_iteration + (4 if nd.max() >= 1024 else 0)
            if method == "colored":
                total += 1 + (4 if nd.max() >= 4096 else 0)
            if info and s == S - 1:
                total += 4
    return total


def run(ctx, method, schedule, clouds, pairs, inits, colors=None, **kw):
    return ctx.icp_multiscale(clouds, pairs, schedule, inits, method=method,
                              colors=colors if method == "colored" else None, **kw)


CASES = [("point_to_point", None, 0.968), ("point_to_plane", None, 0.968), ("point_to_plane", HUBER, 0.968),
         ("generalized", None, 0.968), ("generalized", HUBER, 0.968), ("colored", None, 0.968),
         ("colored", HUBER, 0.968), ("colored", None, 1.0), ("colored", HUBER, 1.0)]


@pytest.mark.parametrize("method,kernel,lam", CASES,
                         ids=[f"{m}-{'huber' if k else 'l2'}-{l}" for m, k, l in CASES])
def test_equals_the_public_chain(ctx, method, kernel, lam):
    clouds, cols, pairs, inits = scene()
    colors = cols if method == "colored" else None
    l0 = ctx.kernel_launches()
    rec, n_down, info, cnt = run(ctx, method, SCHEDULE, clouds, pairs, inits, cols, kernel=kernel,
                                 lambda_geometric=lam, information=True)
    launches = ctx.kernel_launches() - l0
    want, nd_want, st_want, info_want, cnt_want, chain_launches = chain(ctx, method, SCHEDULE, clouds, pairs, inits,
                                                                        colors, kernel, lam, info=True)
    assert np.array_equal(n_down, nd_want) and not st_want.any()
    # the routes switch mid-schedule: the targets c1 and c2 are below 1024 at the first scale and c2 crosses it at the
    # second (ICP's grid), c1 crosses 4096 at the third (the normals' and gradients' grid)
    assert n_down[[1, 2], 0].max() < 1024 <= n_down[2, 1] and n_down[:, 1].max() < 4096 <= n_down[1, 2]
    assert rec.tobytes() == want.tobytes()
    assert info.tobytes() == info_want.tobytes() and np.array_equal(cnt, cnt_want)
    assert (rec["n_correspondences"] > 0).all() and (rec["iterations"] > 0).all()
    assert rec[1, 0]["transform"]["scale"] == 1.02
    assert launches == expected_launches(method, SCHEDULE, n_down, pairs, True)
    # the chain's own launches plus a pose load and store per scale and the information's 4 (the grid is reused)
    assert launches == chain_launches + 2 * len(SCHEDULE) + 4


@pytest.mark.parametrize("method", ["point_to_plane", "colored"])
def test_one_scale_equals_the_single_scale_chain(ctx, method):
    clouds, cols, pairs, inits = scene()
    sched = [SCHEDULE[1]]
    rec, n_down = run(ctx, method, sched, clouds, pairs, inits, cols)
    want = chain(ctx, method, sched, clouds, pairs, inits, cols if method == "colored" else None)[0]
    assert rec.shape == (3, 1) and rec.tobytes() == want.tobytes()


@pytest.mark.parametrize("method", METHODS)
def test_dense_scale_and_zero_iterations(ctx, method):
    """A scale at voxel_size 0 (the clouds as given) and one with max_iteration 0, whose record is the pose carried in
    and evaluated."""
    clouds, cols, pairs, inits = scene()
    clouds, cols = [c[:2500] for c in clouds], [c[:2500] for c in cols]
    sched = [dict(voxel_size=0.08, max_correspondence_distance=0.12, max_iteration=4),
             dict(voxel_size=0.0, max_correspondence_distance=0.03, normal_search_radius=0.06, max_iteration=3),
             dict(voxel_size=0.04, max_correspondence_distance=0.06, max_iteration=0)]
    colors = cols if method == "colored" else None
    l0 = ctx.kernel_launches()
    rec, n_down = run(ctx, method, sched, clouds, pairs, inits, cols)
    launches = ctx.kernel_launches() - l0
    want, nd_want = chain(ctx, method, sched, clouds, pairs, inits, colors)[:2]
    assert np.array_equal(n_down[:, 1], [2500, 2500, 2500, 2000]) and np.array_equal(n_down, nd_want)
    assert rec.tobytes() == want.tobytes()
    assert (rec[:, 2]["iterations"] == 0).all() and (rec[:, 2]["n_correspondences"] > 0).all()
    assert rec[:, 2]["transform"].tobytes() == rec[:, 1]["transform"].tobytes()
    assert launches == expected_launches(method, sched, n_down, pairs, False)


@pytest.mark.parametrize("method", ["point_to_point", "generalized", "colored"])
def test_all_nan_cloud_carries_its_pairs(ctx, method):
    clouds, cols, pairs, inits = scene()
    clouds = clouds + [np.full((700, 3), np.nan, dtype=np.float32)]
    cols = cols + [np.full((700, 3), 0.5, dtype=np.float32)]
    pairs = pairs + [(4, 1), (0, 4)]
    inits = inits + [inits[0], inits[2]]
    colors = cols if method == "colored" else None
    rec, n_down = run(ctx, method, SCHEDULE, clouds, pairs, inits, cols)
    assert (n_down[4] == 0).all()
    for p in (3, 4):
        for s in range(len(SCHEDULE)):
            assert rec[p, s].tobytes() == carry(inits[p]).tobytes()
    want = chain(ctx, method, SCHEDULE, clouds[:4], pairs[:3], inits[:3], None if colors is None else colors[:4])[0]
    assert rec[:3].tobytes() == want.tobytes()


def test_voxel_grid_too_large_runs_only_the_voxel_kernels(ctx):
    clouds, cols, pairs, inits = scene()
    far = clouds[3].copy()
    far[17] = (6e7, 0.0, 0.0)  # 0.02 INT_MAX < 6e7 < 0.04 INT_MAX: Open3D's check fails at the finest scale only
    clouds[3] = far
    l0 = ctx.kernel_launches()
    with pytest.raises(capi.TzrError, match="TOO_LARGE|too large") as e:
        run(ctx, "point_to_plane", SCHEDULE, clouds, pairs, inits, information=True)
    assert ctx.kernel_launches() - l0 == 10 * len(SCHEDULE)
    st = e.value.status
    assert st[3, 2] == capi.TZR_ERR_TOO_LARGE and (st[3, :2] == 0).all() and (np.delete(st, 3, 0) == 0).all()
    rec, n_down, info, cnt = e.value.result
    assert not rec.tobytes().strip(b"\0") and not info.any() and not cnt.any()
    assert n_down[3, 2] == 0 and (n_down[:3] > 0).all()


def test_normals_overflow_zeroes_the_pairs_from_that_scale(ctx):
    """A clump of 5000 points inside 1e-3: collapsed by the voxel scale, more than 4096 neighbours at the dense one."""
    clouds, cols, pairs, inits = scene()
    rng = np.random.default_rng(3)
    clump = np.concatenate([clouds[0][:1500], (np.asarray(CENTER) + rng.uniform(0, 1e-3, (5000, 3)))]).astype(np.float32)
    clouds = [clouds[0][:2000], clouds[1][:2000], clump]
    pairs = [(0, 1), (2, 1), (1, 0)]
    inits = [inits[0], inits[0], capi.similarity(None)]
    sched = [dict(voxel_size=0.08, max_correspondence_distance=0.12, max_iteration=3),
             dict(voxel_size=0.0, max_correspondence_distance=0.03, normal_search_radius=0.02, max_iteration=2)]
    with pytest.raises(capi.TzrError) as e:
        run(ctx, "point_to_plane", sched, clouds, pairs, inits, information=True)
    st = e.value.status
    assert st[2, 1] == capi.TZR_ERR_TOO_LARGE and st.sum() == capi.TZR_ERR_TOO_LARGE
    rec, _, info, cnt = e.value.result
    want, _, st_want, info_want, cnt_want, _ = chain(ctx, "point_to_plane", sched, clouds, pairs, inits, info=True)
    assert np.array_equal(st, st_want)
    assert rec[1, 0].tobytes() == want[1, 0].tobytes() and not rec[1, 1].tobytes().strip(b"\0")
    assert rec[[0, 2]].tobytes() == want[[0, 2]].tobytes()
    assert not info[1].any() and cnt[1] == 0
    assert info[[0, 2]].tobytes() == info_want[[0, 2]].tobytes()


def _c_args(clouds, pairs, inits, sched, method=1, eps=1e-3, lam=0.968, kernel=None, colors=None):
    K, P, S = len(clouds), len(pairs), len(sched)
    fp = C.POINTER(C.c_float)
    keep = [np.ascontiguousarray(c, dtype=np.float32) for c in clouds]
    n = np.array([len(c) for c in keep], dtype=np.int32)
    pc = np.ascontiguousarray(pairs, dtype=np.int32)
    res = (capi.IcpResult * (P * S))()
    cols = None if colors is None else (fp * K)(*[c.ctypes.data_as(fp) for c in colors])
    args = [int(method), S, (capi.IcpScale * S)(*sched), K, n.ctypes.data_as(C.POINTER(C.c_int32)),
            (fp * K)(*[c.ctypes.data_as(fp) for c in keep]), cols, P, pc.ctypes.data_as(C.POINTER(C.c_int32)),
            (capi.Similarity * P)(*[capi.similarity(x) for x in inits]), eps, lam,
            None if kernel is None else C.byref(kernel), res, None, None, None, None]
    return args, (keep, n, pc, res)


REFUSED = ["S0", "voxel_negative", "voxel_nan", "distance_zero", "distance_inf", "normal_radius_zero", "iterations",
           "fitness_nan", "pair_index", "seed_nan", "seed_scale", "method", "kernel_point_to_point", "kernel_bad",
           "epsilon", "lambda_nan", "colors_missing", "colors_entry"]


@pytest.mark.parametrize("case", REFUSED)
def test_refusals_launch_nothing(ctx, case):
    clouds, cols, pairs, inits = scene()
    clouds, cols = [c[:300] for c in clouds], [c[:300] for c in cols]
    sched = scale_list(SCHEDULE)
    kw = {}
    if case == "S0":
        sched = sched[:0] + [sched[0]]
    elif case == "voxel_negative":
        sched[1].voxel_size = -0.01
    elif case == "voxel_nan":
        sched[1].voxel_size = float("nan")
    elif case == "distance_zero":
        sched[2].max_correspondence_distance = 0.0
    elif case == "distance_inf":
        sched[0].max_correspondence_distance = float("inf")
    elif case == "normal_radius_zero":
        sched[2].normal_search_radius = 0.0
    elif case == "iterations":
        sched[1].max_iteration = -1
    elif case == "fitness_nan":
        sched[0].relative_fitness = float("nan")
    elif case == "pair_index":
        pairs = pairs + [(0, 4)]
        inits = inits + [inits[0]]
    elif case == "seed_nan":
        inits = [dict(inits[0], translation=[np.nan, 0, 0])] + inits[1:]
    elif case == "seed_scale":
        inits = [dict(inits[0], scale=0.0)] + inits[1:]
    elif case == "method":
        kw["method"] = 4
    elif case == "kernel_point_to_point":
        kw.update(method=0, kernel=capi.robust_kernel(HUBER))
    elif case == "kernel_bad":
        kw["kernel"] = capi.robust_kernel(("huber", 0.0))
    elif case == "epsilon":
        kw.update(method=2, eps=0.0)
    elif case == "lambda_nan":
        kw.update(method=3, lam=float("nan"), colors=cols)
    elif case == "colors_missing":
        kw.update(method=3)
    elif case == "colors_entry":
        kw.update(method=3, colors=cols)
    args, keep = _c_args(clouds, pairs, inits, sched, **kw)
    if case == "S0":
        args[1] = 0
    if case == "colors_entry":
        args[6][2] = None
    l0 = ctx.kernel_launches()
    assert capi.lib().tzr_icp_multiscale_batch(ctx._h, *args) == capi.TZR_ERR_INVALID_ARG
    assert ctx.kernel_launches() == l0
    # the point-to-point method reads no normal radius: the same scales pass there
    if case == "normal_radius_zero":
        args[0] = 0
        assert capi.lib().tzr_icp_multiscale_batch(ctx._h, *args) == capi.TZR_OK


def test_lambda_outside_the_range_is_the_default(ctx):
    clouds, cols, pairs, inits = scene()
    clouds, cols = [c[:2000] for c in clouds], [c[:2000] for c in cols]
    a = run(ctx, "colored", SCHEDULE[:2], clouds, pairs, inits, cols, lambda_geometric=1.5)[0]
    b = run(ctx, "colored", SCHEDULE[:2], clouds, pairs, inits, cols, lambda_geometric=0.968)[0]
    assert a.tobytes() == b.tobytes()


def test_retained_solve_survives(ctx):
    rng = np.random.default_rng(11)
    src = rng.uniform(-1, 1, (200, 3))
    R = Rotation.from_rotvec([0.1, 0.2, -0.1]).as_matrix()
    dst = src @ R.T + 0.3
    dst[:40] = rng.uniform(-1, 1, (40, 3))
    ctx.solve(src, dst, capi.default_params(noise_bound=0.01))
    before = [m.tobytes() for m in ctx.last_inliers(0)]
    info0 = ctx.last_graph_info()
    clouds, cols, pairs, inits = scene()
    run(ctx, "colored", SCHEDULE, [c[:3000] for c in clouds], pairs, inits, [c[:3000] for c in cols])
    assert [m.tobytes() for m in ctx.last_inliers(0)] == before
    assert ctx.last_graph_info() == info0


def test_seeded_from_register_cloud_pairs(ctx):
    """register_cloud_pairs' solutions array seeds the call directly, as the same seeds given one by one and as the
    chain seeded with them."""
    clouds = _sequence([1500, 1800, 1200, 1600], seed=5)
    pairs = [(0, 1), (1, 2), (2, 3)]
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=0, rotation_cost_threshold=1e-12)
    sols = ctx.register_cloud_pairs(clouds, pairs, prm, **PAIR_FLAGS)[0]
    keep = np.flatnonzero(sols["valid"])
    assert sols.dtype == capi.SOLUTION_DTYPE and len(keep) >= 2
    pairs, sols = [pairs[k] for k in keep], sols[keep]
    sched = [dict(voxel_size=0.08, max_correspondence_distance=0.12, max_iteration=6),
             dict(voxel_size=0.04, max_correspondence_distance=0.06, max_iteration=4)]
    rec = run(ctx, "point_to_plane", sched, clouds, pairs, sols)[0]
    listed = run(ctx, "point_to_plane", sched, clouds, pairs, [dict(scale=x["scale"], rotation=x["rotation"],
                                                                     translation=x["translation"]) for x in sols])[0]
    want = chain(ctx, "point_to_plane", sched, clouds, pairs, list(sols))[0]
    assert rec.tobytes() == listed.tobytes() == want.tobytes()
    assert (rec["n_correspondences"] > 0).all()
    mats = np.stack([np.eye(4)] * len(sols))
    mats[:, :3, :3] = sols["rotation"].reshape(-1, 3, 3).transpose(0, 2, 1)
    mats[:, :3, 3] = sols["translation"]
    by_matrix = run(ctx, "point_to_plane", sched, clouds, pairs, mats)[0]
    assert by_matrix.tobytes() == run(ctx, "point_to_plane", sched, clouds, pairs, list(mats))[0].tobytes()


@pytest.mark.parametrize("method", ["point_to_point", "point_to_plane", "generalized"])
def test_colours_are_ignored_by_the_geometric_methods(ctx, method):
    clouds, cols, pairs, inits = scene()
    clouds, cols = [c[:2000] for c in clouds], [c[:2000] for c in cols]
    a = ctx.icp_multiscale(clouds, pairs, SCHEDULE[:2], inits, method=method)[0]
    b = ctx.icp_multiscale(clouds, pairs, SCHEDULE[:2], inits, method=method, colors=cols)[0]
    assert a.tobytes() == b.tobytes()


def test_counts_alone_run_the_information_pass(ctx):
    clouds, cols, pairs, inits = scene()
    clouds = [c[:3000] for c in clouds]
    rec, _, info, cnt = run(ctx, "point_to_plane", SCHEDULE, clouds, pairs, inits, information=True)
    assert (cnt > 0).all()
    args, keep = _c_args(clouds, pairs, inits, scale_list(SCHEDULE))
    counts = np.full(len(pairs), -1, dtype=np.int32)
    args[-1] = counts.ctypes.data_as(C.POINTER(C.c_int32))
    assert capi.lib().tzr_icp_multiscale_batch(ctx._h, *args) == capi.TZR_OK
    assert np.array_equal(counts, cnt)
    assert bytes(keep[3]) == rec.tobytes()


# ---- façades -----------------------------------------------------------------------------------------------------------
def test_cpp_facade_equals_the_c_abi(tmp_path):
    """MultiScaleICP::refineBatch against tzr_icp_multiscale_batch (tests/cpp/icp_multiscale_test.cc)."""
    subprocess.check_call(["make", "-s", "-C", HOST])
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    exe = str(tmp_path / "icp_multiscale_test")
    subprocess.check_call([cxx, "-std=c++17", "-O1", "-I", os.path.join(HOST, "include"), "-I",
                           os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "icp_multiscale_test.cc"),
                           "-L", HOST, "-lteaser_registration", "-L", CSRC, "-lteaser_b200",
                           f"-Wl,-rpath,{HOST}:{CSRC}", "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr


@pytest.mark.parametrize("method,kernel", [("point_to_plane", HUBER), ("generalized", None), ("colored", HUBER)])
def test_pybind_equals_ctypes(ctx, method, kernel):
    subprocess.check_call(["make", "-s", "-C", HOST])
    sys.path.insert(0, os.path.join(HOST, "python"))
    import teaserpp_python as tpp
    clouds, cols, pairs, inits = scene()
    clouds, cols = [c[:4000] for c in clouds], [c[:4000] for c in cols]
    colors = cols if method == "colored" else None
    want, n_down, info, cnt = run(ctx, method, SCHEDULE, clouds, pairs, inits, cols, kernel=kernel,
                                  lambda_geometric=0.9, information=True)
    seeds = []
    for x in inits:
        s = tpp.RegistrationSolution()
        s.scale = x["scale"]
        s.rotation = np.asarray(x["rotation"], dtype=np.float64)
        s.translation = np.asarray(x["translation"], dtype=np.float64)
        seeds.append(s)
    tk = tpp.RobustKernel() if kernel is None else tpp.RobustKernel(*kernel)
    icp = tpp.MultiScaleICP(SCHEDULE, method=method, lambda_geometric=0.9, kernel=tk)
    got = icp.refine_batch(clouds, pairs, seeds, colors=colors, information=True)
    fn = tpp.multiscale_icp(clouds, pairs, [(d["voxel_size"], d["max_correspondence_distance"], d["max_iteration"])
                                            for d in SCHEDULE], seeds, method=method, colors=colors,
                            lambda_geometric=0.9, kernel=tk, information=True)
    for res in (got, fn):
        assert not res["too_large"] and np.array_equal(np.asarray(res["n_down"]), n_down)
        assert np.array_equal(np.asarray(res["status"]), np.zeros_like(n_down))
        for p in range(len(pairs)):
            for s in range(len(SCHEDULE)):
                r, w = res["records"][p][s], want[p, s]
                assert np.asarray(r["solution"].rotation).T.tobytes() == w["transform"]["rotation"].tobytes()
                assert np.asarray(r["solution"].translation).ravel().tobytes() == w["transform"]["translation"].tobytes()
                assert (r["solution"].scale, r["fitness"], r["inlier_rmse"], r["iterations"], r["converged"]) == \
                    (w["transform"]["scale"], w["fitness"], w["inlier_rmse"], w["iterations"], bool(w["converged"]))
            assert np.asarray(res["information"][p]).tobytes() == info[p].tobytes()
        assert list(res["info_counts"]) == list(cnt)
