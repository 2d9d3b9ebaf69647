"""tzr_voxel_downsample / tzr_voxel_downsample_batch on the device (run on an H100: `pytest -m gpu`).

Unless a test says otherwise, points, counts and voxel_of are compared bit for bit with the numpy restatement
(tests/voxel_reference.py): wavy scans at several voxel sizes, lattices on voxel edges and the division-versus-inverse
point, non-finite points, sparse input, one voxel of 200k points, a large offset, both size limits, a ragged batch
against single calls in both orders, the launch count and the retained solve, the tutorial from raw scans
(downsampling, then register_cloud_pairs_icp), and the C++ and pybind façades.
"""
import ctypes as C
import importlib
import os
import subprocess
import sys

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import test_voxel_cpu as arg_cases
import voxel_reference as ref

capi = importlib.import_module("teaser-plusplus_b200.capi")

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "teaser-plusplus_b200", "host")
CSRC = os.path.join(ROOT, "teaser-plusplus_b200", "csrc")


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


def surface(rng, n, offset=(0.5, -0.2, 2.0), half=1.0):
    uv = rng.uniform(-half, half, size=(n, 2))
    z = 0.3 * np.sin(3 * uv[:, 0]) * np.cos(2 * uv[:, 1]) + 0.25 * np.exp(-((uv[:, 0] - 0.3) ** 2 + (uv[:, 1] + 0.4) ** 2) / 0.05)
    pts = np.stack([uv[:, 0], uv[:, 1], z], axis=1)
    return (pts + rng.normal(scale=0.003, size=pts.shape) + np.asarray(offset)).astype(np.float32)


def check(ctx, pts, v):
    """The device against the reference on one cloud, through the single entry; returns the reference result."""
    want = ref.downsample(pts, v)
    got, trace = ctx.voxel_downsample(pts, v, return_trace=True)
    assert want[2] == ref.TZR_OK
    assert got.shape == want[0].shape and got.tobytes() == want[0].tobytes()
    assert np.array_equal(trace, want[1])
    return want


@pytest.mark.parametrize("seed,n,v", [(1, 1000, 0.01), (2, 20000, 0.05), (3, 100000, 0.05), (4, 300000, 0.02),
                                      (5, 50000, 0.003), (6, 300000, 0.1)])
def test_against_reference(ctx, seed, n, v):
    pts = surface(np.random.default_rng(seed), n)
    want = check(ctx, pts, v)
    per = np.bincount(want[1][want[1] >= 0])
    print(f"n={n} v={v}: {len(want[0])} voxels, {per.min()} to {per.max()} points per voxel")


@pytest.mark.parametrize("v", [0.125, 0.05])
def test_points_on_voxel_edges(ctx, v):
    check(ctx, ref.lattice_on_edges(v, k=12), v)
    rng = np.random.default_rng(7)
    j = rng.integers(-40, 40, size=(5000, 3))
    check(ctx, ((j + 0.5) * v).astype(np.float32), v)


def test_index_is_a_division(ctx):
    pts, v = ref.division_case()
    want = check(ctx, pts, v)
    assert want[1].tolist() == [0, 1, 1, 2]


def test_non_finite_points(ctx):
    rng = np.random.default_rng(8)
    pts = surface(rng, 5000)
    bad = rng.choice(5000, 60, replace=False)
    pts[bad[:20]] = np.nan
    pts[bad[20:40], 1] = np.inf
    pts[bad[40:], 2] = -np.inf
    pts[bad[0]] = [1e30, np.nan, -1e30]  # would stretch the bounds if it counted
    want = check(ctx, pts, 0.05)
    assert (want[1][bad] == -1).all()
    # the bounds ignore them: the finite points alone give the same voxels
    keep = np.setdiff1d(np.arange(5000), bad)
    assert ctx.voxel_downsample(pts[keep], 0.05).tobytes() == want[0].tobytes()
    out, trace = ctx.voxel_downsample(np.full((9, 3), np.nan, dtype=np.float32), 0.05, return_trace=True)
    assert out.shape == (0, 3) and (trace == -1).all()
    outs, traces = ctx.voxel_downsample_batch([np.full((4, 3), np.inf, dtype=np.float32), pts], 0.05, return_trace=True)
    assert outs[0].shape == (0, 3) and (traces[0] == -1).all()
    assert outs[1].tobytes() == want[0].tobytes() and np.array_equal(traces[1], want[1])


def test_sparse_input_comes_back_unchanged(ctx):
    rng = np.random.default_rng(9)
    cells = rng.permutation(np.stack(np.meshgrid(*[np.arange(30)] * 3, indexing="ij"), -1).reshape(-1, 3))
    # jitter in [0, 0.03): the grid starts half a voxel below the smallest coordinate (in [0.2, 0.23)), so every point
    # stays inside its own cell's voxel
    pts = (cells * 0.1 + rng.uniform(0, 0.03, size=cells.shape) + 0.2).astype(np.float32)
    check(ctx, pts, 0.1)
    out, trace = ctx.voxel_downsample(pts, 0.1, return_trace=True)
    assert out.tobytes() == pts.tobytes() and np.array_equal(trace, np.arange(len(pts)))


def test_one_large_voxel_is_the_sequential_sum(ctx):
    """200k points in one voxel, 10k of them at x = +1e30 and 10k at -1e30: while the running float64 sum is near
    1e30 it absorbs the small coordinates, so only the sequential order gives the reference's bits (a pairwise sum
    does not)."""
    rng = np.random.default_rng(10)
    n = 200000
    pts = rng.uniform(0, 1, size=(n, 3)).astype(np.float32)
    big = rng.choice(n, 20000, replace=False)
    pts[big[:10000], 0] = np.float32(1e30)
    pts[big[10000:], 0] = np.float32(-1e30)
    want = check(ctx, pts, 1e31)
    assert want[0].shape == (1, 3)
    p64 = pts.astype(np.float64)
    pairwise = (np.array([np.sum(np.ascontiguousarray(p64[:, k])) for k in range(3)]) / n).astype(np.float32)
    assert pairwise.tobytes() != want[0].tobytes()


def test_large_offset(ctx):
    pts = surface(np.random.default_rng(11), 60000, offset=(1e4, -1e4, 1e4))
    check(ctx, pts, 0.05)


def test_int_max_check(ctx):
    v = 2.0 ** -20
    ok = np.array([[0, 0, 0], [2048 - 2.0 ** -13, 0, 0]], dtype=np.float32)
    bad = np.array([[0, 0, 0], [2048, 0, 0]], dtype=np.float32)
    check(ctx, ok, v)
    with pytest.raises(capi.TzrError):
        ctx.voxel_downsample(bad, v)


def test_cell_limit_in_a_batch(ctx):
    at = np.array([[0, 0, 0], [2 ** 21 - 1, 2 ** 21 - 1, 2 ** 20 - 1], [3, 3, 3]], dtype=np.float32)
    over = np.array([[0, 0, 0], [2 ** 21 - 1, 2 ** 21 - 1, 2 ** 20], [3, 3, 3]], dtype=np.float32)
    rng = np.random.default_rng(12)
    others = [surface(rng, 3000), surface(rng, 1), surface(rng, 8000)]
    batch = [others[0], over, at, others[1], over, others[2]]
    with pytest.raises(capi.TzrError) as e:
        ctx.voxel_downsample_batch(batch, 1.0, return_trace=True)
    assert e.value.status.tolist() == [0, capi.TZR_ERR_TOO_LARGE, 0, 0, capi.TZR_ERR_TOO_LARGE, 0]
    outs, traces = e.value.result
    for k, pts in enumerate(batch):
        want = ref.downsample(pts, 1.0)
        assert want[2] == e.value.status[k]
        assert outs[k].tobytes() == want[0].tobytes() and np.array_equal(traces[k], want[1]), k
    assert outs[2].shape == (3, 3) and outs[1].shape == (0, 3) and (traces[1] == -1).all()


def ragged(seed):
    rng = np.random.default_rng(seed)
    sizes = [1, 5000, 37, 120000, 1, 2, 60000, 999]
    clouds = [surface(rng, n) for n in sizes]
    clouds[2][5] = np.nan
    clouds[5][:] = np.nan
    return clouds


def test_batch_equals_single_forward_and_reverse(ctx):
    clouds = ragged(13)
    v = 0.04
    single = [ctx.voxel_downsample(c, v, return_trace=True) for c in clouds]
    for order in (list(range(len(clouds))), list(range(len(clouds)))[::-1]):
        outs, traces = ctx.voxel_downsample_batch([clouds[k] for k in order], v, return_trace=True)
        for pos, k in enumerate(order):
            assert outs[pos].tobytes() == single[k][0].tobytes() and np.array_equal(traces[pos], single[k][1]), k
    # without traces, and against the reference
    outs = ctx.voxel_downsample_batch(clouds, v)
    for k, c in enumerate(clouds):
        want = ref.downsample(c, v)
        assert outs[k].tobytes() == want[0].tobytes() and np.array_equal(single[k][1], want[1]), k


def test_launch_count_does_not_depend_on_B(ctx):
    pts = surface(np.random.default_rng(14), 3000)
    counts = []
    for B in (1, 7, 64):
        l0 = ctx.kernel_launches()
        ctx.voxel_downsample_batch([pts] * B, 0.05)
        counts.append(ctx.kernel_launches() - l0)
    assert counts == [10, 10, 10]


def test_retained_solve_survives_a_downsample(ctx):
    rng = np.random.default_rng(3)
    src = rng.uniform(-1, 1, (120, 3))
    R = Rotation.from_rotvec([0.1, 0.2, -0.1]).as_matrix()
    dst = src @ R.T + [0.1, 0.0, 0.2]
    dst[:30] = rng.uniform(-1, 1, (30, 3))
    prm = capi.default_params(noise_bound=0.01, estimate_scaling=0, rotation_cost_threshold=1e-12)
    ctx.solve(src, dst, prm)
    before = ctx.last_inliers(0)
    cert_before = ctx.certify_last(noise_bound=0.02)
    ctx.voxel_downsample_batch(ragged(15), 0.05)
    after = ctx.last_inliers(0)
    assert all(np.array_equal(a, b) for a, b in zip(before, after))
    cert_after = ctx.certify_last(noise_bound=0.02)
    assert cert_before[0]["best_suboptimality"] == cert_after[0]["best_suboptimality"]
    assert np.array_equal(cert_before[0]["suboptimality_traj"], cert_after[0]["suboptimality_traj"])


@pytest.mark.parametrize("case", ["v_zero", "v_negative", "v_nan", "v_inf", "B_zero", "n_zero", "n_negative",
                                  "n_null", "pts_null", "pts_entry_null", "pts_out_null", "pts_out_entry_null",
                                  "n_out_null"])
def test_argument_checks_with_a_context(ctx, case):
    """Each malformed call is refused by its own check (a real context here, so no earlier check can answer)."""
    assert arg_cases.call_batch(ctx._h, **arg_cases.CASES[case]) == capi.TZR_ERR_INVALID_ARG
    assert arg_cases.call_batch(ctx._h) == 0


def test_more_than_int_max_points_is_too_large(ctx):
    """The size check runs before any point is read, so the counts alone decide it."""
    x = np.zeros((1, 3), dtype=np.float32)
    fp, i32p = C.POINTER(C.c_float), C.POINTER(C.c_int32)
    n = np.array([2 ** 30, 2 ** 30], dtype=np.int32)
    m = np.zeros(2, dtype=np.int32)
    ptrs = (fp * 2)(x.ctypes.data_as(fp), x.ctypes.data_as(fp))
    assert capi.lib().tzr_voxel_downsample_batch(ctx._h, 2, n.ctypes.data_as(i32p), ptrs, 0.1, ptrs,
                                                 m.ctypes.data_as(i32p), None, None) == capi.TZR_ERR_TOO_LARGE


# ---- the tutorial from raw scans: voxel_down_sample(0.05), FPFH at 2v / 5v, mutual matching, the solve, ICP at v ------
V = 0.05


def raw_pair(seed, n=200000):
    """Two independent dense samplings of one surface; the second moved by a ground-truth (R, t)."""
    rng = np.random.default_rng(seed)
    src = surface(rng, n)
    R = Rotation.from_rotvec(rng.normal(size=3) / np.sqrt(3) * np.radians(25)).as_matrix()
    t = rng.normal(size=3) * 0.3
    dst = (surface(rng, n).astype(np.float64) @ R.T + t).astype(np.float32)
    return src, dst, R, t


def test_tutorial_from_raw_scans(ctx):
    pairs_gt = [raw_pair(20), raw_pair(21)]
    src0 = pairs_gt[0][0]
    # the raw scans are too dense for the descriptor stage at the tutorial's radii: more than 4096 neighbours
    crop = src0[np.linalg.norm(src0[:, :2] - src0[:, :2].mean(axis=0), axis=1) < 0.3]
    with pytest.raises(capi.TzrError):
        ctx.compute_fpfh(crop, 2 * V, 5 * V)
    raw = [c for s, d, _, _ in pairs_gt for c in (s, d)]
    down = ctx.voxel_downsample_batch(raw, V)
    print("downsampled", [len(r) for r in raw], "->", [len(d) for d in down])
    assert all(len(d) < len(r) // 20 for d, r in zip(down, raw))
    ctx.compute_fpfh(down[0], 2 * V, 5 * V)  # now within the limit
    prm = capi.default_params(noise_bound=V, estimate_scaling=0, rotation_cost_threshold=1e-12)
    res = ctx.register_cloud_pairs_icp(down, [(0, 1), (2, 3)], prm, V, normal_search_radius=2 * V,
                                       fpfh_search_radius=5 * V, use_absolute_scale=False, use_crosscheck=True,
                                       use_tuple_test=False)
    sols, status, icp_res = res[0], res[1], res[6]
    for p, (src, _, R, t) in enumerate(pairs_gt):
        assert status[p] == 0 and sols[p]["valid"], p
        d = capi.icp_result_dict(icp_res[p])
        moved = src.astype(np.float64) @ d["R"].T + d["t"]
        truth = src.astype(np.float64) @ R.T + t
        err = np.linalg.norm(moved - truth, axis=1)
        rot_err = np.degrees(Rotation.from_matrix(d["R"] @ R.T).magnitude())
        print(f"pair {p}: mean displacement error {err.mean():.4f}, max {err.max():.4f}, rotation {rot_err:.3f} deg")
        assert err.max() < 2 * V, p


def test_cpp_facade_equals_the_c_abi(tmp_path):
    """voxelDownSample / voxelDownSampleBatch against tzr_voxel_downsample (tests/cpp/voxel_test.cc)."""
    subprocess.check_call(["make", "-s", "-C", HOST])
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    exe = str(tmp_path / "voxel_test")
    subprocess.check_call([cxx, "-std=c++17", "-O1", "-I", os.path.join(HOST, "include"), "-I",
                           os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "voxel_test.cc"),
                           "-L", HOST, "-lteaser_registration", "-L", CSRC, "-lteaser_b200",
                           f"-Wl,-rpath,{HOST}:{CSRC}", "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr


def test_pybind_voxel_down_sample(ctx):
    subprocess.check_call(["make", "-s", "-C", HOST])
    sys.path.insert(0, os.path.join(HOST, "python"))
    import teaserpp_python as tpp
    clouds = ragged(16)
    for c in clouds:
        got = tpp.voxel_down_sample(c, 0.03)
        assert got.dtype == np.float32 and got.tobytes() == ctx.voxel_downsample(c, 0.03).tobytes()
    got = tpp.voxel_down_sample_batch(clouds, 0.03)
    want = ctx.voxel_downsample_batch(clouds, 0.03)
    assert len(got) == len(want) and all(a.tobytes() == b.tobytes() for a, b in zip(got, want))
    with pytest.raises(ValueError):
        tpp.voxel_down_sample(clouds[0], 0.0)
