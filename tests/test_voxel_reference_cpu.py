"""CPU checks of tests/voxel_reference.py: the vectorised numpy restatement of voxel-grid downsampling against a plain
dict loop that restates Open3D's VoxelDownSample line by line, bit for bit, on small clouds built to sit on the rules'
edges; and that the voxel index is a division, not a product with 1/v."""
import numpy as np
import pytest

import voxel_reference as ref


def same(a, b):
    (pa, ta, sa), (pb, tb, sb) = a, b
    return sa == sb and pa.shape == pb.shape and pa.tobytes() == pb.tobytes() and np.array_equal(ta, tb)


@pytest.mark.parametrize("v", [0.125, 0.05])
def test_points_on_voxel_edges(v):
    pts = ref.lattice_on_edges(v)
    got = ref.downsample(pts, v)
    assert same(got, ref.downsample_dict_loop(pts, v))
    assert got[2] == ref.TZR_OK and 0 < got[0].shape[0] <= pts.shape[0]


@pytest.mark.parametrize("v", [0.125, 0.05, 0.3])
def test_random_clouds(v):
    rng = np.random.default_rng(int(v * 1000))
    pts = rng.uniform(-1, 1, size=(400, 3)).astype(np.float32)
    got = ref.downsample(pts, v)
    assert same(got, ref.downsample_dict_loop(pts, v))
    assert got[0].shape[0] < 400 and (got[1] >= 0).all()


def test_duplicate_points():
    rng = np.random.default_rng(1)
    base = rng.uniform(0, 1, size=(30, 3)).astype(np.float32)
    pts = np.concatenate([base, base[::-1], base[:7]])
    got = ref.downsample(pts, 0.05)
    assert same(got, ref.downsample_dict_loop(pts, 0.05))
    assert np.array_equal(got[1][:30], got[1][30:60][::-1]) and np.array_equal(got[1][60:], got[1][:7])


def test_non_finite_rows():
    rng = np.random.default_rng(2)
    pts = rng.uniform(0, 1, size=(60, 3)).astype(np.float32)
    pts[3] = np.nan
    pts[10, 1] = np.inf
    pts[11, 2] = -np.inf
    pts[12] = [1e6, np.nan, 0.0]   # would stretch the bounds if it counted
    got = ref.downsample(pts, 0.1)
    assert same(got, ref.downsample_dict_loop(pts, 0.1))
    assert (got[1][[3, 10, 11, 12]] == -1).all() and (np.delete(got[1], [3, 10, 11, 12]) >= 0).all()
    assert np.array_equal(got[0], ref.downsample(np.delete(pts, [3, 10, 11, 12], axis=0), 0.1)[0])


def test_single_point_and_all_nan():
    one = np.array([[0.3, -2.0, 7.5]], dtype=np.float32)
    got = ref.downsample(one, 0.05)
    assert same(got, ref.downsample_dict_loop(one, 0.05))
    assert got[0].tobytes() == one.tobytes() and got[1].tolist() == [0]
    nan = np.full((5, 3), np.nan, dtype=np.float32)
    got = ref.downsample(nan, 0.05)
    assert same(got, ref.downsample_dict_loop(nan, 0.05))
    assert got[0].shape == (0, 3) and (got[1] == -1).all() and got[2] == ref.TZR_OK


def test_output_order_is_first_member_and_sparse_input_comes_back():
    rng = np.random.default_rng(3)
    cells = rng.permutation(np.stack(np.meshgrid(*[np.arange(5)] * 3, indexing="ij"), -1).reshape(-1, 3))
    pts = (cells * 0.1 + rng.uniform(-0.02, 0.02, size=cells.shape)).astype(np.float32)
    got = ref.downsample(pts, 0.1)
    assert got[0].tobytes() == pts.tobytes() and np.array_equal(got[1], np.arange(len(pts)))
    assert same(got, ref.downsample_dict_loop(pts, 0.1))


def test_index_is_a_division():
    pts, v = ref.division_case()
    p = pts.astype(np.float64)
    vmin = p.min(axis=0) - v * 0.5
    by_div = np.floor((p[2, 0] - vmin[0]) / v)
    by_inv = np.floor((p[2, 0] - vmin[0]) * (1.0 / v))
    assert (by_div, by_inv) == (2.0, 3.0)
    assert ref.voxel_indices(p[2:3], vmin, v)[0, 0] == 2
    got = ref.downsample(pts, v)
    assert same(got, ref.downsample_dict_loop(pts, v))
    assert got[1].tolist() == [0, 1, 1, 2]


def test_size_limits():
    # Open3D's INT_MAX check: with v = 2^-20 the extent X + v is rejected from X = 2048 on
    v = 2.0 ** -20
    ok = np.array([[0, 0, 0], [2048 - 2.0 ** -13, 0, 0]], dtype=np.float32)
    bad = np.array([[0, 0, 0], [2048, 0, 0]], dtype=np.float32)
    assert ref.downsample(ok, v)[2] == ref.TZR_OK and ref.downsample(ok, v)[0].shape == (2, 3)
    assert ref.downsample(bad, v)[2] == ref.TZR_ERR_TOO_LARGE
    assert same(ref.downsample(ok, v), ref.downsample_dict_loop(ok, v))
    assert same(ref.downsample(bad, v), ref.downsample_dict_loop(bad, v))
    # 2^62 cells: counts (2^21, 2^21, 2^20) fit, (2^21, 2^21, 2^20 + 1) do not
    at = np.array([[0, 0, 0], [2 ** 21 - 1, 2 ** 21 - 1, 2 ** 20 - 1]], dtype=np.float32)
    over = np.array([[0, 0, 0], [2 ** 21 - 1, 2 ** 21 - 1, 2 ** 20]], dtype=np.float32)
    assert ref.grid(at, 1.0)[2] == [2 ** 21, 2 ** 21, 2 ** 20]
    assert ref.downsample(at, 1.0)[2] == ref.TZR_OK and ref.downsample(at, 1.0)[0].shape == (2, 3)
    assert ref.downsample(over, 1.0)[2] == ref.TZR_ERR_TOO_LARGE
    assert same(ref.downsample(over, 1.0), ref.downsample_dict_loop(over, 1.0))


def test_one_large_voxel_is_summed_in_order():
    rng = np.random.default_rng(4)
    pts = (rng.uniform(0, 0.01, size=(5000, 3)) + [1e3, -7.0, 0.5]).astype(np.float32)
    got = ref.downsample(pts, 1.0)
    assert got[0].shape == (1, 3)
    s = np.zeros(3)
    for q in pts.astype(np.float64):
        s = s + q
    assert got[0].tobytes() == (s / 5000.0).astype(np.float32).tobytes()
