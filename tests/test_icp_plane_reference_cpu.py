"""The numpy point-to-plane ICP restatement (tests/icp_plane_reference.py) against independent facts: numpy's solver,
the truncation rule on rank-deficient systems, scipy's Euler angles, exact recovery on a smooth surface, the
origin-linearised (Open3D) form's fixed point, and the centred form's accuracy far from the origin.  No GPU."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import icp_plane_reference as ref


@pytest.mark.parametrize("seed", range(5))
def test_solve_matches_numpy_on_spd_systems(seed):
    rng = np.random.default_rng(seed)
    M = rng.normal(size=(6, 6))
    A = M @ M.T + 0.1 * np.eye(6)
    g = rng.normal(size=6)
    x = ref.solve6(A, g)
    np.testing.assert_allclose(x, np.linalg.solve(A, -g), rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize("rank", [0, 1, 3, 5])
def test_truncation_on_rank_deficient_systems(rank):
    """A = B^T B of rank k with g in its range: zero in A's null directions, A x = -g."""
    rng = np.random.default_rng(10 + rank)
    B = rng.normal(size=(rank, 6))
    A = B.T @ B
    g = B.T @ rng.normal(size=rank)
    x = ref.solve6(A, g)
    _, _, Vt = np.linalg.svd(A)
    null = Vt[rank:]
    if rank:
        np.testing.assert_allclose(A @ x, -g, atol=1e-9 * (1 + np.abs(g).max()))
    else:
        assert np.array_equal(x, np.zeros(6))
    # the truncated components of the permuted solution are exactly zero, so x has at most `rank` non-zeros
    assert np.count_nonzero(x) <= rank
    # x lies in no null direction beyond what solving on the leading block forces: A x = -g fixes x up to null(A),
    # and the solve picks the representative with the unpivoted components 0
    assert null.shape[0] == 6 - rank


def test_flat_target_has_no_in_plane_motion():
    """All normals parallel (a plane z = const): only the offset along the normal and the rotations about the in-plane
    axes that tilt it are observable; x moves along none of the rest."""
    rng = np.random.default_rng(3)
    P = np.concatenate([rng.uniform(-1, 1, (400, 2)), np.zeros((400, 1))], axis=1)
    n = np.tile([0.0, 0.0, 1.0], (400, 1))
    u = P - P.mean(axis=0)
    J = np.concatenate([np.cross(u, n), n], axis=1)
    r = np.full(400, -0.01)
    x = ref.solve6(J.T @ J, J.T @ r)
    assert x[2] == 0.0 and x[3] == 0.0 and x[4] == 0.0  # rotation about z, translation in x and y
    assert abs(x[5] - 0.01) < 1e-12


def test_euler_matches_scipy():
    rng = np.random.default_rng(4)
    for _ in range(20):
        x = rng.uniform(-np.pi, np.pi, 3)
        want = Rotation.from_euler("ZYX", [x[2], x[1], x[0]]).as_matrix()
        np.testing.assert_allclose(ref.euler(*x), want, atol=1e-15)


def _wavy(n, seed):
    """A noise-free smooth surface z = f(x, y) with its analytic unit normals."""
    rng = np.random.default_rng(seed)
    uv = rng.uniform(-1, 1, (n, 2))
    z = 0.3 * np.sin(3 * uv[:, 0]) * np.cos(2 * uv[:, 1])
    fx = 0.9 * np.cos(3 * uv[:, 0]) * np.cos(2 * uv[:, 1])
    fy = -0.6 * np.sin(3 * uv[:, 0]) * np.sin(2 * uv[:, 1])
    P = np.stack([uv[:, 0], uv[:, 1], z], axis=1)
    N = np.stack([-fx, -fy, np.ones(n)], axis=1)
    return P, N / np.linalg.norm(N, axis=1, keepdims=True)


def _moved_pair(seed, n=1500, offset=(0.0, 0.0, 0.0)):
    """The target: the surface at `offset` moved by (R, t), float32, with its rotated normals; the source: the same
    sampling unmoved (the identical points, so (R, t) is the exact solution)."""
    P, N = _wavy(n, seed)
    off = np.asarray(offset, dtype=np.float64)
    R = Rotation.from_rotvec([0.02, -0.015, 0.03]).as_matrix()
    t = np.array([0.01, -0.02, 0.015])
    c = off
    tt = c - R @ c + t  # the motion about the cloud's own centre
    src = (P + off).astype(np.float32)
    dst = (src.astype(np.float64) @ R.T + tt).astype(np.float32)
    nrm = np.concatenate([N @ R.T, np.zeros((n, 1))], axis=1).astype(np.float32)
    return src, dst, nrm, R, tt


def test_exact_recovery_on_a_smooth_surface():
    src, dst, nrm, R, t = _moved_pair(5)
    out = ref.icp(src, dst, nrm, 0.2, max_iteration=60, relative_fitness=0, relative_rmse=0)
    # float32 targets: the exact motion of the float sources, rounded; the loop reaches it to the float rounding
    np.testing.assert_allclose(out["R"], R, atol=1e-6)
    np.testing.assert_allclose(out["t"], t, atol=1e-6)
    assert out["inlier_rmse"] < 1e-6 and out["n_correspondences"] == len(src)


def _uncentred_update(ev, y, normals):
    """Open3D's TransformationEstimationPointToPlane: the same system linearised about the origin, t_u = tau."""
    m = ev["idx"] >= 0
    if not m.any():
        return np.eye(3), np.zeros(3)
    A, g = ref.system(ev, y, normals, np.zeros(3))
    x = ref.solve6(A, g)
    return ref.euler(*x[:3]), x[3:]


def test_same_fixed_point_as_the_origin_form():
    src, dst, nrm, R, t = _moved_pair(6)
    kw = dict(max_iteration=60, relative_fitness=0, relative_rmse=0)
    a = ref.icp(src, dst, nrm, 0.2, **kw)
    b = ref.icp(src, dst, nrm, 0.2, update_fn=_uncentred_update, **kw)
    np.testing.assert_allclose(a["R"], b["R"], atol=1e-9)
    np.testing.assert_allclose(a["t"], b["t"], atol=1e-9)
    assert np.array_equal(a["corr"], b["corr"])


def test_centring_at_large_offset():
    """A pure translation of float32 planes far from the origin: both forms' linear model is exact (r + J x = 0 at
    x = (0, tau)), so every error is rounding.  At |x| ~ 1e5 the uncentred system's rotation block is ~1e10 times its
    Schur complement and loses the rotation's digits; the centred one stays at the float32 inputs' rounding."""
    errs = {}
    for name, off in (("origin", (0.0, 0.0, 0.0)), ("far", (1e5, -1e5, 5e4))):
        P, N = _wavy(2000, 7)
        # points on a 2^-16 grid and a shift by whole float steps at 1e5 (2^-7): every target is exactly its source
        # point moved by tau, here and at the origin
        src = (np.round(P * 2.0 ** 16) * 2.0 ** -16 + np.asarray(off)).astype(np.float32)
        tau = np.array([3.0, -2.0, 1.0]) * 2.0 ** -7
        dst = (src.astype(np.float64) + tau).astype(np.float32)
        assert np.array_equal(dst.astype(np.float64) - src.astype(np.float64), np.tile(tau, (2000, 1)))
        nrm = np.concatenate([N, np.zeros((2000, 1))], axis=1).astype(np.float32)
        ev = dict(p=ref.transform(src, 1.0, np.eye(3), np.zeros(3)), idx=np.arange(2000))
        for form, fn in (("centred", ref.update), ("uncentred", _uncentred_update)):
            Ru, tu = fn(ev, dst, nrm)
            c = src.astype(np.float64).mean(axis=0)
            errs[name, form] = (np.abs(Ru - np.eye(3)).max(), np.abs((Ru @ c + tu) - (c + tau)).max())
    print(errs)
    rc, tc = errs["far", "centred"]
    ru, tu_ = errs["far", "uncentred"]
    r0, t0 = errs["origin", "centred"]
    assert r0 < 1e-12 and t0 < 1e-12
    # the centred step far away is as exact as at the origin, up to the rounding of p - c at |p| ~ 1e5 (2^-36)
    assert rc < 1e-9 and tc < 1e-9
    assert ru > 1e3 * max(rc, 1e-13) and tu_ > 1e3 * max(tc, 1e-12)
