"""The numpy ICP restatement (tests/icp_reference.py) against independent facts: a KD-tree, exact recoveries and the
edge rules of tzr_icp.  No GPU."""
import numpy as np
import pytest
from scipy.spatial import cKDTree
from scipy.spatial.transform import Rotation

import icp_reference as ref


def _cloud(n, seed, scale=1.0):
    return (np.random.default_rng(seed).uniform(-1, 1, (n, 3)) * scale).astype(np.float32)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_nearest_matches_kdtree(seed):
    x, y = _cloud(700, seed), _cloud(900, seed + 10)
    p = ref.transform(x, 1.0, Rotation.from_rotvec([0.1, -0.2, 0.05]).as_matrix(), [0.01, 0.02, -0.03])
    r = 0.15
    idx, d2 = ref.nearest(p, y, r * r)
    dist, j = cKDTree(y.astype(np.float64)).query(p, k=1)
    hit = dist < r
    assert hit.sum() > 100 and (~hit).sum() > 10
    assert np.array_equal(idx >= 0, hit)
    assert np.array_equal(idx[hit], j[hit])
    np.testing.assert_allclose(d2[hit], dist[hit] ** 2, rtol=1e-12)


def test_strict_bound_ties_and_non_finite():
    y = np.array([[1, 0, 0], [0, 1, 0], [-1, 0, 0], [0.5, 0, 0], [np.nan, 0, 0], [np.inf, 0, 0]], dtype=np.float32)
    p = np.array([[0, 0, 0], [0.25, 0, 0], [0, 0, 2], [np.nan, 0, 0], [1e30, 0, 0]], dtype=np.float64)
    idx, _ = ref.nearest(p, y, 1.0)
    # (0,0,0): d^2 = 1 to three targets and 0.25 to (0.5,0,0); (0.25,0,0): 0.0625 to (0.5,0,0)
    assert idx.tolist() == [3, 3, -1, -1, -1]
    idx, _ = ref.nearest(p[:1], y[:3], 1.0)  # only d^2 = r^2 exactly: strict bound, no match
    assert idx.tolist() == [-1]
    idx, _ = ref.nearest(p[:1], y[:3], 1.0 + 2 ** -40)  # equidistant: the lowest index
    assert idx.tolist() == [0]


def test_recovers_known_motion_in_one_update():
    x = _cloud(500, 3)
    R = Rotation.from_rotvec([0.02, 0.01, -0.03]).as_matrix()
    t = np.array([0.01, -0.02, 0.015])
    # the source moved by (R, t)^-1: one update with exact correspondences onto the float targets x recovers (R, t)
    P = ref.transform(x, 1.0, R.T, -R.T @ t)
    Ru, tu = ref.update(dict(p=P, idx=np.arange(500)), x)
    np.testing.assert_allclose(Ru, R, atol=1e-12)
    np.testing.assert_allclose(tu, t, atol=1e-12)
    np.testing.assert_allclose(Ru @ P.T + tu[:, None], x.astype(np.float64).T, atol=1e-12)


def test_count_rules():
    y = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], dtype=np.float32)
    far = np.array([[10, 10, 10], [11, 10, 10]], dtype=np.float32)
    out = ref.icp(far, y, 0.5)
    assert (out["iterations"], out["converged"], out["n_correspondences"]) == (1, True, 0)
    assert out["fitness"] == 0.0 and out["inlier_rmse"] == 0.0
    np.testing.assert_array_equal(out["R"], np.eye(3))
    np.testing.assert_array_equal(out["t"], np.zeros(3))
    # one correspondence: a pure translation onto it
    one = np.array([[0.1, 0.05, 0], [5, 5, 5]], dtype=np.float32)
    ev = ref.evaluate(one, y, 1.0, np.eye(3), np.zeros(3), 0.25)
    assert ev["count"] == 1
    Ru, tu = ref.update(ev, y)
    np.testing.assert_array_equal(Ru, np.eye(3))
    np.testing.assert_allclose(tu, -one[0].astype(np.float64), rtol=0, atol=0)
    # two correspondences: the mean translation
    two = np.array([[0.1, 0, 0], [0.9, 0.1, 0]], dtype=np.float32)
    ev = ref.evaluate(two, y, 1.0, np.eye(3), np.zeros(3), 0.25)
    Ru, tu = ref.update(ev, y)
    assert ev["count"] == 2
    np.testing.assert_array_equal(Ru, np.eye(3))
    np.testing.assert_allclose(tu, (y[[0, 1]].astype(np.float64) - two.astype(np.float64)).mean(axis=0))
    # max_iteration = 0: the initial transform and its evaluation
    R0 = Rotation.from_rotvec([0, 0, 0.1]).as_matrix()
    out = ref.icp(two, y, 0.5, R=R0, t=[0.01, 0, 0], max_iteration=0)
    assert out["iterations"] == 0 and not out["converged"]
    np.testing.assert_array_equal(out["R"], R0)


def test_fixed_scale():
    x = _cloud(400, 5)
    R = Rotation.from_rotvec([0.0, 0.03, 0.01]).as_matrix()
    t = np.array([0.02, 0.0, -0.01])
    s = 0.5
    y = (s * (x.astype(np.float64) @ R.T) + t).astype(np.float32)
    out = ref.icp(x, y, 0.1, s=s, R=Rotation.from_rotvec([0, 0.02, 0]).as_matrix(), t=[0.015, 0, 0])
    assert out["scale"] == s
    np.testing.assert_allclose(out["R"], R, atol=1e-6)
    np.testing.assert_allclose(out["t"], t, atol=1e-6)
    assert out["inlier_rmse"] < 1e-6


def test_centring_at_large_offset():
    """At |x| ~ 1e5 the centred covariance keeps its digits; the uncentred sum p q^T - n mu_p mu_q^T loses them."""
    rng = np.random.default_rng(7)
    P = rng.uniform(-0.5, 0.5, (2000, 3))
    R = Rotation.from_rotvec([0.01, -0.02, 0.015]).as_matrix()
    Q = P @ R.T
    off = np.array([1e5, -1e5, 5e4])
    Po, Qo = P + off, Q + off
    mp, mq = Po.mean(axis=0), Qo.mean(axis=0)
    Hc = (Po - mp).T @ (Qo - mq)
    Hu = Po.T @ Qo - len(Po) * np.outer(mp, mq)
    err_c = np.abs(ref.rotation_from_H(Hc) - R).max()
    err_u = np.abs(ref.rotation_from_H(Hu) - R).max()
    assert err_c < 1e-9
    assert err_u > 1e3 * err_c and err_u > 1e-6
