"""The numpy generalized-ICP restatement (tests/icp_generalized_reference.py) against independent facts: Open3D's
form of the system (Rodrigues covariances, W = M^-1/2 and three weighted rows per correspondence), the normals' sign
and validity rules, Kabsch as the epsilon = 1 fixed point, exact recovery on a smooth surface and the centred step's
accuracy far from the origin.  No GPU."""
import numpy as np
import pytest

import icp_generalized_reference as ref
from icp_reference import rotation_from_H
from test_icp_plane_reference_cpu import _moved_pair, _wavy


def _skew(v):
    return np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])


def _rotation_e1_to(x):
    """Open3D's GetRotationFromE1ToX: Rodrigues' rotation taking e1 onto the unit vector x."""
    e1 = np.array([1.0, 0.0, 0.0])
    c = e1 @ x
    assert c >= -0.99  # the tests stay off Open3D's identity branch
    sv = _skew(np.cross(e1, x))
    return np.eye(3) + sv + (sv @ sv) / (1.0 + c)


def _open3d_system(P, Q, Ms, Nt, R, s, epsilon):
    """Open3D's TransformationEstimationForGeneralizedICP::ComputeTransformation with the L2 loss, linearised about the
    origin: per correspondence C = Rx diag(eps, 1, 1) Rx^T for both clouds, the source's moved by (sR), W = sqrt(M^-1)
    by eigh, rows W [-[p]x, I] and residual W (p - q)."""
    A, g = np.zeros((6, 6)), np.zeros(6)
    D = np.diag([epsilon, 1.0, 1.0])
    sR = s * np.asarray(R)
    for p, q, m, n in zip(P, Q, Ms, Nt):
        Rs, Rt = _rotation_e1_to(m), _rotation_e1_to(n)
        M = sR @ (Rs @ D @ Rs.T) @ sR.T + Rt @ D @ Rt.T
        w, V = np.linalg.eigh(np.linalg.inv(M))
        W = V @ np.diag(np.sqrt(w)) @ V.T
        rows = W @ np.concatenate([-_skew(p), np.eye(3)], axis=1)
        A += rows.T @ rows
        g += rows.T @ (W @ (p - q))
    return A, g


def _random_case(seed, n=300):
    rng = np.random.default_rng(seed)
    P = rng.uniform(-1, 1, (n, 3))
    Q = (P + rng.normal(scale=0.02, size=P.shape)).astype(np.float32)

    def normals():
        v = rng.normal(size=(n, 3))
        v /= np.linalg.norm(v, axis=1, keepdims=True)
        v[v[:, 0] < -0.9, 0] *= -1  # away from GetRotationFromE1ToX's e1 . x < -0.99 branch
        return v.astype(np.float32)

    Ms, Nt = normals(), normals()
    R = ref.plane.euler(*rng.uniform(-0.3, 0.3, 3))
    return P, Q, Ms, Nt, R


@pytest.mark.parametrize("seed,s,epsilon", [(0, 1.0, 1e-3), (1, 1.7, 1e-3), (2, 0.6, 0.05), (3, 1.0, 0.5)])
def test_system_equals_the_open3d_form(seed, s, epsilon):
    P, Q, Ms, Nt, R = _random_case(seed)
    # the source normals m play the part of the unmoved cloud's normals; R is the current rotation
    ev = dict(p=P, idx=np.arange(len(P)))
    A, g = ref.system(ev, Q, Ms, Nt, R, s, epsilon, np.zeros(3))
    Ms64 = Ms.astype(np.float64)
    Ms64 /= np.linalg.norm(Ms64, axis=1, keepdims=True)
    Nt64 = Nt.astype(np.float64)
    Nt64 /= np.linalg.norm(Nt64, axis=1, keepdims=True)
    A_o, g_o = _open3d_system(P, Q.astype(np.float64), Ms64, Nt64, R, s, epsilon)
    assert np.abs(A - A_o).max() <= 1e-9 * np.abs(A_o).max()
    assert np.abs(g - g_o).max() <= 1e-9 * np.abs(g_o).max()


def test_normal_signs_and_invalid_normals():
    P, Q, Ms, Nt, R = _random_case(5)
    ev = dict(p=P, idx=np.arange(len(P)))
    args = (R, 1.3, 1e-3, P.mean(axis=0))
    A, g = ref.system(ev, Q, Ms, Nt, *args)
    rng = np.random.default_rng(5)
    fm, fn = rng.random(len(P)) < 0.5, rng.random(len(P)) < 0.5
    Ms2, Nt2 = Ms.copy(), Nt.copy()
    Ms2[fm] *= -1
    Nt2[fn] *= -1
    A2, g2 = ref.system(ev, Q, Ms2, Nt2, *args)
    assert np.array_equal(A, A2) and np.array_equal(g, g2)
    # zero-length and NaN normals on either side drop the correspondence from the system only
    bad = np.zeros(len(P), dtype=bool)
    bad[[3, 10, 50, 77]] = True
    Ms3, Nt3 = Ms.copy(), Nt.copy()
    Ms3[3] = 0.0
    Nt3[10] = 0.0
    Ms3[50, 1] = np.nan
    Nt3[77, 2] = np.inf
    A3, g3 = ref.system(ev, Q, Ms3, Nt3, *args)
    keep = ~bad
    ev_k = dict(p=P[keep], idx=np.arange(keep.sum()))
    A4, g4 = ref.system(ev_k, Q[keep], Ms[keep], Nt[keep], *args)
    np.testing.assert_allclose(A3, A4, rtol=1e-12, atol=1e-12 * np.abs(A4).max())
    np.testing.assert_allclose(g3, g4, rtol=1e-12, atol=1e-12 * np.abs(g4).max())
    assert not np.allclose(A3, A)


def test_epsilon_one_converges_to_kabsch():
    """epsilon = 1 makes every covariance I, so the system is point-to-point's Gauss-Newton step; iterated on fixed
    correspondences it converges to the Kabsch solution."""
    rng = np.random.default_rng(8)
    X = rng.uniform(-1, 1, (200, 3))
    Rg = ref.plane.euler(0.2, -0.1, 0.3)
    Y = X @ Rg.T + [0.1, -0.2, 0.05] + rng.normal(scale=0.01, size=X.shape)
    Y32 = Y.astype(np.float32)
    Ms = rng.normal(size=(200, 3)).astype(np.float32)
    Nt = rng.normal(size=(200, 3)).astype(np.float32)
    upd = ref.Update(Ms, 1.0, None, 1.0)
    R, t = np.eye(3), np.zeros(3)
    for _ in range(30):
        ev = dict(p=X @ R.T + t, idx=np.arange(200))
        Ru, tu = upd(ev, Y32, Nt)
        R, t = Ru @ R, Ru @ t + tu
    Yd = Y32.astype(np.float64)
    Rk = rotation_from_H((X - X.mean(0)).T @ (Yd - Yd.mean(0)))
    tk = Yd.mean(0) - Rk @ X.mean(0)
    np.testing.assert_allclose(R, Rk, atol=1e-12)
    np.testing.assert_allclose(t, tk, atol=1e-12)


def test_exact_recovery_on_a_smooth_surface():
    src, dst, nrm, R, t = _moved_pair(5)
    _, N = _wavy(len(src), 5)
    src_n = np.concatenate([N, np.zeros((len(N), 1))], axis=1).astype(np.float32)
    out = ref.icp(src, dst, src_n, nrm, 0.2, max_iteration=60, relative_fitness=0, relative_rmse=0)
    np.testing.assert_allclose(out["R"], R, atol=1e-6)
    np.testing.assert_allclose(out["t"], t, atol=1e-6)
    assert out["inlier_rmse"] < 1e-6 and out["n_correspondences"] == len(src)


def test_centred_step_at_large_offset():
    """A pure translation of float32 surface points on a 2^-16 grid, at the origin and at 1e5 (test_icp_plane_reference
    _cpu's check): the linear model is exact, so the centred step recovers tau to rounding at both places."""
    errs = {}
    for name, off in (("origin", (0.0, 0.0, 0.0)), ("far", (1e5, -1e5, 5e4))):
        P, N = _wavy(2000, 7)
        src = (np.round(P * 2.0 ** 16) * 2.0 ** -16 + np.asarray(off)).astype(np.float32)
        tau = np.array([3.0, -2.0, 1.0]) * 2.0 ** -7
        dst = (src.astype(np.float64) + tau).astype(np.float32)
        assert np.array_equal(dst.astype(np.float64) - src.astype(np.float64), np.tile(tau, (2000, 1)))
        nrm = np.concatenate([N, np.zeros((2000, 1))], axis=1).astype(np.float32)
        ev = dict(p=ref.transform(src, 1.0, np.eye(3), np.zeros(3)), idx=np.arange(2000))
        Ru, tu = ref.Update(nrm, 1.0, None, 1e-3)(ev, dst, nrm)
        c = src.astype(np.float64).mean(axis=0)
        errs[name] = (np.abs(Ru - np.eye(3)).max(), np.abs((Ru @ c + tu) - (c + tau)).max())
    print(errs)
    assert max(errs["origin"]) < 1e-12
    assert max(errs["far"]) < 1e-9
