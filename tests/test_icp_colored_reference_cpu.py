"""The premises of the coloured ICP restatement (tests/icp_colored_reference.py), on the CPU: the gradient of a linear
colour field, the neighbour-count and collinear rules, normal signs, lambda = 1 against point-to-plane, the float step
against the exact one, and the textured plane that point-to-plane cannot align."""
import numpy as np
import pytest

import icp_colored_reference as ref
import icp_plane_reference as plane

R = 0.05


def _plane_cloud(step=0.01, extent=0.1, tilt=None):
    g = np.arange(-extent, extent + 1e-9, step)
    X, Y = np.meshgrid(g, g)
    P = np.stack([X.ravel(), Y.ravel(), np.zeros(X.size)], axis=1)
    n = np.array([0.0, 0.0, 1.0])
    if tilt is not None:
        P, n = P @ tilt.T, tilt @ n
    return P.astype(np.float32), np.tile(np.append(n, 0.0), (len(P), 1)).astype(np.float32)


def _tilt():
    a, b = 0.3, -0.2
    Rx = np.array([[1, 0, 0], [0, np.cos(a), -np.sin(a)], [0, np.sin(a), np.cos(a)]])
    Ry = np.array([[np.cos(b), 0, np.sin(b)], [0, 1, 0], [-np.sin(b), 0, np.cos(b)]])
    return Ry @ Rx


def test_linear_colour_field_gives_its_in_plane_gradient():
    T = _tilt()
    P, N = _plane_cloud(tilt=T)
    grad_true = np.array([0.8, -0.5, 2.0])  # only its in-plane part is observable
    tangent = grad_true - (grad_true @ N[0, :3].astype(np.float64)) * N[0, :3].astype(np.float64)
    level = 0.5 + P.astype(np.float64) @ grad_true
    colors = np.stack([level, level, level], axis=1).astype(np.float32)
    G = ref.color_gradients(P, N, colors, 0.035)
    inner = np.abs(P.astype(np.float64) @ T[:, :2]).max(axis=1) < 0.06  # full neighbourhoods
    assert inner.sum() > 20
    np.testing.assert_allclose(G[inner], np.tile(tangent, (inner.sum(), 1)), rtol=0, atol=2e-5)
    assert np.abs(G[inner] @ N[0, :3].astype(np.float64)).max() < 2e-5


def test_fewer_than_four_neighbours_give_zero():
    P = np.array([[0, 0, 0], [0.01, 0, 0], [0, 0.01, 0], [0.5, 0.5, 0]], dtype=np.float32)
    N = np.tile(np.array([0, 0, 1, 0], dtype=np.float32), (4, 1))
    C = np.random.default_rng(0).random((4, 3)).astype(np.float32)
    G = ref.color_gradients(P, N, C, 0.05)
    assert (G == 0).all()
    assert [len(x) for x in ref.neighbours(P, 0.05)] == [3, 3, 3, 1]


def test_collinear_neighbours_leave_the_unobservable_direction_at_zero():
    x = np.arange(-0.04, 0.041, 0.01)
    P = np.stack([x, np.zeros_like(x), np.zeros_like(x)], axis=1).astype(np.float32)
    N = np.tile(np.array([0, 0, 1, 0], dtype=np.float32), (len(P), 1))
    level = 0.3 + 2.0 * P[:, 0].astype(np.float64)
    C = np.stack([level] * 3, axis=1).astype(np.float32)
    G = ref.color_gradients(P, N, C, 0.1)
    assert (G[:, 1] == 0).all() and (G[:, 2] == 0).all()
    np.testing.assert_allclose(G[:, 0], 2.0, rtol=1e-5)


def test_selection_is_the_first_thirty_of_the_full_order():
    """A lattice with exact ties at the 30th place: the (d^2, index) order decides."""
    g = np.arange(-3, 4) * 0.25
    X, Y, Z = np.meshgrid(g, g, g, indexing="ij")
    P = np.stack([X.ravel(), Y.ravel(), Z.ravel()], axis=1).astype(np.float32)
    nb = ref.neighbours(P, 0.6)
    k = len(P) // 2
    d = P - P[k]
    d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
    order = np.lexsort((np.arange(len(P)), d2))
    assert np.array_equal(nb[k], order[:30])
    assert d2[order[29]] == d2[order[30]]  # a tie straddles the cut


def test_normal_signs_change_no_bit():
    rng = np.random.default_rng(3)
    P = rng.uniform(-0.1, 0.1, (400, 3)).astype(np.float32)
    P[:, 2] *= 0.1
    N = rng.normal(size=(400, 4)).astype(np.float32)
    C = rng.random((400, 3)).astype(np.float32)
    flip = N.copy()
    flip[rng.random(400) < 0.5, :3] *= -1
    a, b = ref.color_gradients(P, N, C, 0.04), ref.color_gradients(P, flip, C, 0.04)
    assert np.array_equal(a.view(np.uint64), b.view(np.uint64))


def _scan(seed=0, n=600):
    rng = np.random.default_rng(seed)
    uv = rng.uniform(-0.3, 0.3, (n, 2))
    z = 0.1 * np.sin(4 * uv[:, 0]) * np.cos(3 * uv[:, 1])
    y = np.stack([uv[:, 0], uv[:, 1], z], axis=1).astype(np.float32)
    nrm = np.stack([-0.4 * np.cos(4 * uv[:, 0]) * np.cos(3 * uv[:, 1]), 0.3 * np.sin(4 * uv[:, 0]) * np.sin(3 * uv[:, 1]),
                    np.ones(n)], axis=1)
    nrm = np.concatenate([nrm / np.linalg.norm(nrm, axis=1, keepdims=True), np.zeros((n, 1))], axis=1).astype(np.float32)
    dcol = ref.texture(uv)
    x = (y.astype(np.float64) + [0.004, -0.003, 0.002]).astype(np.float32)
    scol = dcol.copy()
    return x, y, nrm, scol, dcol


def test_lambda_one_equals_point_to_plane():
    x, y, nrm, sc, dc = _scan()
    grad = ref.color_gradients(y, nrm, dc, 2 * R)
    ev = ref.evaluate(x, y, 1.0, np.eye(3), np.zeros(3), R * R)
    c = ev["p"][ev["idx"] >= 0].mean(axis=0)
    A1, g1 = ref.system(ev, y, nrm, sc, dc, grad, c, 1.0)
    A0, g0 = plane.system(ev, y, nrm, c)
    assert np.array_equal(A1, A0) and np.array_equal(g1, g0)
    a = ref.icp(x, y, nrm, sc, dc, R, lam=1.0, grad=grad, max_iteration=5)
    b = plane.icp(x, y, nrm, R, max_iteration=5)
    assert np.array_equal(a["R"], b["R"]) and np.array_equal(a["t"], b["t"])


@pytest.mark.parametrize("lam,loss,k", [(0.968, None, 1.0), (0.0, None, 1.0), (0.5, "huber", 0.01),
                                        (0.968, "tukey", 0.05)])
def test_float_step_agrees_with_the_exact_step(lam, loss, k):
    x, y, nrm, sc, dc = _scan(1, 300)
    sc = (sc + 0.02 * np.random.default_rng(1).standard_normal(sc.shape)).astype(np.float32)
    grad = ref.color_gradients(y, nrm, dc, 2 * R)
    ev = ref.evaluate(x, y, 1.0, np.eye(3), np.zeros(3), R * R)
    Ru, tu = ref.ColoredUpdate(sc, dc, grad, lam, loss, k)(ev, y, nrm)
    src = np.nonzero(ev["idx"] >= 0)[0]
    corr = np.stack([src, ev["idx"][src]], axis=1)
    e = ref.step_exact(x, y, nrm, sc, dc, grad, corr, 1.0, np.eye(3), np.zeros(3), lam, loss, k)
    tol = 1e-9 * (e["lam_max"] / e["lam_min"])
    np.testing.assert_allclose(Ru, e["R"], rtol=0, atol=tol)
    np.testing.assert_allclose(tu, e["t"], rtol=0, atol=tol)


def test_textured_plane_offset_removed_where_point_to_plane_leaves_it():
    src, dst, nrm, sc, dc, off = ref.textured_plane(step=0.02, extent=0.5)
    col = ref.icp(src, dst, nrm, sc, dc, R, max_iteration=30)
    pp = plane.icp(src, dst, nrm, R, max_iteration=30)
    err_pp = np.linalg.norm(pp["t"][:2] - off[:2])
    err_col = np.linalg.norm(col["t"][:2] - off[:2])
    assert err_pp > 0.99 * np.linalg.norm(off[:2])  # point-to-plane leaves the in-plane offset
    assert err_col < 0.1 * err_pp, (err_col, err_pp)
