"""The exact one-step reference (tests/icp_exact_reference.py) checked without a GPU: against the four numpy
restatements on their clutter fixture, on hand cases whose answer is known in closed form, and the truncated solve on
systems whose rank and solution are known."""
from fractions import Fraction as F

import numpy as np
import pytest

import icp_exact_reference as ex
import icp_generalized_reference as gref
import icp_plane_reference as pref
import icp_reference as ref
import icp_robust_reference as rref


@pytest.fixture(scope="module")
def fixture():
    d = rref.clutter_pair(0, n=300)
    ev = ref.evaluate(d["src"], d["dst"], 1.0, d["R0"], d["t0"], d["r"] ** 2)
    m = ev["idx"] >= 0
    return d, ev, np.stack([np.nonzero(m)[0], ev["idx"][m]], axis=1)


def _close(e, Ru, tu, R0, t0, atol=1e-13):
    """The restatement's step (Ru, tu) composed onto the seed against the exact step: float64 rounding of a
    well-conditioned step (the fixture's conditions are printed by the GPU tests; here gap and lambda_min are O(1))."""
    np.testing.assert_allclose(e["R"], Ru @ R0, rtol=0, atol=atol)
    np.testing.assert_allclose(e["t"], Ru @ t0 + tu, rtol=0, atol=atol)


def test_point_to_point_agrees_with_the_restatement(fixture):
    d, ev, corr = fixture
    e = ex.step_point(d["src"], d["dst"], corr, 1.0, d["R0"], d["t0"])
    assert e["count"] == len(corr) > 100 and e["gap"] > 1.0
    _close(e, *ref.update(ev, d["dst"]), d["R0"], d["t0"])


@pytest.mark.parametrize("loss", [None, "l1", "huber", "cauchy", "gm", "tukey"])
def test_point_to_plane_agrees_with_the_restatement(fixture, loss):
    d, ev, corr = fixture
    e = ex.step_plane(d["src"], d["dst"], d["dst_normals"], corr, 1.0, d["R0"], d["t0"], loss, d["k_plane"])
    assert e["rank"] == 6
    upd = pref.update if loss is None else rref.PlaneUpdate(rref.LOSSES[loss], d["k_plane"])
    _close(e, *(upd(ev, d["dst"], d["dst_normals"])), d["R0"], d["t0"])


@pytest.mark.parametrize("loss", [None, "l1", "huber", "cauchy", "gm", "tukey"])
def test_generalized_agrees_with_the_restatement(fixture, loss):
    d, ev, corr = fixture
    sub = corr[:120]  # the whitening's eigendecompositions at 256 bits take a few ms each
    evs = dict(ev, idx=np.full_like(ev["idx"], -1))
    evs["idx"][sub[:, 0]] = sub[:, 1]
    e = ex.step_generalized(d["src"], d["dst"], d["src_normals"], d["dst_normals"], sub, 1.0, d["R0"], d["t0"], 1e-3,
                            loss, d["k_gicp"])
    assert e["rank"] == 6 and e["used"] == len(sub)
    if loss is None:
        upd = gref.Update(d["src_normals"], 1.0, d["R0"], 1e-3)
    else:
        upd = rref.GicpUpdate(d["src_normals"], 1.0, d["R0"], 1e-3, rref.LOSSES[loss], d["k_gicp"])
    # A's entries have condition up to kappa(M) = 1 / epsilon in float64
    _close(e, *(upd(evs, d["dst"], d["dst_normals"])), d["R0"], d["t0"], atol=1e-11)


# ---- hand cases --------------------------------------------------------------------------------------------------------
def _lattice(k=4):
    g = np.arange(k, dtype=np.float64) * 0.25
    X, Y, Z = np.meshgrid(g, g, g * 0.5, indexing="ij")
    return np.stack([X.ravel(), Y.ravel(), Z.ravel()], axis=1).astype(np.float32)


def test_pure_translation_is_exact():
    x = _lattice()
    tr = np.array([0.125, -0.5, 0.0625])
    y = (x.astype(np.float64) + tr).astype(np.float32)
    corr = np.stack([np.arange(len(x))] * 2, axis=1)
    e = ex.step_point(x, y, corr, 1.0, np.eye(3), np.zeros(3))
    assert np.array_equal(e["R"], np.eye(3)) and np.array_equal(e["t"], tr)
    e = ex.step_plane(x, y, np.tile([1.0, 0.0, 0.0], (len(x), 1)), corr, 1.0, np.eye(3), np.zeros(3))
    assert e["rank"] == 3 and e["x"][3] == F(0.125) and e["x"][:3] == [0, 0, 0]


def test_quarter_turn_about_z_on_a_dyadic_lattice():
    x = _lattice()
    Rz = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
    y = (x.astype(np.float64) @ Rz.T + [0.5, 0.25, -1.0]).astype(np.float32)
    corr = np.stack([np.arange(len(x))] * 2, axis=1)
    e = ex.step_point(x, y, corr, 1.0, np.eye(3), np.zeros(3))
    np.testing.assert_allclose(e["R"], Rz, rtol=0, atol=1e-70 + 1e-16)
    np.testing.assert_allclose(e["t"], [0.5, 0.25, -1.0], rtol=0, atol=1e-15)
    # from the seed Rz^T the step is R_u = Rz^2, and R_u R0, R_u t0 + t_u land on the same motion
    e2 = ex.step_point(x, y, corr, 1.0, Rz.T, np.zeros(3))
    np.testing.assert_allclose(e2["R"], Rz, rtol=0, atol=1e-15)
    np.testing.assert_allclose(e2["t"], [0.5, 0.25, -1.0], rtol=0, atol=1e-15)


@pytest.mark.parametrize("count", [0, 1, 2, 3])
def test_small_counts(count):
    x = np.array([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0]], dtype=np.float32)
    Rz = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
    y = (x.astype(np.float64) @ Rz.T + [0.25, 0.5, 0.75]).astype(np.float32)
    corr = np.stack([np.arange(count)] * 2, axis=1)
    e = ex.step_point(x, y, corr, 1.0, np.eye(3), np.zeros(3))
    if count == 0:
        assert np.array_equal(e["R"], np.eye(3)) and np.array_equal(e["t"], np.zeros(3))
    elif count < 3:  # the translation of the centroids, no rotation
        want = (y[:count].astype(np.float64) - x[:count].astype(np.float64)).mean(axis=0)
        assert np.array_equal(e["R"], np.eye(3)) and np.allclose(e["t"], want, rtol=0, atol=1e-16)
    else:  # three points fix the rotation (sigma_3 = 0, sigma_2 > 0)
        np.testing.assert_allclose(e["R"], Rz, rtol=0, atol=1e-15)
        assert e["sigma"][2] < 1e-60 and e["gap"] > 0.1


def test_collinear_points_compare_the_cost_only():
    """Collinear correspondences leave the rotation about the line free (sigma_2 = sigma_3 = 0), so Kabsch is not unique
    and only the cost can be compared: the exact step reaches the least cost (0 here, the line's image being exactly a
    moved copy of it), which no other step, the float64 SVD's included, undercuts."""
    s = np.arange(8, dtype=np.float64)[:, None] * 0.25
    x = (s * [1.0, 0.5, 0.25]).astype(np.float32)
    y = (s * [0.25, 1.0, -0.5] + [0.5, 0.0, 0.0]).astype(np.float32)  # the same length: 1.3125 = 1 + 1/4 + 1/16
    corr = np.stack([np.arange(8)] * 2, axis=1)
    e = ex.step_point(x, y, corr, 1.0, np.eye(3), np.zeros(3))
    assert e["gap"] < 1e-60
    Ru, tu = ref.update(dict(p=x.astype(np.float64), idx=np.arange(8)), y)  # the same correspondences
    X, Y = x.astype(np.float64), y.astype(np.float64)
    cost = lambda R, t: float(((X @ R.T + t - Y) ** 2).sum())  # noqa: E731
    assert cost(e["R"], e["t"]) < 1e-28
    assert cost(e["R"], e["t"]) <= cost(Ru, tu) + 1e-28


# ---- the truncated solve -----------------------------------------------------------------------------------------------
def test_solve_on_a_diagonal_system():
    A = np.diag([4.0, 1.0, 9.0, 2.0, 0.5, 3.0])
    g = np.array([1.0, -2.0, 3.0, 0.25, 1.0, -6.0])
    x, rank, piv = ex.solve6([[F(v) for v in r] for r in A], [F(v) for v in g])
    assert rank == 6 and piv == [2, 0, 5, 3, 1, 4]  # descending diagonal
    assert x == [-F(g[i]) / F(A[i, i]) for i in range(6)]


def test_solve_truncates_below_the_tolerance_and_takes_the_lowest_index_on_ties():
    tol = F(1e-10) * 8
    A = [[F(0)] * 6 for _ in range(6)]
    for i, v in enumerate([F(8), F(8), tol, tol * (1 + F(1, 2 ** 40)), F(0), F(8)]):
        A[i][i] = v
    g = [F(1)] * 6
    x, rank, piv = ex.solve6(A, g)
    assert piv == [0, 1, 5, 3] and rank == 4  # ties 0, 1, 5 in index order; 2 equals tol (strict > fails)
    assert x == [F(-1, 8), F(-1, 8), 0, -1 / A[3][3], 0, F(-1, 8)]


@pytest.mark.parametrize("k", [1, 2, 3, 4, 5])
def test_solve_on_rank_k_systems(k):
    """A = V diag(d) V^T of rank k with g in its range: the truncated solve reaches rank k and returns the x of
    smallest pivoted support, which satisfies A x = -g exactly."""
    rng = np.random.default_rng(k)
    V = rng.integers(-4, 5, size=(6, k)).astype(np.int64)
    A = [[F(int(v)) for v in row] for row in V @ V.T]
    z = rng.integers(-3, 4, size=k)
    g = [F(int(v)) for v in V @ z]
    x, rank, piv = ex.solve6(A, g)
    assert rank == np.linalg.matrix_rank(V)
    Ax = [sum((A[i][j] * x[j] for j in range(6)), F(0)) for i in range(6)]
    assert Ax == [-v for v in g]
    assert all(x[i] == 0 for i in range(6) if i not in piv)
