"""CPU checks of tests/dense_cholesky_reference.py: the exact systems are exact in the device's order and in LAPACK's,
each failure variant fails at its stated column, and the backward-error bounds hold for scipy's factor and solve and
fail for a factor perturbed by 8u in one entry."""
import numpy as np
import pytest
import scipy.linalg

import dense_cholesky_reference as dc


@pytest.mark.parametrize("n", [0, 1, 2, 31, 32, 33, 64, 65, 97, 130, 193])
@pytest.mark.parametrize("density", [0.1, 0.6])
def test_exact_systems_are_exact_in_any_order(n, density):
    rng = np.random.default_rng(1000 * n + int(10 * density))
    A, b, L, x = dc.exact_system(rng, n, density)
    assert np.array_equal(A, A.T)
    if n > 1:
        assert len(set(np.diag(L).tolist())) > 1 and (np.diag(L) != 1).any()  # divisions and square roots show
    got, info = dc.right_looking(A)
    assert info == 0 and got.tobytes() == L.tobytes()
    for nb in (1, 7, 64):  # other panel widths: the same bits
        assert dc.right_looking(A, nb)[0].tobytes() == L.tobytes()
    if n:
        assert np.linalg.cholesky(A).tobytes() == L.tobytes()
        assert scipy.linalg.cho_solve((L, True), b).tobytes() == x.tobytes()
    assert dc.substitute(L, b).tobytes() == x.tobytes()


def test_exact_system_at_the_largest_size():
    rng = np.random.default_rng(834)
    A, b, L, x = dc.exact_system(rng, 834)
    assert np.linalg.cholesky(A).tobytes() == L.tobytes()
    assert dc.substitute(L, b).tobytes() == x.tobytes()


def test_the_magnitude_check_refuses_an_inexact_system():
    rng = np.random.default_rng(3)
    with pytest.raises(AssertionError):
        dc.exact_system(rng, 64, density=1.0, off_max=2.0 ** 20)


@pytest.mark.parametrize("variant", dc.VARIANTS)
@pytest.mark.parametrize("n,j", [(33, 1), (33, 32), (96, 31), (96, 64), (190, 65), (190, 189), (70, 33)])
def test_failure_variants_fail_at_their_column(variant, n, j):
    rng = np.random.default_rng(7 * n + j)
    A, b, L, x = dc.exact_system(rng, n)
    Af, info = dc.failure(A, L, variant, j)
    assert info == j + 1
    got, got_info = dc.right_looking(Af)
    assert got_info == info
    # the finished panels are the exact L (with the NaN row for a NaN below the diagonal)
    c = (j // dc.NB) * dc.NB
    want = dc.finished_columns(L, variant, j)
    assert np.array_equal(got[:, :c], want, equal_nan=True)
    if variant in ("zero", "negative"):
        assert got[:, :c].tobytes() == want.tobytes()
        assert np.isnan(want).sum() == 0
        with pytest.raises(np.linalg.LinAlgError):  # LAPACK agrees (it does not test NaN pivots)
            np.linalg.cholesky(Af)


@pytest.mark.parametrize("n,kappa", [(1, 1.0), (5, 1e3), (40, 1e6), (96, 1e9), (64, 1e12), (200, 1e4)])
def test_bounds_hold_for_scipy(n, kappa):
    rng = np.random.default_rng(n)
    A = dc.spd(rng, n, kappa)
    x_true = rng.standard_normal(n)
    b = A @ x_true
    c, low = scipy.linalg.cho_factor(A, lower=True)
    Lh = np.tril(c)
    xh = scipy.linalg.cho_solve((c, low), b)
    assert dc.factor_violation(A, Lh) <= 1.0
    assert dc.solve_violation(A, b, Lh, xh) <= 1.0
    fb = dc.forward_bound(A, Lh)
    assert fb is not None
    assert dc.forward_error(xh, dc.longdouble_solve(A, b)) <= fb


def test_bounds_hold_for_a_nearly_singular_matrix():
    rng = np.random.default_rng(5)
    A = dc.nearly_singular(rng, 120, 100)
    b = rng.standard_normal(120)
    c, low = scipy.linalg.cho_factor(A, lower=True)
    assert dc.factor_violation(A, np.tril(c)) <= 1.0
    assert dc.solve_violation(A, b, np.tril(c), scipy.linalg.cho_solve((c, low), b)) <= 1.0


@pytest.mark.parametrize("n", [2, 3])
def test_factor_bound_fails_for_a_perturbed_factor(n):
    """L^(0, 0) off by 8u: (L^ L^T)(0, 0) moves by about 16u L^(0,0)^2 while the bound allows (2 n + 2) u of it."""
    rng = np.random.default_rng(11 + n)
    A = dc.spd(rng, n, 10.0)
    Lh = np.tril(scipy.linalg.cho_factor(A, lower=True)[0])
    assert dc.factor_violation(A, Lh) <= 1.0
    P = Lh.copy()
    P[0, 0] = P[0, 0] * (1.0 + 8 * dc.U)
    assert dc.factor_violation(A, P) > 1.0
    P = Lh.copy()
    P[0, 0] = P[0, 0] * (1.0 - 8 * dc.U)
    assert dc.factor_violation(A, P) > 1.0


def test_solve_bound_fails_for_a_perturbed_solution():
    rng = np.random.default_rng(17)
    A = dc.spd(rng, 3, 10.0)
    b = rng.standard_normal(3)
    c, low = scipy.linalg.cho_factor(A, lower=True)
    xh = scipy.linalg.cho_solve((c, low), b)
    assert dc.solve_violation(A, b, np.tril(c), xh) <= 1.0
    k = int(np.argmax(np.abs(xh)))
    xp = xh.copy()
    xp[k] = xp[k] * (1.0 + 64 * dc.U)
    assert dc.solve_violation(A, b, np.tril(c), xp) > 1.0


def test_batch_cap_on_an_h100():
    """227 KB of opt-in shared memory (the H100's 232448 bytes): K = 139, n = 834 in 230928 bytes."""
    assert dc.batch_cap(232448) == 139
    assert dc.batch_smem(834) == 230928 and dc.batch_smem(840) > 232448
