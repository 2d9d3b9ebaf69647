"""CPU checks of tests/certifier_reference.py: every exact matrix the certifier boundary tests decompose is exact in
FP64, and LAPACK (oracle/certifier_oracle.py) meets the tolerance rules on them, so the rules are set by the
mathematics and not fitted to the device."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "oracle"))
sys.path.insert(0, HERE)
import certifier_oracle as co  # noqa: E402
import certifier_reference as cr  # noqa: E402

CASES = cr.psd_cases()


@pytest.mark.parametrize("n,kind", CASES, ids=[f"{n}-{k}" for n, k in CASES])
def test_exact_matrix_is_exact_and_lapack_meets_the_bound(n, kind):
    M, P, lam, Q = cr.exact_matrix(n, kind)
    assert cr.exactness(Q, lam), "dyadic bit growth exceeds FP64 for this matrix"
    assert np.array_equal(M, M.T)
    assert np.all(np.diff(lam) >= 0)
    # the product in another summation order, and the positive part from the spectrum, are the same bits
    assert np.array_equal(M, Q @ (lam[:, None] * Q.T))
    assert np.array_equal(P, Q @ (np.maximum(lam, 0)[:, None] * Q.T))
    assert np.array_equal(np.ldexp(M, -40) * 2.0 ** 40, M)   # the scaled copies are exact too
    got = co.nearest_psd(M)
    assert np.linalg.norm(got - P) <= cr.psd_bound(M)
    w = np.linalg.eigvalsh(M)
    assert np.abs(w - lam).max() <= cr.eig_bound(lam)


def test_first_positive_indices_straddle_the_k_slabs():
    for n in cr.PSD_SIZES:
        ps = [n - 1 if k == "first_pos_last" else int(k.split("_")[-1]) for k in cr.first_positive_kinds(n)]
        assert 0 in ps and n - 1 in ps
        if n >= 64:
            assert {p % 16 for p in ps} >= {0, 1, 15}
        for p, k in zip(ps, cr.first_positive_kinds(n)):
            lam = cr.spectrum(n, k)
            assert int(np.argmax(lam > 0)) == p


def test_spectra_have_the_named_shape():
    n = 132
    assert np.all(cr.spectrum(n, "all_positive") > 0) and np.all(cr.spectrum(n, "all_negative") < 0)
    assert np.count_nonzero(cr.spectrum(n, "zeros") == 0) == n // 8
    assert np.unique(cr.spectrum(n, "repeated")).size == 3
    w = np.abs(cr.spectrum(n, "wide"))
    assert w.max() / w.min() >= 2.0 ** 36


def test_bit_growth_is_detected():
    """The exactness check refuses a matrix whose products need more than 53 bits."""
    Q, _ = cr.orthogonal(1028, 3)
    lam = np.ldexp(np.ones(1028), np.arange(1028) % 41 - 20)
    assert not cr.exactness(Q, lam)
    M = (Q * lam).astype(np.longdouble) @ Q.T.astype(np.longdouble)
    assert not np.array_equal((Q * lam) @ Q.T, M)


def test_psd_bound_is_not_vacuous():
    """A rank-one error of a few ulps of ||M|| per entry already exceeds the PSD bound at n = 1028, and the
    eigenvalue bound is far below one spectral gap of the test spectra."""
    M, P, lam, _ = cr.exact_matrix(1028, "first_pos_512")
    assert cr.psd_bound(M) < 1e-9 * np.linalg.norm(M)
    assert cr.eig_bound(lam) < 1e-9


def _random_W(rng, N):
    n = 4 * N + 4
    return rng.standard_normal((n, n)) * np.ldexp(1.0, rng.integers(-8, 9, (n, n)))


@pytest.mark.parametrize("N", [1, 2, 7, 31, 40])
def test_dual_projection_closed_form_meets_the_bound_against_dense(N):
    rng = np.random.default_rng(N)
    W = _random_W(rng, N)
    thp = np.concatenate([[1.0], rng.choice([-1.0, 1.0], N)])
    a = co.get_optimal_dual_projection(W, thp)
    b = co.get_optimal_dual_projection(W, thp, A_inv=co.get_linear_projection(thp))
    assert np.abs(a - b).max() <= cr.dual_bound(W, N)
