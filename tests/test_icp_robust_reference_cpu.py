"""The numpy robust-kernel restatement (tests/icp_robust_reference.py) against independent facts: each weight is
rho'(r) / r of its published loss, L2 reproduces the point-to-plane and generalized references, the device's A~ form
equals Open3D's per-row form, normal signs do not matter, Tukey drops what lies beyond k, the device-order SVD gives
M^-1/2, and on a cluttered scan Tukey lands far closer to the truth than L2.  No GPU."""
import numpy as np
import pytest

import icp_generalized_reference as gref
import icp_plane_reference as pref
import icp_robust_reference as ref
from test_icp_generalized_reference_cpu import _random_case

L = ref.LOSSES


@pytest.mark.parametrize("name,k", [("l2", 1.0), ("l1", 1.0), ("huber", 0.3), ("cauchy", 0.3), ("gm", 0.09),
                                    ("tukey", 0.3)])
def test_weight_is_the_derivative_of_rho_over_r(name, k):
    r = np.array([-0.8, -0.31, -0.2, -0.05, 0.01, 0.07, 0.25, 0.29, 0.33, 0.6, 1.7])
    h = 1e-6
    d = (ref.rho(L[name], k, r + h) - ref.rho(L[name], k, r - h)) / (2 * h)
    np.testing.assert_allclose(ref.weight(L[name], k, r), d / r, rtol=1e-6, atol=1e-9)
    # the sign of a residual never matters
    assert np.array_equal(ref.weight(L[name], k, r), ref.weight(L[name], k, -r))


def test_weights_at_their_edges():
    assert np.isinf(ref.weight(L["l1"], 0.0, 0.0))
    assert ref.weight(L["huber"], 0.5, 0.5) == 1.0 and ref.weight(L["huber"], 0.5, 1.0) == 0.5
    assert ref.weight(L["tukey"], 0.5, 0.5) == 0.0 and ref.weight(L["tukey"], 0.5, 0.5000001) == 0.0
    assert ref.weight(L["tukey"], 0.5, 0.0) == 1.0 and ref.weight(L["cauchy"], 0.5, 0.0) == 1.0
    assert ref.weight(L["gm"], 0.25, 0.0) == 4.0  # k / k^2: GM's k is in squared residual units


def _plane_case(seed, n=400):
    rng = np.random.default_rng(seed)
    P = rng.uniform(-1, 1, (n, 3))
    Q = (P + rng.normal(scale=0.05, size=P.shape)).astype(np.float32)
    N = rng.normal(size=(n, 3))
    N /= np.linalg.norm(N, axis=1, keepdims=True)
    return dict(p=P, idx=np.arange(n)), Q, np.concatenate([N, np.zeros((n, 1))], axis=1).astype(np.float32)


def test_l2_and_huge_huber_reproduce_point_to_plane():
    ev, Q, N = _plane_case(1)
    c = ev["p"].mean(axis=0)
    A0, g0 = pref.system(ev, Q, N, c)
    for loss, k in ((L["l2"], 1.0), (L["huber"], 1e6)):
        A, g = ref.plane_system(ev, Q, N, c, loss, k)
        # the same products (w = 1 exactly); numpy may order J^T J's sums differently from w J^T J's
        np.testing.assert_allclose(A, A0, rtol=1e-14, atol=1e-14 * np.abs(A0).max())
        np.testing.assert_allclose(g, g0, rtol=1e-14, atol=1e-14 * np.abs(g0).max())


@pytest.mark.parametrize("seed,s,epsilon", [(0, 1.0, 1e-3), (1, 1.7, 1e-3), (2, 0.6, 0.05)])
def test_l2_and_huge_huber_reproduce_generalized(seed, s, epsilon):
    P, Q, Ms, Nt, R = _random_case(seed)
    ev = dict(p=P, idx=np.arange(len(P)))
    c = P.mean(axis=0)
    A0, g0 = gref.system(ev, Q, Ms, Nt, R, s, epsilon, c)
    A, g = ref.gicp_system(ev, Q, Ms, Nt, R, s, epsilon, c, L["l2"], 1.0)
    # W W = M^-1 only to rounding: the row form and the adjugate form agree to a few ulps of the conditioning
    assert np.abs(A - A0).max() <= 1e-9 * np.abs(A0).max()
    assert np.abs(g - g0).max() <= 1e-9 * np.abs(g0).max()
    Ah, gh = ref.gicp_system(ev, Q, Ms, Nt, R, s, epsilon, c, L["huber"], 1e6)
    assert np.array_equal(Ah, A) and np.array_equal(gh, g)


@pytest.mark.parametrize("name,k", [("l1", 1.0), ("huber", 0.5), ("cauchy", 0.5), ("gm", 0.25), ("tukey", 1.0)])
def test_atilde_form_equals_the_per_row_form(name, k):
    P, Q, Ms, Nt, R = _random_case(3)
    ev = dict(p=P, idx=np.arange(len(P)))
    args = (ev, Q, Ms, Nt, R, 1.3, 1e-3, P.mean(axis=0), L[name], k)
    A, g = ref.gicp_system(*args)
    At, gt = ref.gicp_system_atilde(*args)
    assert np.abs(A - At).max() <= 1e-11 * np.abs(A).max()
    assert np.abs(g - gt).max() <= 1e-11 * np.abs(g).max()


@pytest.mark.parametrize("name,k", [("l1", 1.0), ("cauchy", 0.5), ("tukey", 1.0)])
def test_normal_signs_change_nothing(name, k):
    rng = np.random.default_rng(11)
    ev, Q, N = _plane_case(4)
    c = ev["p"].mean(axis=0)
    N2 = N.copy()
    N2[rng.random(len(N)) < 0.5] *= -1
    A, g = ref.plane_system(ev, Q, N, c, L[name], k * 0.1)
    A2, g2 = ref.plane_system(ev, Q, N2, c, L[name], k * 0.1)
    assert np.array_equal(A, A2) and np.array_equal(g, g2)
    P, Q, Ms, Nt, R = _random_case(6)
    ev = dict(p=P, idx=np.arange(len(P)))
    Ms2, Nt2 = Ms.copy(), Nt.copy()
    Ms2[rng.random(len(P)) < 0.5] *= -1
    Nt2[rng.random(len(P)) < 0.5] *= -1
    for whiten in (ref.whitening_eigh, ref.whitening_svd3):
        args = (R, 1.3, 1e-3, P.mean(axis=0), L[name], k)
        A, g = ref.gicp_system_atilde(ev, Q, Ms, Nt, *args, whiten=whiten)
        A2, g2 = ref.gicp_system_atilde(ev, Q, Ms2, Nt2, *args, whiten=whiten)
        assert np.array_equal(A, A2) and np.array_equal(g, g2)


def test_tukey_beyond_k_drops_the_correspondence():
    ev, Q, N = _plane_case(5)
    c = ev["p"].mean(axis=0)
    r = np.abs(np.einsum("ni,ni->n", ev["p"] - Q.astype(np.float64), N[:, :3].astype(np.float64)))
    k = float(np.median(r))
    A, g = ref.plane_system(ev, Q, N, c, L["tukey"], k)
    near = r <= k
    ev_n = dict(p=ev["p"][near], idx=np.arange(near.sum()))
    An, gn = ref.plane_system(ev_n, Q[near], N[near], c, L["tukey"], k)
    np.testing.assert_allclose(A, An, rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(g, gn, rtol=1e-12, atol=1e-14)
    # every residual beyond k: no system at all, so the step is the identity
    A0, g0 = ref.plane_system(ev, Q, N, c, L["tukey"], float(r.min()) * 0.5)
    assert not A0.any() and not g0.any()
    Ru, tu = ref._step(A0, g0, c)
    assert np.array_equal(Ru, np.eye(3)) and not tu.any()
    P, Qg, Ms, Nt, R = _random_case(7)
    evg = dict(p=P, idx=np.arange(len(P)))
    A1, g1 = ref.gicp_system(evg, Qg, Ms, Nt, R, 1.0, 1e-3, P.mean(axis=0), L["tukey"], 1e-9)
    assert not A1.any() and not g1.any()


def test_l1_zero_residual_is_dropped_not_nan():
    """Exact recovery reaches r = 0, where L1's weight is infinite: the correspondence leaves the system."""
    ev, Q, N = _plane_case(8)
    P = ev["p"].copy()
    P[:50] = Q[:50].astype(np.float64)  # zero residual on the first 50
    ev = dict(p=P, idx=ev["idx"])
    c = P.mean(axis=0)
    A, g = ref.plane_system(ev, Q, N, c, L["l1"], 0.0)
    assert np.isfinite(A).all() and np.isfinite(g).all()
    ev_r = dict(p=P[50:], idx=np.arange(len(P) - 50))
    Ar, gr = ref.plane_system(ev_r, Q[50:], N[50:], c, L["l1"], 0.0)
    np.testing.assert_allclose(A, Ar, rtol=1e-12)
    np.testing.assert_allclose(g, gr, rtol=1e-12)


def _aligned_M(n, s, epsilon, rng, jitter=0.0):
    """M = s^2 C(m) + C(n) with m = n (plus a jitter): the eigenvalue (s^2 + 1) is repeated."""
    m = n + jitter * rng.normal(size=n.shape)
    return s * s * gref.covariance(m, epsilon) + gref.covariance(n, epsilon)


@pytest.mark.parametrize("s,epsilon,jitter", [(1.0, 1e-3, 0.0), (1.7, 1e-3, 0.0), (0.4, 0.05, 0.0), (2.5, 1e-3, 1e-9),
                                              (1.0, 1e-3, 0.3)])
def test_device_svd_whitening_matches_eigh(s, epsilon, jitter):
    """W from rotation_reference.svd3 (the device's Jacobi, step for step) against numpy.linalg.eigh, including
    aligned normals (a repeated eigenvalue) with s != 1.  Tolerance: 5e-13 of ||W||_2 = 1 / sqrt(sigma_min) (the
    largest difference seen is 1.5e-13, at epsilon = 1e-3 where sigma spans three decades).  The difference is eigh's
    as much as the Jacobi's: W M W - I is smaller with the device's W than with eigh's."""
    rng = np.random.default_rng(int(s * 100) + int(jitter * 1e9))
    n = rng.normal(size=(200, 3))
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    M = _aligned_M(n, s, epsilon, rng, jitter)
    We, se = ref.whitening_eigh(M)
    Ws, ss = ref.whitening_svd3(M)
    err = np.abs(We - Ws).max(axis=(1, 2)) * np.sqrt(se.min(axis=1))
    assert (err <= 5e-13).all()
    np.testing.assert_allclose(np.sort(ss, axis=1), np.sort(se, axis=1), rtol=1e-12)
    I = np.eye(3)
    res_s = np.abs(np.einsum("nab,nbc,ncd->nad", Ws, M, Ws) - I).max()
    res_e = np.abs(np.einsum("nab,nbc,ncd->nad", We, M, We) - I).max()
    assert res_s <= res_e and res_s < 1e-12


@pytest.fixture(scope="module")
def clutter():
    return ref.clutter_pair(0, n=1500)


def test_clutter_fixture_tukey_point_to_plane(clutter):
    f = clutter
    kw = dict(R=f["R0"], t=f["t0"], max_iteration=30)
    l2 = ref.icp_plane(f["src"], f["dst"], f["dst_normals"], f["r"], L["l2"], **kw)
    tk = ref.icp_plane(f["src"], f["dst"], f["dst_normals"], f["r"], L["tukey"], f["k_plane"], **kw)
    e_l2 = ref.pose_error(l2["R"], l2["t"], f["R"], f["t"])
    e_tk = ref.pose_error(tk["R"], tk["t"], f["R"], f["t"])
    print(e_l2, e_tk)
    assert e_tk * 10 <= e_l2 and e_l2 > ref.pose_error(f["R0"], f["t0"], f["R"], f["t"])
    # L2 is the unweighted reference itself
    l2p = pref.icp(f["src"], f["dst"], f["dst_normals"], f["r"], **kw)
    np.testing.assert_allclose(l2["R"], l2p["R"], atol=1e-12)


def test_clutter_fixture_tukey_generalized(clutter):
    f = clutter
    kw = dict(R=f["R0"], t=f["t0"], max_iteration=30)
    l2 = ref.icp_gicp(f["src"], f["dst"], f["src_normals"], f["dst_normals"], f["r"], L["l2"], **kw)
    tk = ref.icp_gicp(f["src"], f["dst"], f["src_normals"], f["dst_normals"], f["r"], L["tukey"], f["k_gicp"], **kw)
    e_l2 = ref.pose_error(l2["R"], l2["t"], f["R"], f["t"])
    e_tk = ref.pose_error(tk["R"], tk["t"], f["R"], f["t"])
    print(e_l2, e_tk)
    assert e_tk * 10 <= e_l2 and e_l2 > ref.pose_error(f["R0"], f["t0"], f["R"], f["t"])
    l2g = gref.icp(f["src"], f["dst"], f["src_normals"], f["dst_normals"], f["r"], **kw)
    np.testing.assert_allclose(l2["R"], l2g["R"], atol=1e-9)
