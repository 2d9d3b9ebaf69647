"""The restatement's boundary pieces against their definitions (tests/pose_graph_reference.py), CPU only: the GNC-TLS mu
rule at max r-bar = 1/2 and one ulp either side, the 13 rejections before the damping passes 1e8, the log at tied
diagonals and at pi against scipy, and the self-loop probe of tests/test_gpu_pose_graph_boundary.py."""
from fractions import Fraction

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import pose_graph_reference as ref
from test_gpu_pose_graph_boundary import (PI_EXACT, gnc_graph, log_probe, log_rbar, log_readback, overflow_graph,
                                          probe_tau)


@pytest.mark.parametrize("rmax,iters", [(0.5, 1), (np.nextafter(0.5, 0), 1), (np.nextafter(0.5, 1), 2)])
def test_mu_rule_at_half(rmax, iters):
    """1 / (2 r - 1) is +inf at r = 1/2: the restatement must stop with weights 1 there, as below it (mu < 0); one ulp
    above, mu is finite (about 2.3e15), every weight is 1 at once and the unchanged cost stops the next iteration."""
    edges, T, L, unc = gnc_graph([0.1, rmax])
    out = ref.optimize(2, edges, T, L, 1.0, unc)
    assert out["residuals"][2] == rmax
    assert out["iterations"] == iters
    assert (out["weights"] == 1).all() and out["mask"].all()
    if iters == 2:
        with np.errstate(divide="ignore"):
            assert np.isfinite(1.0 / (2.0 * rmax - 1.0))


def test_thirteen_rejections_pass_the_damping_cap():
    lam, k = ref.LAMBDA0, 0
    while not lam > ref.LAMBDA_MAX:
        lam, k = lam * 10.0, k + 1
    assert k == 13
    edges, T, L, unc = overflow_graph()
    tr = []
    with np.errstate(over="ignore", invalid="ignore"):
        out = ref.optimize(5, edges, T, L, 0.05, unc, max_inner_iterations=20, trace=tr)
    assert out["inner_iterations"] == 13 * out["iterations"] and out["iterations"] > 1
    inner = [x for x in tr if x["kind"] == "inner"]
    assert all(x["outcome"] == "reject" for x in inner if x["lam"] < 1e8)
    assert all(x["outcome"] == "reject-stop" for x in inner if x["lam"] >= 1e8)


@pytest.mark.parametrize("name", sorted(PI_EXACT))
def test_log_at_pi_with_tied_diagonals(name):
    """At theta = pi exactly v = 0: the first of the tied columns gives +pi a, which scipy's log matches up to sign."""
    R, a = PI_EXACT[name]
    w = ref.so3_log(R)
    np.testing.assert_allclose(w, np.pi * a, rtol=0, atol=1e-12)
    s = Rotation.from_matrix(R).as_rotvec()
    assert min(np.abs(s - w).max(), np.abs(s + w).max()) < 1e-12


@pytest.mark.parametrize("axis", [(1.0, 1.0, 0.0), (1.0, 1.0, 1.0), (1.0, -1.0, 0.0), (0.48, -0.6, 0.64)])
@pytest.mark.parametrize("theta", [np.arccos(-0.9) + 1e-9, 3.0, np.pi - 1e-9])
def test_log_near_pi_against_scipy(axis, theta):
    a = np.asarray(axis) / np.linalg.norm(axis)
    R = Rotation.from_rotvec(theta * a).as_matrix()
    np.testing.assert_allclose(ref.so3_log(R), Rotation.from_matrix(R).as_rotvec(), rtol=0, atol=1e-12)
    np.testing.assert_allclose(ref.so3_log(R.T.copy()), -theta * a, rtol=0, atol=1e-12)


def test_probe_tau_is_the_device_order():
    """probe_tau sums -(R^T t) as ((R[0,r] t0 + R[1,r] t1) + R[2,r] t2): each step rounded once, so within 1.5 ulps
    (of the largest partial) of the exact value, and exactly that value when every product and sum is representable."""
    rng = np.random.default_rng(1)
    for _ in range(20):
        R = Rotation.from_rotvec(rng.normal(size=3) * 1.5).as_matrix()
        t = rng.normal(size=3) * 3
        got = probe_tau(R, t)
        for r in range(3):
            p = [float(R[q, r]) * float(t[q]) for q in range(3)]
            assert got[r] == -((p[0] + p[1]) + p[2])
            exact = -sum(Fraction(float(R[q, r])) * Fraction(float(t[q])) for q in range(3))
            assert abs(Fraction(float(got[r])) - exact) <= 3 * Fraction(float(np.spacing(max(abs(x) for x in p))))
    P = np.array([[0.0, 1, 0], [0, 0, -1], [-1, 0, 0]])
    assert np.array_equal(probe_tau(P, [2.0, -3.0, 0.5]), -(P.T @ [2.0, -3.0, 0.5]))


def test_log_probe_reads_back_the_log():
    """The probe's r-bar, rounded as the device rounds it, gives omega back to about ulp(theta)."""
    for theta, a in [(0.0, (1, 0, 0)), (1e-7, (0, 1, 0)), (0.5, (0.48, -0.6, 0.64)), (3.0, (1, -1, 0)),
                     (np.pi - 1e-9, (0.48, -0.6, 0.64))]:
        a = np.asarray(a, dtype=np.float64) / np.linalg.norm(a)
        R = Rotation.from_rotvec(theta * a).as_matrix()
        _, Ls, tau2 = log_probe(R, theta)
        assert tau2 > 1.9 * theta
        w = ref.so3_log(R.T.copy())
        back = np.array([log_readback(log_rbar(w[k], tau2), tau2) for k in range(3)])
        assert np.abs(back - w).max() <= 8 * np.spacing(max(theta, 1.0 if theta == 0 else theta))
        for k in range(3):
            assert Ls[k][k, k] == Ls[k][k, 5] == Ls[k][5, 5] == 1.0 and Ls[k].sum() == 4.0
