"""GPU parity tests of the certifier (`pytest -m gpu`): tzr_certify and its building blocks through the C-ABI against
the reference's own fixtures (tests/golden/certification_*, tolerance 1e-7 as in certification-test.cc:29) and against
oracle/certifier_oracle.py."""
import importlib
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
import certifier_oracle as co  # noqa: E402
import certifier_fixtures as cf  # noqa: E402

capi = importlib.import_module("teaser-plusplus_b200.capi")
synth = importlib.import_module("teaser-plusplus_b200.synth")

pytestmark = pytest.mark.gpu
TOL = 1e-7
SMALL = cf.cases("small")
LARGE = cf.cases("large")


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


@pytest.mark.parametrize("c", SMALL, ids=[c["name"] for c in SMALL])
def test_initial_matrix_and_mu_from_fixture_blocks(ctx, c):
    """M_init = D^T Q_cost D - mu J - lambda_bar_init assembled from the reference's stored Q_cost, block_diag_omega,
    lambda_bar_init and mu (GetQCost / GetBlockDiagOmega / GetLambdaGuess fixtures)."""
    N = c["v1"].shape[1]
    nb, cb = c["params"]["noise_bound"], c["params"]["cbar2"]
    M, mu = ctx.certifier_initial_matrix(c["R_est"], c["v1"], c["v2"], c["theta_est"], noise_bound=nb, cbar2=cb)
    D = c["block_diag_omega"]
    want = D.T @ c["Q_cost"] @ D - c["lambda_bar_init"]
    want[:4, :4] -= c["mu"] * np.eye(4)
    assert abs(mu - c["mu"]) < TOL
    assert np.abs(M - want).max() < TOL


@pytest.mark.parametrize("c", SMALL, ids=[c["name"] for c in SMALL])
def test_dual_projection_fixture(ctx, c):
    """GetOptimalDualProjection (certification-test.cc:448-482): W_1st_iter -> W_dual_1st_iter."""
    Wd = ctx.certifier_dual_projection(c["W_1st_iter"], c["theta_est"])
    assert np.abs(Wd - c["W_dual_1st_iter"]).max() < TOL


@pytest.mark.parametrize("c", SMALL + LARGE, ids=[c["name"] for c in SMALL + LARGE])
def test_certify_trajectory_fixture(ctx, c):
    """Certify / LargeInstance (certification-test.cc:499-527)."""
    mi = c["params"].get("max_iterations", 200)
    r = ctx.certify(c["R_est"], c["v1"], c["v2"], c["theta_est"], noise_bound=c["params"]["noise_bound"],
                    cbar2=c["params"]["cbar2"], max_iterations=mi)
    want = c["suboptimality_traj"]
    assert len(r["suboptimality_traj"]) == len(want)
    assert np.abs(r["suboptimality_traj"] - want).max() < TOL
    assert abs(r["best_suboptimality"] - want.min()) < TOL
    assert r["is_optimal"] == bool(want.min() < 1e-3)


@pytest.mark.parametrize("N,seed", [(100, 0), (100, 1), (200, 2)])
def test_random_instances_certify_optimal(ctx, N, seed):
    """Random100Points / RandomLargeInstances (certification-test.cc:529-644): exact rotation, 10 % outliers ->
    certified optimal with a tiny gap; and the same trajectory as the oracle."""
    rng = np.random.default_rng(seed)
    v1 = rng.uniform(-1, 1, size=(3, N))
    R = synth.random_rotation(rng)
    v2 = R @ v1
    theta = np.ones(N)
    k0 = int(N * 0.9)
    v2[:, k0:] = rng.uniform(-1, 1, size=(3, N - k0)) * 5 + 5
    theta[k0:] = -1
    r = ctx.certify(R, v1, v2, theta, noise_bound=0.01, cbar2=1.0)
    assert r["is_optimal"] and r["best_suboptimality"] <= 1e-5
    o = co.certify(R, v1, v2, theta, 0.01, 1.0)
    assert len(o["suboptimality_traj"]) == len(r["suboptimality_traj"])
    assert np.abs(o["suboptimality_traj"] - r["suboptimality_traj"]).max() < 1e-6


def test_bool_theta_and_iteration_cap(ctx):
    c = SMALL[1]
    kw = dict(noise_bound=c["params"]["noise_bound"], cbar2=c["params"]["cbar2"])
    r1 = ctx.certify(c["R_est"], c["v1"], c["v2"], c["theta_est"], **kw)
    r2 = ctx.certify(c["R_est"], c["v1"], c["v2"], c["theta_est"] > 0, **kw)
    assert np.array_equal(r1["suboptimality_traj"], r2["suboptimality_traj"])
    r3 = ctx.certify(c["R_est"], c["v1"], c["v2"], c["theta_est"], max_iterations=3, **kw)
    assert len(r3["suboptimality_traj"]) == 3 and not r3["is_optimal"]
    assert np.abs(r3["suboptimality_traj"] - c["suboptimality_traj"][:3]).max() < TOL


def test_single_entry_launch_counts(ctx):
    """tzr_certify with k iterations (sub_optimality < 0: it never stops early) launches 16k + 2: the setup's 3
    kernels, per iteration 13 kernels and 2 cusolverDnDsyevd calls, and an update after every iteration but the last.
    The building blocks: initial matrix 3, nearest-PSD step 4 (one of them Dsyevd), dual projection 5."""
    c = SMALL[0]
    args = (c["R_est"], c["v1"], c["v2"], c["theta_est"])
    kw = dict(noise_bound=c["params"]["noise_bound"], cbar2=c["params"]["cbar2"])

    def launches(fn):
        before = ctx.kernel_launches()
        fn()
        return ctx.kernel_launches() - before

    for k in (1, 2, 5):
        assert launches(lambda: ctx.certify(*args, max_iterations=k, sub_optimality=-1.0, **kw)) == 16 * k + 2
    assert launches(lambda: ctx.certifier_initial_matrix(*args, **kw)) == 3
    assert launches(lambda: ctx.certifier_psd_projection(c["W_1st_iter"])) == 4
    assert launches(lambda: ctx.certifier_dual_projection(c["W_1st_iter"], c["theta_est"])) == 5


def test_solve_then_certify_end_to_end(ctx):
    """solve() -> DRSCertifier on the clique's chain TIMs with the rotation inlier mask, the way the reference's
    certification example chains them."""
    pr = synth.config_problem("C2", 1, n=600)
    p = capi.default_params(noise_bound=pr["noise_bound"], cbar2=1.0, estimate_scaling=0, rotation_cost_threshold=1e-12)
    res = ctx.solve(pr["src"], pr["dst"], p)
    cl = res["clique"]
    m = len(cl)
    src_t = (pr["src"][cl[(np.arange(m) + 1) % m]] - pr["src"][cl]).T
    dst_t = (pr["dst"][cl[(np.arange(m) + 1) % m]] - pr["dst"][cl]).T
    r = ctx.certify(res["R"], src_t, dst_t, res["rot_inliers"], noise_bound=2 * pr["noise_bound"], cbar2=1.0)
    o = co.certify(res["R"], src_t, dst_t, res["rot_inliers"], 2 * pr["noise_bound"], 1.0)
    assert len(r["suboptimality_traj"]) == len(o["suboptimality_traj"])
    assert np.abs(r["suboptimality_traj"] - o["suboptimality_traj"]).max() < 1e-6 * max(1.0, o["suboptimality_traj"].max())
    assert r["is_optimal"] == o["is_optimal"]


def test_pybind_certifier_matches_fixture():
    """teaserpp_python.DRSCertifier (reference binding names, teaserpp_python.cc:249-291) through the C++ façade."""
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    host = os.path.join(root, "teaser-plusplus_b200", "host")
    subprocess.check_call(["make", "-s", "-C", host])
    sys.path.insert(0, os.path.join(host, "python"))
    import teaserpp_python as tpp
    c = SMALL[0]
    p = tpp.DRSCertifier.Params()
    p.noise_bound = c["params"]["noise_bound"]
    p.cbar2 = c["params"]["cbar2"]
    p.eig_decomposition_solver = tpp.DRSCertifier.EIG_SOLVER_TYPE.EIGEN
    cert = tpp.DRSCertifier(p)
    r = cert.certify(c["R_est"], c["v1"], c["v2"], c["theta_est"])
    assert np.abs(np.asarray(r.suboptimality_traj) - c["suboptimality_traj"]).max() < TOL
    assert r.is_optimal and abs(r.best_suboptimality - c["suboptimality_traj"].min()) < TOL
    r2 = cert.certify(c["R_est"], c["v1"], c["v2"], c["theta_est"] > 0)   # bool overload (certification.cc:22-38)
    assert np.array_equal(np.asarray(r2.suboptimality_traj), np.asarray(r.suboptimality_traj))
    assert "CertificationResult" in repr(r)
