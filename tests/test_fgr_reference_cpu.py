"""The premises of tests/fgr_reference.py, the numpy restatement of Fast Global Registration (include/teaser_b200.h,
DESIGN.md §3.20) that the GPU tests hold the device to: exact recovery, the unweighted limit of one step, the mu
schedule of both scale modes and the transform back to the input frame."""
import numpy as np
import pytest

import fgr_reference as fr


def rot(axis, angle):
    a = np.asarray(axis, dtype=np.float64)
    a = a / np.linalg.norm(a)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(angle) * K + (1 - np.cos(angle)) * K @ K


def scene(n, outlier_rate, seed, scale=1.0, offset=(0.0, 0.0, 0.0), angle=0.6):
    """float32 clouds x (n) and y = R x + t (exactly, in float64, then rounded to float32), and n correspondences of
    which a fraction are random pairs."""
    rng = np.random.default_rng(seed)
    x = (rng.uniform(-1, 1, (n, 3)) * scale + np.asarray(offset)).astype(np.float32)
    R = rot(rng.normal(size=3), angle)
    t = rng.uniform(-0.5, 0.5, 3) * scale
    y = (x.astype(np.float64) @ R.T + t).astype(np.float32)
    corr = np.stack([np.arange(n), np.arange(n)], axis=1)
    m = int(round(outlier_rate * n))
    bad = rng.choice(n, m, replace=False)
    corr[bad, 1] = rng.integers(0, n, m)
    return x, y, corr, R, t


def fit(x, y):
    """Least-squares rigid fit of y ~ R x + t over float64 copies (Kabsch): the truth of the float32-rounded clouds."""
    x, y = x.astype(np.float64), y.astype(np.float64)
    mx, my = x.mean(0), y.mean(0)
    U, _, Vt = np.linalg.svd((x - mx).T @ (y - my))
    D = np.diag([1, 1, np.sign(np.linalg.det(Vt.T @ U.T))])
    R = Vt.T @ D @ U.T
    return R, my - R @ mx


@pytest.mark.parametrize("outlier_rate", [0.0, 0.5, 0.9])
def test_noise_free_recovery_with_outliers(outlier_rate):
    # float32 rounding of y makes the inliers consistent to ~1e-7 relative: the truth is the float64 fit of the inlier
    # pairs as stored; mu is driven far below that (max_dist 1e-9) so that no outlier keeps a weight that could bias it
    x, y, corr, _, _ = scene(1000, outlier_rate, seed=3)
    inl = corr[:, 0] == corr[:, 1]
    R_fit, t_fit = fit(x[corr[inl, 0]], y[corr[inl, 1]])
    res = fr.fgr(x, y, corr, maximum_correspondence_distance=1e-9, iteration_number=160)
    assert res["converged"] == 1 and res["iterations"] == 160
    # the float32 rounding of y leaves the inliers consistent only to ~1e-8, where FGR's weights and the plain fit
    # settle slightly apart; FGR's residual over the inlier pairs must match the least-squares fit's to 1e-9 (the
    # exact-points test below recovers the truth itself to 1e-9)
    X, Y = x[corr[inl, 0]].astype(np.float64), y[corr[inl, 1]].astype(np.float64)
    e_fgr = np.sqrt(((X @ res["R"].T + res["t"] - Y) ** 2).sum(1).mean())
    e_fit = np.sqrt(((X @ R_fit.T + t_fit - Y) ** 2).sum(1).mean())
    assert e_fgr <= e_fit + 1e-9, (e_fgr, e_fit)
    assert np.abs(res["R"] - R_fit).max() < 1e-6 and np.abs(res["t"] - t_fit).max() < 1e-6


@pytest.mark.parametrize("outlier_rate", [0.0, 0.5, 0.9])
def test_exact_recovery_on_exact_points(outlier_rate):
    # clouds whose float32 values satisfy y = R x + t exactly to float64 rounding: R a quarter turn about z (a signed
    # permutation) and t a small dyadic vector, so the ground truth is recovered to 1e-9
    rng = np.random.default_rng(7)
    x = rng.integers(-512, 512, (800, 3)).astype(np.float32) / 256
    R = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
    t = np.array([0.25, -0.5, 0.125])
    y = (x.astype(np.float64) @ R.T + t).astype(np.float32)
    assert np.array_equal(y.astype(np.float64), x.astype(np.float64) @ R.T + t)
    corr = np.stack([np.arange(800), np.arange(800)], axis=1)
    m = int(round(outlier_rate * 800))
    bad = rng.choice(800, m, replace=False)
    corr[bad, 1] = rng.integers(0, 800, m)
    res = fr.fgr(x, y, corr, maximum_correspondence_distance=1e-9, iteration_number=200)
    assert np.abs(res["R"] - R).max() < 1e-9 and np.abs(res["t"] - t).max() < 1e-9, (res["R"], res["t"])


def test_huge_mu_step_is_the_unweighted_least_squares_step():
    x, y, corr, _, _ = scene(300, 0.3, seed=11)
    p, q, info = fr.normalise(x, y, corr)
    trace = []
    fr.optimise(p, q, 1e30, iteration_number=1, max_dist=0.025, decrease_mu=0, trace=trace)
    assert trace[0]["mu"] == 1e30
    assert np.all(np.abs(trace[0]["w"] - 1.0) <= 4e-16)
    # the unweighted linearisation about T = I, stacked and solved independently
    z, one = np.zeros(len(p)), np.ones(len(p))
    J = np.concatenate([np.stack([z, -q[:, 2], q[:, 1], -one, z, z], 1), np.stack([q[:, 2], z, -q[:, 0], z, -one, z], 1),
                        np.stack([-q[:, 1], q[:, 0], z, z, z, -one], 1)])
    r = np.concatenate([p[:, 0] - q[:, 0], p[:, 1] - q[:, 1], p[:, 2] - q[:, 2]])
    xi = -np.linalg.lstsq(J, r, rcond=None)[0]
    assert np.abs(trace[0]["xi"] - xi).max() < 1e-12 * max(1.0, np.abs(xi).max())


def test_mu_schedule_relative_scale():
    # mu_start = 1, divided at iterations 0, 4 and 8 (0.714..., 0.510..., 0.364...: 0.510 is still above 0.5), then
    # never again
    got = fr.mu_schedule(1.0, 16, 0.5)
    a = 1.0 / 1.4
    b = a / 1.4
    c = b / 1.4
    assert got == [a] * 4 + [b] * 4 + [c] * 8
    assert fr.mu_schedule(1.0, 6, 0.5, decrease_mu=0) == [1.0] * 6
    # another factor: 1 / 2 = 0.5 is not above 0.5, so the division stops after one step
    assert fr.mu_schedule(1.0, 9, 0.5, division_factor=2.0) == [0.5] * 9


def test_mu_schedule_absolute_scale():
    # a cloud whose farthest point from its mean is exactly 2: mu_start = sigma = 2 and scale_global = 1
    x = np.array([[2, 0, 0], [-2, 0, 0], [0, 1, 0], [0, -1, 0]], dtype=np.float32)
    y = x.copy()
    corr = np.stack([np.arange(4), np.arange(4)], 1)
    _, _, rel = fr.normalise(x, y, corr, use_absolute_scale=0)
    _, _, ab = fr.normalise(x, y, corr, use_absolute_scale=1)
    assert rel["sigma"] == 2.0 and rel["scale_global"] == 2.0 and rel["mu0"] == 1.0
    assert ab["scale_global"] == 1.0 and ab["mu0"] == 2.0
    got = fr.mu_schedule(ab["mu0"], 16, 0.9)
    assert got == [2.0 / 1.4] * 4 + [2.0 / 1.4 / 1.4] * 4 + [2.0 / 1.4 / 1.4 / 1.4] * 8
    got = fr.mu_schedule(rel["mu0"], 16, 0.9)
    assert got == [1.0 / 1.4] * 16  # 0.714... is below 0.9 after the first division


def test_back_transform_of_a_translated_and_scaled_cloud():
    # a cloud 300 units from the origin and 40 units across: the normalised frame's exact answer maps back onto the
    # ground truth, and the whole run recovers it
    x, y, corr, R, t = scene(500, 0.0, seed=5, scale=20.0, offset=(300.0, -120.0, 75.0))
    p, q, info = fr.normalise(x, y, corr)
    # truth in the normalised frame, where T maps q onto p: with y = R x + t, p = (x - mu_s) / s = R^T q +
    # (R^T (mu_t - t) - mu_s) / s
    Rn = R.T
    tn = (Rn @ (info["mean_t"] - t) - info["mean_s"]) / info["scale_global"]
    assert np.abs(q @ Rn.T + tn - p).max() < 1e-6  # the float32 clouds satisfy it to their rounding
    Ro, to = fr.to_input_frame(Rn, tn, info)
    assert np.abs(Ro - R).max() < 1e-12 and np.abs(to - t).max() < 1e-9 * 300
    res = fr.fgr(x, y, corr, maximum_correspondence_distance=1e-9, iteration_number=96)
    assert np.abs(res["R"] - R).max() < 1e-6 and np.abs(res["t"] - t).max() < 1e-4


def test_block_sum_is_a_sum():
    rng = np.random.default_rng(0)
    for n in (1, 255, 256, 257, 5000):
        a = rng.normal(size=(n, 3))
        assert np.allclose(fr.block_sum(a), a.sum(0), rtol=1e-13, atol=1e-12)


def test_fallback_below_ten_rows_and_at_zero_iterations():
    x, y, corr, _, _ = scene(50, 0.0, seed=1)
    for kw, c in ((dict(), corr[:9]), (dict(iteration_number=0), corr)):
        res = fr.fgr(x, y, c, **kw)
        assert res["iterations"] == 0 and res["converged"] == 0
        assert np.array_equal(res["R"], np.eye(3)) and np.array_equal(res["t"], np.zeros(3))
    # a non-finite end drops its row: ten rows with one NaN end are nine usable ones
    x2 = x.copy()
    x2[corr[3, 0]] = np.nan
    assert fr.fgr(x2, y, corr[:10])["converged"] == 0
    assert fr.fgr(x2, y, corr[:11])["converged"] == 1
