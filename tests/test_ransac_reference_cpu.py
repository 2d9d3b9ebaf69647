"""The premises of tests/ransac_reference.py (the restatement of tzr_ransac_batch, DESIGN.md §3.21), without a device:
hand-listed draws, each checker at equality on both sides of its bound, the exit bound's edge cases, exact recovery at
90 % outliers, and agreement with a literal transcription of the loop."""
import math

import numpy as np
import pytest

import ransac_reference as rr


def test_draws_hand_listed():
    # splitmix64(0) and splitmix64(1): the published SplitMix64 outputs of seeds -0x9E37... and 1 - 0x9E37...
    assert rr.splitmix64(0) == 0xE220A8397B1DCDAF
    assert rr.splitmix64(1) == 0x910A2DEC89025CC1
    # draw j of hypothesis itr: mulhi64(splitmix64(seed + n itr + j), K)
    assert rr.draws(0, 3, 0, 10) == [(rr.splitmix64(j) * 10) >> 64 for j in range(3)]
    assert rr.draws(5, 4, 2, 7) == [(rr.splitmix64(5 + 8 + j) * 7) >> 64 for j in range(4)]
    # the seed wraps modulo 2^64
    assert rr.draws(2 ** 64 - 1, 3, 0, 100)[1] == (rr.splitmix64(0) * 100) >> 64
    assert all(0 <= d < 13 for itr in range(50) for d in rr.draws(77, 8, itr, 13))


def test_edge_checker_is_strict():
    P = np.array([[0.0, 0, 0], [2.0, 0, 0]])
    Q = np.array([[0.0, 0, 0], [1.0, 0, 0]])
    assert rr.edge_ok(P, Q, 0.5)  # d_y = d_x s exactly: passes
    assert not rr.edge_ok(P, Q, np.nextafter(0.5, 1.0))
    assert rr.edge_ok(Q, P, 0.5) and not rr.edge_ok(Q, P, np.nextafter(0.5, 1.0))
    assert rr.edge_ok(P, P, 1.0) and not rr.edge_ok(P, P, np.nextafter(1.0, 2.0))


def test_distance_checker_is_strict():
    R, t = np.eye(3), np.zeros(3)
    P = np.array([[0.0, 0, 0]])
    Q = np.array([[0.0, 0.75, 0]])
    assert rr.distance_ok(R, t, P, Q, 0.75)  # ||T x - y|| = thr: passes
    assert not rr.distance_ok(R, t, P, Q, np.nextafter(0.75, 0.0))


def test_normal_checker_is_strict():
    R = np.eye(3)
    a = np.array([[1.0, 0, 0]])
    b = np.array([[0.5, 0.0, 0.0]])
    assert rr.normal_ok(R, a, b, 0.5)  # the dot product = cos: passes
    assert not rr.normal_ok(R, a, b, np.nextafter(0.5, 1.0))
    assert rr.normal_ok(R, a, np.array([[np.nan, 0, 0]]), 0.9)  # a NaN never fails


def test_score_counts_strictly_inside_and_sums_by_segment():
    X = np.zeros((1100, 3))
    Y = np.zeros((1100, 3))
    Y[:, 0] = np.linspace(0, 2, 1100)
    cnt, total, f, rm = rr.score(np.eye(3), np.zeros(3), X, Y, 1.0)
    d2 = Y[:, 0] ** 2
    assert cnt == int((d2 < 1.0).sum()) and f == cnt / 1100
    want = 0.0
    for s0 in range(0, 1100, rr.SEG):
        seg = 0.0
        for v in d2[s0:s0 + rr.SEG]:
            if v < 1.0:
                seg = seg + v
        want = want + seg
    assert total == want and rm == math.sqrt(want / cnt)
    Y[:, 0] = 1.0  # d^2 = r^2 exactly: no inlier, fitness and rmse 0
    assert rr.score(np.eye(3), np.zeros(3), X, Y, 1.0) == (0, 0.0, 0.0, 0.0)


def test_exit_bound_edges():
    assert rr.bound(1.0, 3, 0.999)[0] == 0  # fitness 1: stop after this hypothesis
    assert rr.bound(0.5, 3, 0.0)[0] == 0  # confidence 0: stop
    assert rr.bound(0.5, 3, 1.0)[0] == math.inf  # confidence 1: never lowered
    assert rr.bound(1.0, 3, 1.0)[0] == math.inf  # NaN: not lowered
    assert rr.bound(1e-6, 3, 0.999)[0] == math.inf  # 1 - f^3 rounds to 1: -inf, not lowered
    b, q = rr.bound(0.5, 3, 0.999)
    assert b == math.ceil(math.log(0.001) / math.log(0.875)) and q < b


def problem(K, outlier_rate, seed, noise=0.0):
    rng = np.random.default_rng(seed)
    x = rng.uniform(-1, 1, (K, 3)).astype(np.float32)
    a = 0.7
    R = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
    t = np.array([0.2, -0.4, 0.9])
    y = (x.astype(np.float64) @ R.T + t + rng.normal(scale=noise, size=(K, 3))).astype(np.float32)
    j = np.arange(K)
    bad = rng.random(K) < outlier_rate
    j[bad] = rng.integers(0, K, int(bad.sum()))
    return x, y, np.stack([np.arange(K), j], axis=1), R, t


def test_exact_recovery_at_90_percent_outliers():
    x, y, c, R, t = problem(2000, 0.9, seed=3)
    out = rr.ransac(x, y, c, 1e-4, seed=1, edge=0.9)
    assert out["winner"] >= 0 and out["passed"] < out["drawn"]
    assert np.abs(out["R"] - R).max() < 1e-5 and np.abs(out["t"] - t).max() < 1e-5
    assert out["converged"] == 1


@pytest.mark.parametrize("K,out,n,mi,conf", [(20, 0.3, 3, 60, 0.999), (700, 0.5, 4, 40, 1.0), (50, 0.2, 3, 200, 0.0),
                                             (9, 0.6, 8, 30, 0.9)])
def test_agrees_with_the_literal_loop(K, out, n, mi, conf):
    x, y, c, _, _ = problem(K, out, seed=K, noise=1e-3)
    a = rr.ransac(x, y, c, 0.01, seed=5, ransac_n=n, max_iteration=mi, confidence=conf)
    b = rr.literal_ransac(x, y, c, 0.01, seed=5, ransac_n=n, max_iteration=mi, confidence=conf)
    assert (a["drawn"], a["winner"], a["inliers"], a["rmse"]) == (b["drawn"], b["winner"], b["inliers"], b["rmse"])
    if b["winner"] >= 0:
        assert a["R"].tobytes() == b["R"].tobytes() and a["t"].tobytes() == b["t"].tobytes()


def test_fallbacks():
    x, y, c, _, _ = problem(10, 0.0, seed=1)
    for cc, mi in ((c[:2], 100), (c, 0)):
        out = rr.ransac(x, y, cc, 0.01, max_iteration=mi)
        assert out["drawn"] == 0 and out["winner"] == -1 and np.array_equal(out["R"], np.eye(3))
    x[0] = np.nan
    assert rr.ransac(x, y, c, 0.01)["usable"] == 9
