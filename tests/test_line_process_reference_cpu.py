"""The line-process restatement (tests/line_process_reference.py) held to first principles: its Jacobians against
central differences of zeta under the Euler update at inconsistent states, J_d = -J_s exactly, the confidence formula as
the minimiser of its term, the Euler round trip with its sy < 1e-6 branch, the zero node sums of b, a noiseless loop
recovered, a wrong closure pruned, and the reference compensation."""
import numpy as np
import pytest
from scipy.optimize import minimize_scalar

import line_process_reference as lp
import pose_graph_reference as pg
from line_process_graphs import graph, rigid

C_DIST = 0.05


@pytest.mark.parametrize("seed", range(5))
def test_jacobians_against_central_differences(seed):
    rng = np.random.default_rng(seed)
    Ts, Td, X = rigid(rng, 1.0, 1.0), rigid(rng, 1.0, 1.0), rigid(rng, 1.0, 1.0)  # far from consistency
    Js, Jd = lp.jacobians(Ts, Td, X)
    h = 1e-6
    for i in range(6):
        d = np.zeros(6)
        d[i] = h
        ns = (lp.zeta(lp.V(d) @ Ts, Td, X) - lp.zeta(lp.V(-d) @ Ts, Td, X)) / (2 * h)
        nd = (lp.zeta(Ts, lp.V(d) @ Td, X) - lp.zeta(Ts, lp.V(-d) @ Td, X)) / (2 * h)
        np.testing.assert_allclose(Js[:, i], ns, rtol=0, atol=1e-7)
        np.testing.assert_allclose(Jd[:, i], nd, rtol=0, atol=1e-7)


def test_jd_is_minus_js_exactly():
    rng = np.random.default_rng(7)
    for _ in range(20):
        Ts, Td, X = rigid(rng, 2.0, 3.0), rigid(rng, 2.0, 3.0), rigid(rng, 2.0, 3.0)
        Js, Jd = lp.jacobians(Ts, Td, X)
        assert np.array_equal(Jd, -Js)


@pytest.mark.parametrize("mu,c", [(0.5, 0.01), (0.5, 3.0), (2.0, 0.7), (1e-3, 5.0)])
def test_confidence_minimises_its_term(mu, c):
    f = lambda l: l * c + mu * (np.sqrt(l) - 1.0) ** 2
    best = minimize_scalar(f, bounds=(0.0, 1.0), method="bounded", options=dict(xatol=1e-12)).x
    assert abs(lp.confidence(mu, c) - best) < 1e-6
    assert f(lp.confidence(mu, c)) <= f(best) + 1e-12


def test_euler_round_trip_and_gimbal_branch():
    rng = np.random.default_rng(3)
    for _ in range(50):
        d = np.concatenate([rng.uniform(-3, 3, 1), rng.uniform(-1.5, 1.5, 1), rng.uniform(-3, 3, 1), rng.normal(size=3)])
        np.testing.assert_allclose(lp.euler(lp.V(d)), d, rtol=0, atol=1e-12)
    for b in (np.pi / 2, -np.pi / 2):  # sy = 0: z folded into x
        T = lp.V(np.array([0.4, b, 0.0, 1.0, 2.0, 3.0]))
        sy = np.hypot(T[0, 0], T[1, 0])
        assert sy < 1e-6
        e = lp.euler(T)
        assert e[2] == 0.0
        np.testing.assert_allclose(lp.V(e), T, rtol=0, atol=1e-12)


def test_b_node_sums_are_zero():
    gt, edges, T, L, unc = graph(5, 8, [(7, 0), (5, 1)], noise=0.05)
    rng = np.random.default_rng(1)
    P = [rigid(rng) for _ in range(8)]
    terms = lp._terms(P, edges, T, L)
    l = rng.uniform(0.1, 1.0, len(edges))
    H, b = lp.linear_system(8, edges, [True] * len(edges), l, terms)
    np.testing.assert_allclose(b.reshape(8, 6).sum(axis=0), 0.0, atol=1e-9 * np.abs(b).max())
    assert b.max() >= 0
    np.testing.assert_array_equal(H, H.T)


def test_noiseless_loop_recovered():
    gt, edges, T, L, unc = graph(11, 8, [(7, 0), (6, 2)], noise=0.0)
    rng = np.random.default_rng(2)
    init = [rigid(rng, 0.05, 0.05) @ g for g in gt]
    init[0] = np.eye(4)
    r = lp.optimize(8, edges, T, L, C_DIST, unc, init=init)
    assert r["kept"].all() and r["pruned"] == 0
    for p, g in zip(r["poses"], gt):
        np.testing.assert_allclose(p, g, rtol=0, atol=1e-6)


def test_consistent_graph_stops_at_once():
    gt, edges, T, L, unc = graph(12, 6, [(5, 0)], noise=0.0)
    r = lp.optimize(6, edges, T, L, C_DIST, unc)
    assert r["iterations"] == [0, 0] and r["trials"] == [0, 0]
    assert r["stop_reason"] == [lp.STOP["right_term"]] * 2


def test_wrong_closure_pruned_right_ones_kept():
    gt, edges, T, L, unc = graph(21, 16, [(15, 0), (8, 0), (12, 4)], wrong=[(10, 2), (14, 6)], noise=0.004)
    r = lp.optimize(16, edges, T, L, C_DIST, unc)
    assert not r["kept"][-2:].any() and r["kept"][:-2].all() and r["pruned"] == 2
    assert (r["confidence"][-2:] <= 0.25).all()
    odo = pg.bfs(16, edges, T, [d == s + 1 for s, d in edges], [0] * len(edges), 0)
    err_odo = max(np.linalg.norm(p[:3, 3] - g[:3, 3]) for p, g in zip(odo, gt))
    err = max(np.linalg.norm(p[:3, 3] - g[:3, 3]) for p, g in zip(r["poses"], gt))
    assert err < err_odo


def test_compensation():
    gt, edges, T, L, unc = graph(31, 10, [(9, 0), (6, 1)], noise=0.01)
    rng = np.random.default_rng(4)
    init = [rigid(rng, 0.02, 0.02) @ g for g in gt]
    r = lp.optimize(10, edges, T, L, C_DIST, unc, init=init, reference_node=3)
    np.testing.assert_allclose(r["poses"][3], init[3], rtol=0, atol=1e-12)
    free = lp.optimize(10, edges, T, L, C_DIST, unc, init=init, reference_node=-1)
    assert (free["trials"], free["iterations"]) == (r["trials"], r["iterations"])
    Cm = init[3] @ pg.inv(free["poses"][3])
    np.testing.assert_allclose(r["poses"], np.stack([Cm @ p for p in free["poses"]]), rtol=0, atol=1e-12)
    assert not np.allclose(free["poses"][3], init[3], atol=1e-9)


def test_block_sum_order():
    x = np.arange(1, 3000, dtype=np.float64)
    assert lp.block_sum(x, 256) == float(x.sum())
    assert lp.block_sum([], 1024) == 0.0
