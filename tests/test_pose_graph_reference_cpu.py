"""The numpy restatement of the multiway step (tests/pose_graph_reference.py) against its definition: Lambda against a
direct per-correspondence sum, the Jacobians against central finite differences, the log's branches, exact recovery on a
noiseless loop, a corrupted loop closure rejected by GNC-TLS, and the gauge (moving the reference node's initial pose
moves every pose rigidly).  CPU only."""
import numpy as np
from scipy.spatial.transform import Rotation

import pose_graph_reference as ref


def rigid(rng, angle=0.3, shift=0.5):
    T = np.eye(4)
    T[:3, :3] = Rotation.from_rotvec(rng.normal(size=3) * angle).as_matrix()
    T[:3, 3] = rng.normal(size=3) * shift
    return T


def test_information_matches_direct_sum():
    rng = np.random.default_rng(1)
    y = rng.uniform(-1, 1, size=(700, 3)).astype(np.float32)
    x = (y[:600] + rng.normal(scale=0.01, size=(600, 3))).astype(np.float32)
    L, n = ref.information(x, y, 1.0, np.eye(3), np.zeros(3), 0.05)
    Ld, nd = ref.information_direct(x, y, 1.0, np.eye(3), np.zeros(3), 0.05)
    assert n == nd > 300 and L[5, 5] == n
    np.testing.assert_allclose(L, Ld, rtol=1e-12, atol=1e-9)
    assert np.array_equal(L, L.T)
    # G^T G of one point: rank 3, and [-[q]x | I]^T [-[q]x | I] entry by entry
    q = np.array([[0.3, -0.2, 0.7]])
    G = np.hstack([-ref.skew(q[0]), np.eye(3)])
    want = (G.T @ G)[np.triu_indices(6)]
    np.testing.assert_array_equal(ref.g_terms(q)[0], want)


def test_chunk_sum_is_exact_for_integers():
    v = np.arange(3 * 1000, dtype=np.float64).reshape(1000, 3)
    np.testing.assert_array_equal(ref.chunk_sum(v), v.sum(axis=0))


def _fd_jacobian(f, T, h=1e-6):
    cols = []
    for k in range(6):
        d = np.zeros(6)
        d[k] = h
        cols.append((f(ref.se3_exp(d) @ T) - f(ref.se3_exp(-d) @ T)) / (2 * h))
    return np.stack(cols, axis=1)


def test_jacobians_against_finite_differences():
    rng = np.random.default_rng(2)
    for _ in range(5):
        Ts, Td = rigid(rng), rigid(rng)
        Tsd = ref.inv(Td) @ Ts  # consistent edge: E = I
        Js, Jd = ref.jacobians(Td)
        np.testing.assert_allclose(_fd_jacobian(lambda T: ref.residual(T, Td, Tsd), Ts), Js, atol=1e-8)
        np.testing.assert_allclose(_fd_jacobian(lambda T: ref.residual(Ts, T, Tsd), Td), Jd, atol=1e-8)
        # off consistency the first-order Jacobians are off by O(|e|)
        Tsd2 = rigid(rng, 0.01, 0.01) @ Tsd
        e = np.abs(ref.residual(Ts, Td, Tsd2)).max()
        np.testing.assert_allclose(_fd_jacobian(lambda T: ref.residual(T, Td, Tsd2), Ts), Js, atol=20 * e)


def test_log_branches():
    rng = np.random.default_rng(3)
    for th in (0.0, 1e-9, 3e-6, 1e-3, 0.5, 2.0, 2.7, 3.0, np.pi - 1e-7):
        a = rng.normal(size=3)
        a /= np.linalg.norm(a)
        R = Rotation.from_rotvec(th * a).as_matrix()
        w = ref.so3_log(R)
        np.testing.assert_allclose(w, th * a, atol=1e-12 + 1e-9 * th)
    # small-angle branch: (1 + theta^2 / 6) v is exact to O(theta^4)
    w = np.array([4e-6, -3e-6, 1e-6])
    R = Rotation.from_rotvec(w).as_matrix()
    np.testing.assert_allclose(ref.so3_log(R), w, rtol=1e-9, atol=1e-20)
    # exp and log round-trip
    x = np.array([0.2, -0.1, 0.3, 1.0, 2.0, -0.5])
    T = ref.se3_exp(x)
    np.testing.assert_allclose(ref.so3_log(T[:3, :3]), x[:3], atol=1e-14)
    np.testing.assert_allclose(T[:3, :3], Rotation.from_rotvec(x[:3]).as_matrix(), atol=1e-14)


def loop_graph(rng, K=8, noise=0.0, closures=(), wrong=()):
    """Ground-truth poses, odometry edges (k, k+1), loop closures (s, d) and wrong closures; Lambda from a synthetic
    overlap (200 target points per edge)."""
    gt = [np.eye(4)] + [rigid(rng) for _ in range(K - 1)]
    edges, T, L, unc = [], [], [], []
    pts = rng.uniform(-1, 1, size=(200, 3))
    Lam = sum(np.hstack([-ref.skew(q), np.eye(3)]).T @ np.hstack([-ref.skew(q), np.eye(3)]) for q in pts)
    for (s, d, u) in [(k, k + 1, 0) for k in range(K - 1)] + [(s, d, 1) for s, d in closures] + \
            [(s, d, 2) for s, d in wrong]:
        Tsd = ref.inv(gt[d]) @ gt[s]
        if u == 2:
            Tsd = rigid(rng, 0.5, 1.0) @ Tsd
        elif noise:
            Tsd = rigid(rng, noise, noise) @ Tsd
        edges.append((s, d))
        T.append(Tsd)
        L.append(Lam)
        unc.append(1 if u else 0)
    return gt, np.array(edges), T, L, unc


def test_noiseless_loop_recovered_exactly():
    rng = np.random.default_rng(4)
    gt, edges, T, L, unc = loop_graph(rng, closures=[(7, 0), (5, 1)])
    out = ref.optimize(8, edges, T, L, 0.05, unc)
    np.testing.assert_allclose(out["poses"], np.stack(gt), atol=1e-10)
    assert out["mask"].all() and out["cost"] < 1e-20


def test_corrupted_closure_rejected():
    rng = np.random.default_rng(5)
    gt, edges, T, L, unc = loop_graph(rng, K=10, noise=0.002, closures=[(9, 0), (6, 2)], wrong=[(8, 3)])
    out = ref.optimize(10, edges, T, L, 0.05, unc)
    w = out["weights"]
    assert w[-1] == 0.0 and not out["mask"][-1]
    assert w[9] == 1.0 and w[10] == 1.0 and out["mask"][:11].all()
    assert out["iterations"] > 1
    err = max(np.abs(p - g).max() for p, g in zip(out["poses"], gt))
    assert err < 0.05
    # every edge certain: no GNC step, one inner solve
    allc = ref.optimize(10, edges[:9], T[:9], L[:9], 0.05, None)
    assert allc["iterations"] == 1 and (allc["weights"] == 1).all()


def test_gauge_moves_rigidly():
    rng = np.random.default_rng(6)
    gt, edges, T, L, unc = loop_graph(rng, noise=0.003, closures=[(7, 0), (4, 1)])
    base = ref.optimize(8, edges, T, L, 0.05, unc)
    init = ref.bfs(8, edges, T, [True] * len(edges), unc, 0)
    G = rigid(rng, 0.7, 2.0)
    moved = ref.optimize(8, edges, T, L, 0.05, unc, init=[G @ p for p in init])
    np.testing.assert_allclose(moved["poses"], np.stack([G @ p for p in base["poses"]]), atol=1e-8)
    assert np.array_equal(moved["mask"], base["mask"])


def test_disconnected_graph():
    rng = np.random.default_rng(7)
    _, edges, T, L, unc = loop_graph(rng, K=4)
    assert ref.optimize(5, edges, T, L, 0.05, unc) is None
    L0 = [x.copy() for x in L]
    L0[1][:] = 0  # no information: connects nothing
    assert ref.optimize(4, edges, T, L0, 0.05, unc) is None


def test_singular_node_block_does_not_stop_the_graph():
    """A node whose block of H is singular (here its one edge constrains only one direction) must not stop the others:
    the additive part of the damping keeps the system positive definite, the rest converges as without that node."""
    rng = np.random.default_rng(8)
    gt, edges, T, L, unc = loop_graph(rng, K=7, noise=0.002, closures=[(6, 0)])
    base = ref.optimize(7, edges, T, L, 0.05, unc)
    Lsing = np.zeros((6, 6))
    Lsing[5, 5] = 100.0
    out = ref.optimize(8, np.vstack([edges, [[7, 3]]]), T + [ref.inv(gt[3]) @ rigid(rng)], L + [Lsing], 0.05,
                       unc + [1])
    np.testing.assert_allclose(out["poses"][:7], base["poses"], atol=1e-9)
    assert out["mask"].all()
