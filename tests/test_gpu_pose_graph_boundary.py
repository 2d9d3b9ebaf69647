"""The pose graph where it can be wrong (run on an H100: `pytest -m gpu`), against the numpy restatement
(tests/pose_graph_reference.py) and against definitions:
- the device log at its branch switches, near and at pi and at tied diagonals, read back through self-loops on the
  reference node;
- GNC-TLS with exactly representable residuals: mu at max r-bar = 1/2, the full threshold schedule bit for bit, the
  strict cost stop;
- the damping's failure paths: an indefinite Lambda (potrf fails), a cost that overflows (13 rejections), a far start;
- sizes and layouts: edge sums past one warp and one CTA, a hub with parallel edges, other reference nodes, K = 1024;
- the breadth-first start bit for bit, and the graphs it must refuse;
- information matrices past 32 chunks on both search routes.

Self-loops on the reference node make device arithmetic observable.  That node's pose is the identity and never moves,
so for an edge (ref, ref, R_sd, t_sd) the device forms R_E = R_sd^T exactly and t_E = -(R_sd^T t_sd) in the order
probe_tau() states.  The edge connects nothing and enters neither H nor g, but its r-bar is written to `residuals`.  With
Lambda = a a^T, a = e_k + e_5, and c = 1, r-bar = (omega_k + tau_2)^2 as log_rbar() rounds it, so omega_k comes back with
its sign when tau_2 > |omega_k|."""
import importlib
import time

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import pose_graph_reference as ref
from test_gpu_icp import scan_pair

capi = importlib.import_module("teaser-plusplus_b200.capi")

pytestmark = pytest.mark.gpu

BRUTE, GRID = capi.FLAG_ICP_BRUTE_FORCE, capi.FLAG_ICP_GRID
R_CORR = 0.05


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.set_flags(0)
    c.close()


def with_flags(ctx, flags, fn):
    ctx.set_flags(flags)
    try:
        return fn()
    finally:
        ctx.set_flags(0)


def rigid(rng, angle=0.3, shift=0.5):
    T = np.eye(4)
    T[:3, :3] = Rotation.from_rotvec(rng.normal(size=3) * angle).as_matrix()
    T[:3, 3] = rng.normal(size=3) * shift
    return T


def overlap_info(rng, m=200):
    """Lambda of m target points in [-1, 1]^3 (sum of G^T G, G = [-[q]x | I])."""
    pts = rng.uniform(-1, 1, size=(m, 3))
    return sum(np.hstack([-ref.skew(q), np.eye(3)]).T @ np.hstack([-ref.skew(q), np.eye(3)]) for q in pts)


def same_bytes(a, b):
    for k in ("poses", "weights", "mask", "residuals", "iterations", "inner_iterations", "cost"):
        assert np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes(), k


# ---- self-loop probes --------------------------------------------------------------------------------------------------
def probe_tau(R, t):
    """t_E of a self-loop (ref, ref, R, t) as pg_edge_kernel forms it at T_s = T_d = I: -(R^T t), entry r summed as
    (R[0,r] t[0] + R[1,r] t[1]) + R[2,r] t[2] in float64 without FMA."""
    R, t = np.asarray(R, dtype=np.float64), [float(x) for x in t]
    return np.array([-((float(R[0, r]) * t[0] + float(R[1, r]) * t[1]) + float(R[2, r]) * t[2]) for r in range(3)])


def log_probe(R, theta):
    """Three certain self-loops on node 0 that read back omega = log(R^T) through r-bar (c = 1): T_sd = (R, t) with t
    chosen so that tau_2 is about 2 theta (1 at theta = 0), which is above |omega_k| and keeps the read-back's absolute
    rounding near ulp(theta).  Returns (transforms, informations, tau_2)."""
    T = np.eye(4)
    T[:3, :3] = R
    T[:3, 3] = -np.asarray(R) @ np.array([0.0, 0.0, 2.0 * theta if theta > 0 else 1.0])
    tau2 = probe_tau(R, T[:3, 3])[2]
    Ls = []
    for k in range(3):
        a = np.zeros(6)
        a[k] = a[5] = 1.0
        Ls.append(np.outer(a, a))
    return [T] * 3, Ls, tau2


def log_rbar(omega_k, tau2):
    """r-bar of a log probe as the device rounds it: Lambda e sums to s = omega_k + tau_2 in both live rows, then
    e^T (Lambda e) = omega_k s + tau_2 s; the normalisation is 1."""
    s = omega_k + tau2
    return omega_k * s + tau2 * s


def log_readback(rbar, tau2):
    return np.sqrt(rbar) - tau2


def probe_graph(loops_T, loops_L, loops_unc=None):
    """K = 2: the certain edge (0, 1) at T = I, Lambda = I, then the self-loops on node 0."""
    n = len(loops_T)
    edges = np.array([[0, 1]] + [[0, 0]] * n, dtype=np.int32)
    T = [np.eye(4)] + list(loops_T)
    L = [np.eye(6)] + list(loops_L)
    unc = [0] + (list(loops_unc) if loops_unc is not None else [0] * n)
    return edges, T, L, unc


def _axes():
    return {"x": np.array([1.0, 0, 0]), "y": np.array([0, 1.0, 0]), "z": np.array([0, 0, 1.0]),
            "xy": np.array([1.0, 1.0, 0]) / np.sqrt(2), "xyz": np.ones(3) / np.sqrt(3),
            "mixed": np.array([0.48, -0.6, 0.64])}


THETAS = [0.0, 1e-7, 1e-5 * (1 - 2.0 ** -20), 1e-5 * (1 + 2.0 ** -20), 0.5, 2.0, np.arccos(-0.9) - 1e-9,
          np.arccos(-0.9) + 1e-9, 3.0, np.pi - 1e-6, np.pi - 1e-9, np.pi]


def test_device_log_against_its_definition(ctx):
    """log(R_sd^T) = -theta a for every angle and axis (+-pi a at pi), to 1e-12 absolute, and the device's r-bar equal to
    the restatement's log pushed through the same rounding to within 8 ulps of r-bar.  All 72 rotations (216 edges, so
    the cost sums wrap the warp and the edge kernel runs 2 CTAs) go in one call."""
    cases, Ts, Ls, taus = [], [], [], []
    for name, a in _axes().items():
        for th in THETAS:
            R = Rotation.from_rotvec(th * a).as_matrix()
            T3, L3, tau2 = log_probe(R, th)
            cases.append((name, th, a, R))
            Ts += T3
            Ls += L3
            taus.append(tau2)
    edges, T, L, unc = probe_graph(Ts, Ls)
    got = ctx.optimize_pose_graph(2, edges, T, L, 1.0, uncertain=unc)
    rb = got["residuals"][1:].reshape(-1, 3)
    for (name, th, a, R), r3, tau2 in zip(cases, rb, taus):
        w = log_readback(r3, tau2)
        want = -th * a
        if th == np.pi:
            err = min(np.abs(w - want).max(), np.abs(w + want).max())
        else:
            err = np.abs(w - want).max()
        assert err <= 1e-12, (name, th, w, want)
        wr = ref.so3_log(R.T.copy())
        model = np.array([log_rbar(wr[k], tau2) for k in range(3)])
        assert np.all(np.abs(r3 - model) <= 8 * np.spacing(model)), (name, th, r3, model)


# exact rotations by pi: 2 a a^T - I.  Its symmetric part's diagonal is tied, v = 0, so no sign fix applies and the
# strict `>` must keep the first tied column; with a_0 a_1 < 0 (or a_0 a_2 < 0) another column gives -pi a.
PI_EXACT = {
    "xy": (np.array([[0.0, 1, 0], [1, 0, 0], [0, 0, -1]]), np.array([1.0, 1.0, 0]) / np.sqrt(2)),
    "x-y": (np.array([[0.0, -1, 0], [-1, 0, 0], [0, 0, -1]]), np.array([1.0, -1.0, 0]) / np.sqrt(2)),
    "xyz": (2.0 / 3.0 * np.ones((3, 3)) - np.eye(3), np.ones(3) / np.sqrt(3)),
    "xy-z": (2.0 / 3.0 * np.outer([1, 1, -1], [1, 1, -1]) - np.eye(3), np.array([1.0, 1, -1]) / np.sqrt(3)),
}


def test_device_log_tied_diagonals_at_pi(ctx):
    Ts, Ls, taus = [], [], []
    for name, (R, a) in PI_EXACT.items():
        T3, L3, tau2 = log_probe(R, np.pi)
        Ts += T3
        Ls += L3
        taus.append(tau2)
    edges, T, L, unc = probe_graph(Ts, Ls)
    got = ctx.optimize_pose_graph(2, edges, T, L, 1.0, uncertain=unc)
    for (name, (R, a)), r3, tau2 in zip(PI_EXACT.items(), got["residuals"][1:].reshape(-1, 3), taus):
        wr = ref.so3_log(R.T.copy())
        np.testing.assert_allclose(wr, np.pi * a, rtol=0, atol=1e-12)  # the first column's sign: +a
        w = log_readback(r3, tau2)
        np.testing.assert_allclose(w, np.pi * a, rtol=0, atol=1e-12, err_msg=name)
        model = np.array([log_rbar(wr[k], tau2) for k in range(3)])
        assert np.all(np.abs(r3 - model) <= 8 * np.spacing(model)), (name, r3, model)


# ---- GNC-TLS with exact values -----------------------------------------------------------------------------------------
def gnc_graph(rbars, certain_rbars=()):
    """Self-loops on node 0 with T = (I, (1, 0, 0)) and Lambda = diag(0, 0, 0, r, 0, 1): at c = 1 their r-bar is r
    exactly and stays so for the whole call.  Uncertain loops first, then certain ones."""
    Ts, Ls, unc = [], [], []
    for r, u in [(r, 1) for r in rbars] + [(r, 0) for r in certain_rbars]:
        T = np.eye(4)
        T[0, 3] = 1.0
        Lm = np.zeros((6, 6))
        Lm[3, 3], Lm[5, 5] = r, 1.0
        Ts.append(T)
        Ls.append(Lm)
        unc.append(u)
    return probe_graph(Ts, Ls, unc)


def both(ctx, edges, T, L, unc, trace=None, **kw):
    got = ctx.optimize_pose_graph(2, edges, T, L, 1.0, uncertain=unc, **kw)
    want = ref.optimize(2, edges, T, L, 1.0, unc, trace=trace, **kw)
    return got, want


HALF = 0.5


@pytest.mark.parametrize("rmax,iters", [(HALF, 1), (np.nextafter(HALF, 0), 1), (0.3, 1), (np.nextafter(HALF, 1), 2)])
def test_gnc_mu_at_half(ctx, rmax, iters):
    """max r-bar = 1/2 makes 1 / (2 max r-bar - 1) = +inf: the call must stop with weights 1, as for any max r-bar
    below 1/2 (mu < 0).  One ulp above, mu is finite and every weight is 1 at once."""
    edges, T, L, unc = gnc_graph([0.1, rmax, 0.25])
    got, want = both(ctx, edges, T, L, unc)
    assert np.array_equal(got["residuals"][1:], [0.1, rmax, 0.25])
    assert got["iterations"] == want["iterations"] == iters
    assert (got["weights"] == 1).all() and got["mask"].all()
    assert got["weights"].tobytes() == want["weights"].tobytes()


SCHEDULE = [2.5, 2.0, 1.0, 0.5, 0.25, 0.0]


@pytest.mark.parametrize("max_iterations", [1, 2, 3, 4])
def test_gnc_schedule_bit_for_bit(ctx, max_iterations):
    """gnc_factor 2 keeps every mu exact: mu = 1/4, 1/2, 1, 2.  With cost_threshold -1 only max_iterations stops."""
    edges, T, L, unc = gnc_graph(SCHEDULE)
    got, want = both(ctx, edges, T, L, unc, gnc_factor=2.0, cost_threshold=-1.0, max_iterations=max_iterations)
    assert got["iterations"] == want["iterations"] == max_iterations
    assert got["weights"].tobytes() == want["weights"].tobytes()
    assert np.array_equal(got["mask"], want["mask"])
    if max_iterations == 3:  # mu = 1 in the third update: r-bar = 2 sits exactly on th1, r-bar = 1/2 on th2
        assert got["weights"][2] == 0.0 and got["weights"][4] == 1.0


def test_gnc_cost_stop_is_strict(ctx):
    edges, T, L, unc = gnc_graph(SCHEDULE)
    tr = []
    ref.optimize(2, edges, T, L, 1.0, unc, trace=tr, gnc_factor=2.0, cost_threshold=-1.0, max_iterations=4)
    diff = [x["diff"] for x in tr if x["kind"] == "gnc"][1]  # |cost - previous cost| after the second update
    assert 0 < diff < np.inf
    got, want = both(ctx, edges, T, L, unc, gnc_factor=2.0, cost_threshold=diff, max_iterations=6)
    assert got["iterations"] == want["iterations"] > 2
    got, want = both(ctx, edges, T, L, unc, gnc_factor=2.0, cost_threshold=np.nextafter(diff, np.inf),
                     max_iterations=6)
    assert got["iterations"] == want["iterations"] == 2
    assert got["weights"].tobytes() == want["weights"].tobytes()


def test_gnc_ignores_certain_edges(ctx):
    """Certain edges keep weight 1 and do not enter max r-bar: a certain r-bar of 100 beside uncertain ones below 1/2
    stops at once; without uncertain edges one GNC iteration runs."""
    edges, T, L, unc = gnc_graph([0.25, 0.125], certain_rbars=[100.0, 3.0])
    got, want = both(ctx, edges, T, L, unc)
    assert got["iterations"] == want["iterations"] == 1 and (got["weights"] == 1).all()
    edges, T, L, unc = gnc_graph([2.5, 0.25], certain_rbars=[100.0, 3.0])
    got, want = both(ctx, edges, T, L, unc, gnc_factor=2.0)
    assert got["iterations"] == want["iterations"] > 1
    assert got["weights"].tobytes() == want["weights"].tobytes()
    assert (got["weights"][[0, 3, 4]] == 1).all() and got["weights"][1] == 0.0
    edges, T, L, unc = gnc_graph([], certain_rbars=[100.0, 3.0])
    got, want = both(ctx, edges, T, L, unc)
    assert got["iterations"] == want["iterations"] == 1 and (got["weights"] == 1).all()


# ---- the damping's failure paths ----------------------------------------------------------------------------------------
def check_margins(trace, rel=1e-6):
    """Every decision of the restatement's inner solves has a clear margin, so the device must make the same ones:
    a factorisation succeeds or fails with the smallest eigenvalue of the damped H at least 1e-8 |H| from 0; an
    accept / reject compares F' with F at least rel |F| apart; a stop test compares |F - F'| with its tolerance at least
    rel of the tolerance apart."""
    for x in trace:
        if x["kind"] != "inner":
            continue
        lo, big = x["eig"]
        assert abs(lo) >= 1e-8 * big, x
        assert x["factored"] == (lo > 0), x
        if not x["factored"] or not np.isfinite(x["Fc"]):
            continue
        d = abs(x["F"] - x["Fc"])
        assert abs(d - x["tol"]) >= rel * x["tol"], x
        if x["outcome"] != "stop":
            assert d >= rel * abs(x["F"]), x


def compare(got, want, atol=1e-8):
    assert (got["iterations"], got["inner_iterations"]) == (want["iterations"], want["inner_iterations"])
    assert np.array_equal(got["mask"], want["mask"])
    np.testing.assert_allclose(got["poses"], want["poses"], rtol=0, atol=atol)


def indefinite_graph():
    """K = 3: the chain 0 - 1 - 2 and the closure (2, 0), every edge certain.  The closure ends at the reference node,
    so its Lambda enters node 2's block of H as it is; it couples the translation's x and y by 500 against diagonals of
    about 100 (two overlaps of 50 points), so the first damped H is indefinite, potrf fails, and the damping climbs until H is positive definite."""
    rng = np.random.default_rng(5)
    gt = [np.eye(4), rigid(rng), rigid(rng)]
    edges, T, L = [], [], []
    for s, d in [(0, 1), (1, 2), (2, 0)]:
        edges.append((s, d))
        T.append(rigid(rng, 0.02, 0.05) @ ref.inv(gt[d]) @ gt[s])
        L.append(overlap_info(rng, 50))
    L[2][3, 4] = L[2][4, 3] = 500.0
    return np.array(edges, dtype=np.int32), T, L


def test_indefinite_information_takes_the_failure_path(ctx):
    edges, T, L = indefinite_graph()
    assert np.linalg.eigvalsh(L[2])[0] < -100 and L[2][5, 5] > 0  # accepted: finite, Lambda(5,5) >= 0
    tr = []
    want = ref.optimize(3, edges, T, L, R_CORR, None, trace=tr, max_inner_iterations=12)
    inner = [x for x in tr if x["kind"] == "inner"]
    assert not inner[0]["factored"] and sum(not x["factored"] for x in inner) >= 3
    assert any(x["outcome"] == "accept" for x in inner)
    check_margins(tr)
    got = ctx.optimize_pose_graph(3, edges, T, L, R_CORR, max_inner_iterations=12)
    compare(got, want)


def overflow_graph():
    """A chain of 4 certain edges, two uncertain closures (one wrong), and a certain self-loop on node 0 with Lambda =
    1e306 I and a translation residual of 10 per axis: its e^T Lambda e is +inf, so F is +inf at the start and at every
    candidate, whatever the step."""
    rng = np.random.default_rng(6)
    gt = [np.eye(4)] + [rigid(rng) for _ in range(4)]
    edges, T, L, unc = [], [], [], []
    for s, d, u in [(0, 1, 0), (1, 2, 0), (2, 3, 0), (3, 4, 0), (4, 0, 1), (3, 1, 1)]:
        edges.append((s, d))
        Tsd = ref.inv(gt[d]) @ gt[s]
        T.append((rigid(rng, 0.5, 1.0) if (s, d) == (3, 1) else rigid(rng, 0.002, 0.002)) @ Tsd)
        L.append(overlap_info(rng))
        unc.append(u)
    loop = np.eye(4)
    loop[:3, 3] = 10.0
    edges.append((0, 0))
    T.append(loop)
    L.append(1e306 * np.eye(6))
    unc.append(0)
    return np.array(edges, dtype=np.int32), T, L, unc


def test_overflowing_cost_stops_after_13_rejections(ctx):
    edges, T, L, unc = overflow_graph()
    with np.errstate(over="ignore", invalid="ignore"):
        want = ref.optimize(5, edges, T, L, R_CORR, unc, max_inner_iterations=20)
    got = ctx.optimize_pose_graph(5, edges, T, L, R_CORR, uncertain=unc, max_inner_iterations=20)
    assert got["residuals"][-1] == np.inf and got["cost"] == np.inf
    assert got["iterations"] == want["iterations"] > 1
    assert got["inner_iterations"] == want["inner_iterations"] == 13 * got["iterations"]
    live = [s != d for s, d in edges]
    start = ref.bfs(5, edges, T, live, unc, 0)
    assert np.array_equal(got["poses"], np.stack(start))
    assert got["weights"].tobytes() == want["weights"].tobytes()


def far_start_graph():
    """A noiseless ring of 5 with two chords, every edge certain, started 2.5 to 3 rad away from the optimum at every
    free node: the live residuals start in the log's near-pi branch and LM rejects steps on the way."""
    rng = np.random.default_rng(51)
    gt = [np.eye(4)] + [rigid(rng, 0.4, 1.0) for _ in range(4)]
    edges, T, L = [], [], []
    for s, d in [(0, 1), (1, 2), (2, 3), (3, 4), (4, 0), (3, 0), (1, 3)]:
        edges.append((s, d))
        T.append(ref.inv(gt[d]) @ gt[s])
        L.append(overlap_info(rng))
    init = [np.eye(4)]
    for k in range(1, 5):
        a = rng.normal(size=3)
        D = np.eye(4)
        D[:3, :3] = Rotation.from_rotvec(a / np.linalg.norm(a) * rng.uniform(2.5, 3.0)).as_matrix()
        init.append(D @ gt[k])
    return np.array(edges, dtype=np.int32), T, L, init


def test_far_start_against_the_restatement(ctx):
    edges, T, L, init = far_start_graph()
    tr = []
    want = ref.optimize(5, edges, T, L, R_CORR, None, init=init, trace=tr, max_inner_iterations=60)
    inner = [x for x in tr if x["kind"] == "inner"]
    assert any(x["outcome"] == "reject" for x in inner) and inner[-1]["outcome"] == "stop"
    check_margins(tr)
    got = ctx.optimize_pose_graph(5, edges, T, L, R_CORR, initial_poses=init, max_inner_iterations=60)
    compare(got, want)


# ---- size and layout ---------------------------------------------------------------------------------------------------
def make_graph(seed, K, pairs, wrong=(), noise=0.002, certain=None):
    """Ground truth, then one edge per pair (s, d) (noisy) and per wrong pair (off by up to 0.5 rad and 1); an edge is
    certain when d = s + 1 or certain(s, d) says so."""
    rng = np.random.default_rng(seed)
    gt = [np.eye(4)] + [rigid(rng) for _ in range(K - 1)]
    edges, T, L, unc = [], [], [], []
    for j, (s, d) in enumerate(list(pairs) + list(wrong)):
        Tsd = ref.inv(gt[d]) @ gt[s]
        Tsd = (rigid(rng, 0.5, 1.0) if j >= len(pairs) else rigid(rng, noise, noise)) @ Tsd
        edges.append((s, d))
        T.append(Tsd)
        L.append(overlap_info(rng, int(rng.integers(60, 200))))
        unc.append(0 if (d == s + 1 or (certain is not None and certain(s, d))) else 1)
    return gt, np.array(edges, dtype=np.int32), T, L, unc


def test_complete_graph_64(ctx):
    """2016 edges plus 3 wrong ones: every warp sum wraps 63 times, pg_edge_kernel runs 16 CTAs, GNC iterates."""
    K = 64
    pairs = [(a, b) for a in range(K) for b in range(K) if a < b]
    gt, edges, T, L, unc = make_graph(101, K, pairs, wrong=[(40, 3), (7, 60), (34, 33)])
    want = ref.optimize(K, edges, T, L, R_CORR, unc, gnc_factor=2.0)
    got = ctx.optimize_pose_graph(K, edges, T, L, R_CORR, uncertain=unc, gnc_factor=2.0)
    assert want["iterations"] > 1 and not want["mask"][-3:].any() and want["mask"][:-3].all()
    compare(got, want)
    np.testing.assert_allclose(got["weights"], want["weights"], rtol=0, atol=1e-8)


def test_chain_of_200_with_closures(ctx):
    K = 200
    pairs = [(k, k + 1) for k in range(K - 1)] + [(k, k - 10) for k in range(10, K, 7)] + [(K - 1, 0)]
    gt, edges, T, L, unc = make_graph(102, K, pairs, wrong=[(150, 20), (30, 170), (99, 101)])
    want = ref.optimize(K, edges, T, L, R_CORR, unc)
    got = ctx.optimize_pose_graph(K, edges, T, L, R_CORR, uncertain=unc)
    assert not want["mask"][-3:].any()
    compare(got, want)


def test_hub_with_parallel_edges_in_shuffled_order(ctx):
    """Node 5 is joined to every other node (its diagonal block sums K - 1 terms and more), half the hub edges point
    into the hub and half out, two pairs are listed twice (one off-diagonal block lists two terms), and the edge order is
    shuffled, so no block's terms are contiguous."""
    K, hub = 12, 5
    pairs = [(hub, j) if j % 2 else (j, hub) for j in range(K) if j != hub]
    pairs += [(k, k + 1) for k in range(K - 1) if hub not in (k, k + 1)]
    pairs += [(hub, 3), (8, hub)]
    gt, edges, T, L, unc = make_graph(103, K, pairs, wrong=[(9, 2)], certain=lambda s, d: hub in (s, d))
    perm = np.random.default_rng(3).permutation(len(edges))
    edges, T, L, unc = edges[perm], [T[i] for i in perm], [L[i] for i in perm], [unc[i] for i in perm]
    want = ref.optimize(K, edges, T, L, R_CORR, unc)
    got = ctx.optimize_pose_graph(K, edges, T, L, R_CORR, uncertain=unc)
    compare(got, want)
    assert not got["mask"][list(perm).index(len(perm) - 1)]


@pytest.mark.parametrize("where", ["last", "middle"])
def test_other_reference_node_against_the_restatement(ctx, where):
    K = 12
    r = K - 1 if where == "last" else K // 2
    pairs = [(k, k + 1) for k in range(K - 1)] + [(11, 0), (8, 0), (9, 3), (7, 2)]
    gt, edges, T, L, unc = make_graph(104, K, pairs, wrong=[(10, 4)])
    want = ref.optimize(K, edges, T, L, R_CORR, unc, ref=r)
    got = ctx.optimize_pose_graph(K, edges, T, L, R_CORR, uncertain=unc, reference_node=r)
    compare(got, want)
    assert np.array_equal(got["poses"][r], np.eye(4))


# K = 1024: a chain with a closure every 4 nodes (E = 1278), low noise, so max r-bar stays below 1/2 and GNC-TLS stops
# after its first inner solve.  The restatement's dense solve of n = 6138 is slow, so it runs once per module.
BIG_K, BIG_INNER = 1024, 6


@pytest.fixture(scope="module")
def big_graph():
    K = BIG_K
    pairs = [(k, k + 1) for k in range(K - 1)] + [(k, k - 3) for k in range(3, K, 4)]
    gt, edges, T, L, unc = make_graph(105, K, pairs, noise=0.0005)
    t0 = time.perf_counter()
    want = ref.optimize(K, edges, T, L, R_CORR, unc, max_inner_iterations=BIG_INNER)
    return edges, T, L, unc, want, time.perf_counter() - t0


def test_cap_1024_against_the_restatement(ctx, big_graph):
    """Poses to 1e-7: the long chain makes the 6138-unknown system ill-conditioned enough that the restatement's
    LAPACK factorisation and cuSOLVER's agree to about 1e-9 in the poses, not to the 1e-8 of the small graphs'
    margin."""
    edges, T, L, unc, want, _ = big_graph
    l0 = ctx.kernel_launches()
    got = ctx.optimize_pose_graph(BIG_K, edges, T, L, R_CORR, uncertain=unc, max_inner_iterations=BIG_INNER)
    assert ctx.kernel_launches() - l0 == (3 + 4 * BIG_INNER) * got["iterations"]
    assert 1 <= want["iterations"] <= 3
    compare(got, want, atol=1e-7)
    again = ctx.optimize_pose_graph(BIG_K, edges, T, L, R_CORR, uncertain=unc, max_inner_iterations=BIG_INNER)
    same_bytes(got, again)


# ---- the breadth-first start -------------------------------------------------------------------------------------------
def bfs_case(name):
    """(K, edges, T, L, unc).  'second-phase': node 2 is reached only through the uncertain (1, 2), and node 3 only
    after it; 'certain-first': node 0 lists the uncertain (0, 1) before a certain (1, 0) whose transform differs by
    0.3 rad, so the start depends on which one the walk takes."""
    rng = np.random.default_rng(106)
    gt = [np.eye(4)] + [rigid(rng) for _ in range(4)]
    if name == "second-phase":
        spec = [(0, 1, 0), (1, 2, 1), (2, 3, 0), (3, 4, 0), (4, 0, 1)]
    else:
        spec = [(0, 1, 1), (1, 0, 0), (1, 2, 0), (2, 3, 1), (3, 4, 0), (2, 4, 0), (4, 0, 1)]
    edges, T, L, unc = [], [], [], []
    for j, (s, d, u) in enumerate(spec):
        Tsd = ref.inv(gt[d]) @ gt[s]
        edges.append((s, d))
        T.append((rigid(rng, 0.3, 0.3) if j == 0 and name == "certain-first" else rigid(rng, 0.002, 0.002)) @ Tsd)
        L.append(overlap_info(rng))
        unc.append(u)
    return 5, np.array(edges, dtype=np.int32), T, L, unc


@pytest.mark.parametrize("name", ["second-phase", "certain-first"])
def test_breadth_first_start_bit_for_bit(ctx, name):
    K, edges, T, L, unc = bfs_case(name)
    start = ref.bfs(K, edges, T, [True] * len(edges), unc, 0)
    got = ctx.optimize_pose_graph(K, edges, T, L, R_CORR, uncertain=unc)
    given = ctx.optimize_pose_graph(K, edges, T, L, R_CORR, uncertain=unc, initial_poses=start)
    same_bytes(got, given)
    other = ref.bfs(K, edges, T, [True] * len(edges), [0] * len(edges), 0)  # the walk without the certain-first rule
    if name == "certain-first":
        assert not np.allclose(other[1], start[1], atol=1e-3)
    compare(got, ref.optimize(K, edges, T, L, R_CORR, unc))


def test_breadth_first_refuses_edges_that_connect_nothing(ctx):
    K, edges, T, L, unc = bfs_case("second-phase")
    keep = [0, 1, 2, 3]  # drop (4, 0): (3, 4) is node 4's only edge
    edges, T, L, unc = edges[keep], [T[i] for i in keep], [L[i] for i in keep], [unc[i] for i in keep]
    assert ctx.optimize_pose_graph(K, edges, T, L, R_CORR, uncertain=unc)["iterations"] >= 1
    L0 = [x.copy() for x in L]
    L0[3][5, 5] = 0.0  # the only bridge to node 4 carries no information
    assert ref.optimize(K, edges, T, L0, R_CORR, unc) is None
    with pytest.raises(capi.TzrError, match="connect"):
        ctx.optimize_pose_graph(K, edges, T, L0, R_CORR, uncertain=unc)
    e2 = edges.copy()
    e2[3] = (4, 4)  # node 4's only edge is a self-loop
    assert ref.optimize(K, e2, T, L, R_CORR, unc) is None
    with pytest.raises(capi.TzrError, match="connect"):
        ctx.optimize_pose_graph(K, e2, T, L, R_CORR, uncertain=unc)


# ---- information matrices past 32 chunks ------------------------------------------------------------------------------
INFO_NS = [1, 255, 256, 257, 8192, 8193, 20001]


@pytest.fixture(scope="module")
def info_problems():
    return {ns: scan_pair(200 + ns % 97, ns, 3000) for ns in INFO_NS}


@pytest.mark.parametrize("route", ["brute", "grid"])
@pytest.mark.parametrize("ns", INFO_NS)
def test_information_past_32_chunks(ctx, info_problems, ns, route):
    """20001 sources are 79 chunks: the combine's lanes wrap twice.  Both routes, bit for bit."""
    src, dst, R, t = info_problems[ns]
    want, wc = ref.information(src, dst, 1.0, R, t, R_CORR)
    got, gc = with_flags(ctx, BRUTE if route == "brute" else GRID,
                         lambda: ctx.information_matrix(src, dst, dict(scale=1.0, rotation=R, translation=t), R_CORR))
    assert gc == wc and got[5, 5] == gc
    assert got.tobytes() == want.tobytes()


def test_information_batch_of_mixed_sizes(ctx, info_problems):
    probs = [info_problems[ns] for ns in INFO_NS]
    sims = [dict(scale=1.0, rotation=p[2], translation=p[3]) for p in probs]
    singles = [ctx.information_matrix(p[0], p[1], s, R_CORR) for p, s in zip(probs, sims)]
    for order in (list(range(len(probs))), list(range(len(probs)))[::-1]):
        L, n = ctx.information_matrix_batch([probs[k][0] for k in order], [probs[k][1] for k in order],
                                            [sims[k] for k in order], R_CORR)
        for j, k in enumerate(order):
            assert L[j].tobytes() == singles[k][0].tobytes() and n[j] == singles[k][1]
