"""GPU tests of the certifier's building blocks where they can be wrong (`pytest -m gpu`, DESIGN.md 3.9).

* The nearest-PSD step, single call (the batch with B = 1: cbt_psd_kernel over cusolverDnDsyevd on the real block,
  bit for bit the batch entry with one matrix) and batch (cbt_psd_kernel, DMMA, over the batch's padded layout and
  eigen route), against matrices whose spectrum and positive part are exact in FP64
  (tests/certifier_reference.py): the first positive eigenvalue at 0, at n - 1 and either side of the 16-deep k slabs,
  n at and just past the 64-wide tiles, exact zeros, repeated and widely spread eigenvalues, and the batch at scales
  2^-40 .. 2^40, where an identity pad of fixed size would be far from the real block's scale.
* The dual projection, single (bit for bit the batch entry with one problem) and batch, at the N where its reductions change shape (a warp over N + 1 block rows,
  256-thread CTAs, 128-wide pair blocks), against oracle/certifier_oracle.py.
* The whole certifier, single and batch, on inputs scaled by 2^k: the problem is homogeneous, so the trajectory must not
  change.
* The initial matrix at rotations whose quaternion takes the trace <= 0 branch."""
import importlib
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "oracle"))
sys.path.insert(0, HERE)
import certifier_oracle as co  # noqa: E402
import certifier_reference as cr  # noqa: E402

capi = importlib.import_module("teaser-plusplus_b200.capi")
synth = importlib.import_module("teaser-plusplus_b200.synth")

pytestmark = pytest.mark.gpu
LOOP_EIG = 2097152  # debug flag: one cusolverDnDsyevd per problem instead of cusolverDnXsyevBatched


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


_CACHE = {}


def _exact(n, kind, seed=0):
    key = (n, kind, seed)
    if key not in _CACHE:
        _CACHE[key] = cr.exact_matrix(n, kind, seed)
    return _CACHE[key]


def _check_psd(got, M, P, kind, single):
    if kind == "all_negative" and single:
        assert np.all(got == 0)          # first_pos = n: no k slab runs
    err = np.linalg.norm(got - P)
    assert err <= cr.psd_bound(M), (err, cr.psd_bound(M))


# ---- 1. PSD step, single call ----------------------------------------------------------------------------------------
CASES = cr.psd_cases()


@pytest.mark.parametrize("n,kind", CASES, ids=[f"{n}-{k}" for n, k in CASES])
def test_psd_single_against_exact(ctx, n, kind):
    M, P, lam, _ = _exact(n, kind)
    got, w = ctx.certifier_psd_projection(M)
    assert np.array_equal(got, ctx.certifier_batch_psd_projection([M])[0])
    _check_psd(got, M, P, kind, single=True)
    if kind == "all_positive":
        assert np.linalg.norm(got - M) <= cr.psd_bound(M)
    assert np.abs(w - lam).max() <= cr.eig_bound(lam)


@pytest.mark.parametrize("n", [8, 68, 1028])
def test_psd_single_asymmetric_input(ctx, n):
    """An asymmetric M gives P+((M + M^T) / 2): M + K - K^T is dyadic and symmetrises back to M exactly."""
    M, P, lam, _ = _exact(n, "first_pos_1" if n == 8 else "first_pos_33")
    K = np.random.default_rng(n).integers(-64, 64, (n, n)) / 8.0
    A = M + (K - K.T)
    assert np.array_equal((A + A.T) / 2, M)
    got, w = ctx.certifier_psd_projection(A)
    assert np.array_equal(got, ctx.certifier_batch_psd_projection([A])[0])
    _check_psd(got, M, P, "", single=True)
    assert np.abs(w - lam).max() <= cr.eig_bound(lam)


# ---- 2. PSD step, batch ------------------------------------------------------------------------------------------------
_KIND_CYCLE = ("first_pos_15", "zeros", "wide", "all_negative", "repeated", "first_pos_17", "all_positive",
               "first_pos_1", "first_pos_last")
_SIZE_CYCLE = (8, 1028, 64, 132, 68, 128, 1024, 8, 64)


def _batch_problems(B, order):
    probs = []
    for b in range(B):
        n = _SIZE_CYCLE[b % len(_SIZE_CYCLE)]
        kind = _KIND_CYCLE[b % len(_KIND_CYCLE)]
        if kind.startswith("first_pos_") and kind != "first_pos_last" and int(kind.split("_")[-1]) >= n:
            kind = "first_pos_1"
        probs.append((n, kind))
    return probs if order == "forward" else probs[::-1]


@pytest.mark.parametrize("scale", (0,) + cr.SCALES)
@pytest.mark.parametrize("order", ["forward", "reversed"])
@pytest.mark.parametrize("route", ["batched", "loop", "flag"])
def test_psd_batch_against_exact(ctx, route, order, scale):
    """Ragged batches with n = 8 beside n = 1028 on the three eigen routes: 9 problems (one cusolverDnXsyevBatched
    call), 7 problems (one Dsyevd each) and 9 under flag 2097152.  Scaled by 2^s the answer scales exactly."""
    B = 7 if route == "loop" else 9
    probs = _batch_problems(B, order)
    mats = [_exact(n, k) for n, k in probs]
    Ms = [np.ldexp(m[0], scale) for m in mats]
    ctx.set_flags(LOOP_EIG if route == "flag" else 0)
    try:
        before = ctx.kernel_launches()
        outs = ctx.certifier_batch_psd_projection(Ms)
        launches = ctx.kernel_launches() - before
    finally:
        ctx.set_flags(0)
    assert launches == 3 + (1 if route == "batched" else B)   # sym, first_pos, psd + the eigensolver calls
    for (n, kind), (M, P, _, _), got in zip(probs, mats, outs):
        assert got.shape == (n, n)
        err = np.linalg.norm(np.ldexp(got, -scale) - P)
        assert err <= cr.psd_bound(M), (n, kind, err, cr.psd_bound(M))


def test_psd_batch_equal_sizes_match_single(ctx):
    """Nine equal-size problems (no pad at all) on the batched route agree with the single call within the bound."""
    mats = [_exact(132, k) for k in _KIND_CYCLE[:9]]
    outs = ctx.certifier_batch_psd_projection([m[0] for m in mats])
    for (M, P, _, _), got in zip(mats, outs):
        one, _ = ctx.certifier_psd_projection(M)
        assert np.linalg.norm(got - one) <= 2 * cr.psd_bound(M)
        assert np.linalg.norm(got - P) <= cr.psd_bound(M)


# ---- 3. dual projection ------------------------------------------------------------------------------------------------
DUAL_N = [1, 2, 31, 32, 33, 127, 128, 255, 256, 257, 1000]
THETAS = ["plus", "minus", "alternating", "single", "random"]


def _theta(N, kind, seed):
    rng = np.random.default_rng(seed)
    if kind == "plus":
        return np.ones(N)
    if kind == "minus":
        return -np.ones(N)
    if kind == "alternating":
        return np.where(np.arange(N) % 2 == 0, 1.0, -1.0)
    if kind == "single":
        t = -np.ones(N)
        t[N // 2] = 1.0
        return t
    return rng.choice([-1.0, 1.0], N)


def _W(N, seed):
    """Non-symmetric W with entries spread over 2^-8 .. 2^8."""
    rng = np.random.default_rng(seed)
    n = 4 * N + 4
    return rng.standard_normal((n, n)) * np.ldexp(1.0, rng.integers(-8, 9, (n, n)))


def _oracle_dual(W, theta, dense=False):
    thp = np.concatenate([[1.0], theta])
    return co.get_optimal_dual_projection(W, thp, A_inv=co.get_linear_projection(thp) if dense else None)


DUAL_CASES = [(N, t) for N in DUAL_N for t in THETAS if N < 1000 or t in ("single", "random")]


@pytest.mark.parametrize("N,tk", DUAL_CASES, ids=[f"{N}-{t}" for N, t in DUAL_CASES])
def test_dual_projection_single(ctx, N, tk):
    W = _W(N, N)
    th = _theta(N, tk, N + 1)
    got = ctx.certifier_dual_projection(W, th)
    assert np.array_equal(got, ctx.certifier_batch_dual_projection([W], [th])[0])
    want = _oracle_dual(W, th)
    assert np.abs(got - want).max() <= cr.dual_bound(W, N)
    if N <= 40:
        assert np.abs(got - _oracle_dual(W, th, dense=True)).max() <= cr.dual_bound(W, N)


@pytest.mark.parametrize("order", ["forward", "reversed"])
def test_dual_projection_batch(ctx, order):
    """Ragged batch (nmax != n for all but the largest): N = 1 beside N = 257, the warp and CTA wrap sizes between.
    Run twice with different W on the same layout: the second call sees the first call's W_dual in the buffer, as
    every DRS iteration after the first does."""
    Ns = [1, 257, 32, 1, 128, 33, 2, 256]
    if order == "reversed":
        Ns = Ns[::-1]
    ths = [_theta(N, THETAS[b % len(THETAS)], 100 + b) for b, N in enumerate(Ns)]
    for rep in range(2):
        Ws = [_W(N, 1000 * rep + b) for b, N in enumerate(Ns)]
        outs = ctx.certifier_batch_dual_projection(Ws, ths)
        for N, W, th, got in zip(Ns, Ws, ths, outs):
            assert got.shape == W.shape
            assert np.abs(got - _oracle_dual(W, th)).max() <= cr.dual_bound(W, N), (rep, N)
            one = ctx.certifier_dual_projection(W, th)
            assert np.abs(got - one).max() <= cr.dual_bound(W, N)


# ---- 4. whole certifier under scaling ------------------------------------------------------------------------------
def _instance(N, seed, wrong_rotation):
    rng = np.random.default_rng(seed)
    v1 = rng.uniform(-1, 1, size=(3, N))
    R = synth.random_rotation(rng)
    v2 = R @ v1
    theta = np.ones(N)
    k0 = int(N * 0.9)
    v2[:, k0:] = rng.uniform(-1, 1, size=(3, N - k0)) * 5 + 5
    theta[k0:] = -1
    if wrong_rotation:
        R = synth.random_rotation(rng)
    return R, v1, v2, theta


def _scaled(p, s):
    return p[0], s * p[1], s * p[2], p[3]


def _rel_close(a, b, tol):
    """Same length, and within tol of the trajectory's largest gap."""
    return len(a) == len(b) and np.abs(a - b).max() <= tol * max(np.abs(b).max(), 1e-300)


def _close(a, b, tol):
    """As in test_gpu_certifier_batch.py: within tol, relative to gaps above 1."""
    return len(a) == len(b) and np.abs(a - b).max() <= tol * max(1.0, np.abs(b).max())


SCALE_K = [-20, -10, 10, 20]
NB = 0.01
ITERS = 15


@pytest.mark.parametrize("k", SCALE_K)
def test_certify_single_scale_invariant(ctx, k):
    s = 2.0 ** k
    for p in (_instance(40, 5, True), _instance(25, 6, False)):
        base = ctx.certify(*p, noise_bound=NB, cbar2=1.0, max_iterations=ITERS)
        r = ctx.certify(*_scaled(p, s), noise_bound=NB * s, cbar2=1.0, max_iterations=ITERS)
        assert _rel_close(r["suboptimality_traj"], base["suboptimality_traj"], 1e-7)
        o = co.certify(*_scaled(p, s), NB * s, 1.0, max_iterations=ITERS)
        assert _close(r["suboptimality_traj"], o["suboptimality_traj"], 1e-6)
        assert r["is_optimal"] == base["is_optimal"] == o["is_optimal"]


def _batch(ctx, probs, **kw):
    return ctx.certify_batch([p[0] for p in probs], [p[1] for p in probs], [p[2] for p in probs],
                             [p[3] for p in probs], **kw)


@pytest.mark.parametrize("k", SCALE_K)
@pytest.mark.parametrize("route", ["batched", "loop"])
def test_certify_batch_scale_invariant(ctx, route, k):
    """Ten problems, two of them done on iteration 1: the batched call over all ten, then the compact batch of the
    eight still active; and the same batch on the Dsyevd loop.  Unscaled and at 2^k, against the oracle at 2^k."""
    s = 2.0 ** k
    probs = [_instance(8 + 6 * b, 300 + b, wrong_rotation=b not in (2, 7)) for b in range(10)]
    kw = dict(cbar2=1.0, max_iterations=ITERS)
    ctx.set_flags(LOOP_EIG if route == "loop" else 0)
    try:
        base = _batch(ctx, probs, noise_bound=NB, **kw)
        out = _batch(ctx, [_scaled(p, s) for p in probs], noise_bound=NB * s, **kw)
    finally:
        ctx.set_flags(0)
    lens = [len(r["suboptimality_traj"]) for r in base]
    assert lens[2] == lens[7] == 1 and max(lens) == ITERS
    for p, r, b in zip(probs, out, base):
        assert _rel_close(r["suboptimality_traj"], b["suboptimality_traj"], 1e-7)
        o = co.certify(*_scaled(p, s), NB * s, 1.0, max_iterations=ITERS)
        assert _close(r["suboptimality_traj"], o["suboptimality_traj"], 1e-6)
        assert r["is_optimal"] == b["is_optimal"] == o["is_optimal"]


# ---- 5. initial matrix on the quaternion's trace <= 0 branch ---------------------------------------------------------
def _axis_rotation(axis, angle):
    a = np.asarray(axis, dtype=np.float64)
    a = a / np.linalg.norm(a)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(angle) * K + (1 - np.cos(angle)) * K @ K


ROTATIONS = {
    "x_150deg": _axis_rotation([1, 0.1, -0.05], np.deg2rad(150)),
    "y_150deg": _axis_rotation([0.05, 1, 0.1], np.deg2rad(150)),
    "z_150deg": _axis_rotation([-0.1, 0.05, 1], np.deg2rad(150)),
    "halfturn_x": np.diag([1.0, -1.0, -1.0]),
    "halfturn_y": np.diag([-1.0, 1.0, -1.0]),
    "halfturn_z": np.diag([-1.0, -1.0, 1.0]),
    "halfturn_xy_tie": np.array([[0.0, 1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, -1.0]]),
    "trace_zero": _axis_rotation([0.3, -0.5, 0.8], np.deg2rad(120)),
}


@pytest.mark.parametrize("name", list(ROTATIONS))
def test_initial_matrix_trace_nonpositive_branch(ctx, name):
    R = ROTATIONS[name]
    assert np.trace(R) <= 1e-15 and abs(np.linalg.det(R) - 1) < 1e-12
    rng = np.random.default_rng(len(name))
    N = 23
    v1 = rng.uniform(-1, 1, (3, N))
    v2 = R @ v1 + rng.normal(0, 0.003, (3, N))
    theta = np.where(rng.uniform(size=N) < 0.8, 1.0, -1.0)
    M, mu = ctx.certifier_initial_matrix(R, v1, v2, theta, noise_bound=NB, cbar2=1.0)
    o = co.certify(R, v1, v2, theta, NB, 1.0, max_iterations=1, return_intermediates=True)
    # mu = x^T Q x sums N terms of size |v|^2 that cancel down to the residuals' size, so its rounding is relative to
    # M_init's entries (mu sits on M_init's top-left diagonal), not to mu itself
    scale = np.abs(o["M_init"]).max()
    assert abs(mu - o["mu"]) <= 1e-12 * max(abs(o["mu"]), scale)
    assert np.abs(M - o["M_init"]).max() <= 1e-12 * scale
