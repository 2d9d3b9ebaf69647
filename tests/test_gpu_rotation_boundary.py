"""The rotation stage (rot_trans.cu) where it can be wrong (run on an H100: `pytest -m gpu`).

Every device result is compared bit for bit with tests/rotation_reference.py, a float64 replay of the kernel's
operation order (the kernel is compiled with -fmad=false), and held to an exact reference: the SVD rotation to the
Procrustes maximiser of tr(R H) (Horn, 60 digits), the planar closed form to atan2, the loops to the CPU oracle within
summation-order tolerances.

What is covered: the SVD injected directly (src = I, dst = H, one iteration returns svd_rot(H); Quatro returns the yaw
of H's 2x2 block) on random, pi and pi - 1e-7 rotations, integer ties, permutations, signed diagonals, zero, rank 2 and
1, reflections with unique / tied / nearly tied sigma_3, sigma_1/sigma_3 = 1e16 and H scaled by 2^k from 2^-1070 to
2^1015; the GNC-TLS / FGR / Quatro loops at block-size edges and outlier rates, their stop rules and mask rules; whole
solves (CHAIN and COMPLETE TIMs rebuilt from the returned clique and scale, both scale paths, batches of mixed clique
sizes); and the COMPLETE workspace edge, where a clique whose TIM count exceeds the rotation workspace is reported as
too large instead of solved.
"""
import importlib
import math

import numpy as np
import pytest

import oracle_lib as orc
import rotation_reference as ref

capi = importlib.import_module("teaser-plusplus_b200.capi")

pytestmark = pytest.mark.gpu

H3 = ref.h_families()
H2 = ref.h2_families()
SWEEP = (-1070, -1060, -1000, -960, -600, 600, 1000, 1015)


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


def _bits_eq(a, b):
    """Bit-identical doubles (zeros of equal sign); any NaN equals any NaN."""
    a, b = np.asarray(a, dtype=np.float64).ravel(), np.asarray(b, dtype=np.float64).ravel()
    same = (a == b) & (np.signbit(a) == np.signbit(b))
    return a.shape == b.shape and bool(np.all(same | (np.isnan(a) & np.isnan(b))))


def _standalone(ctx, alg, x, y, nb, gnc_factor=1.4, max_iterations=100, cost_threshold=1e-6):
    """Device and replica of tzr_rotation_solve on the same TIMs; asserts they are bit-identical."""
    d = ctx.rotation_solve(alg, x, y, nb, gnc_factor, max_iterations, cost_threshold)
    r = ref.solve(alg, ref.plain_tims(x, y), nb, gnc_factor, max_iterations, cost_threshold)
    assert _bits_eq(d["R"], r["R"]), (d["R"], r["R"])
    assert _bits_eq(d["cost"], r["cost"]), (d["cost"], r["cost"])
    assert d["iterations"] == r["iterations"], (d["iterations"], r["iterations"])
    assert np.array_equal(d["inliers"], r["inliers"])
    return d, r


# ------------------------------------------------------------------------------------------------ SVD, injected
def _sweep_cases():
    H = ref.scale_sweep_h()
    return {f"sweep_2^{k}": np.ldexp(H, k) for k in SWEEP}


SVD_CASES = {**H3, **_sweep_cases()}
YAW_CASES = {**H2, **_sweep_cases()}


@pytest.mark.parametrize("name", list(SVD_CASES))
def test_svd_injected(ctx, name):
    """src = I, dst = H: H = sum_k e_k dst_k^T is H itself, and one GNC-TLS iteration returns rotation_from_H(H)."""
    H = SVD_CASES[name]
    d, _ = _standalone(ctx, 0, np.eye(3), H, 1.0, max_iterations=1)
    assert _bits_eq(d["R"], ref.svd_rot(H))
    ok, detail = ref.within_exact(d["R"], H)
    assert ok, (name, detail)


@pytest.mark.parametrize("name", list(YAW_CASES))
def test_yaw_injected(ctx, name):
    H = YAW_CASES[name]
    d, _ = _standalone(ctx, 2, np.eye(3), H, 1.0, max_iterations=1)
    if not np.any((H == 0) & np.signbit(H)):  # the reduction adds +0.0 to every entry, which turns -0.0 into +0.0
        assert _bits_eq(d["R"], ref.yaw_rot(H))
    ok, detail = ref.within_exact(d["R"], H, planar=True)
    assert ok, (name, detail)


def test_scale_sweep_device_is_invariant(ctx):
    """R(H 2^k) == R(H) bit for bit wherever H 2^k is exact (the power-of-two normalisation of H)."""
    H = ref.scale_sweep_h()
    R0 = ctx.rotation_solve(0, np.eye(3), H, 1.0, max_iterations=1)["R"]
    Y0 = ctx.rotation_solve(2, np.eye(3), H, 1.0, max_iterations=1)["R"]
    for k in (-1000, -960, -600, 600, 1000, 1015):
        Hk = np.ldexp(H, k)
        assert np.array_equal(np.ldexp(Hk, -k), H)
        assert _bits_eq(ctx.rotation_solve(0, np.eye(3), Hk, 1.0, max_iterations=1)["R"], R0), k
        assert _bits_eq(ctx.rotation_solve(2, np.eye(3), Hk, 1.0, max_iterations=1)["R"], Y0), k


# ------------------------------------------------------------------------------------------------ loops, standalone
LOOP_M = (1, 2, 3, 31, 32, 33, 127, 128, 129, 255, 256, 257, 1000, 4097)


def _mask_ok(mask, omask, w, thr):
    diff = mask != omask
    return not diff.any() or bool(np.all(np.abs(w[diff] - thr) <= 1e-9))


@pytest.mark.parametrize("alg", [0, 1, 2])
@pytest.mark.parametrize("outliers", [0.0, 0.3, 0.8])
@pytest.mark.parametrize("m", LOOP_M)
def test_loop_sizes(ctx, m, outliers, alg):
    x, y, _ = ref.tim_problem(m, outliers, 10 * m + alg + int(outliers * 10), planar=alg == 2)
    nb, thr = (0.05, 0.005) if alg == 1 else (0.01, 1e-6)
    d, r = _standalone(ctx, alg, x, y, nb, 1.4, 100, thr)
    o = (orc.gnc_tls, orc.fgr, orc.quatro)[alg](x, y, 100, thr, 1.4, nb)
    assert np.abs(d["R"] - o["R"]).max() <= 1e-9
    assert abs(d["iterations"] - o["iterations"]) <= 1
    assert _mask_ok(d["inliers"], o["inliers"], r["weights"], (0.5, 0.0, 0.4)[alg])


@pytest.mark.parametrize("alg", [0, 2])
def test_gnc_noise_free_stops_at_mu_nonpositive(ctx, alg):
    x, y, _ = ref.tim_problem(200, 0.0, 5, planar=alg == 2, noise=0.0)
    d, _ = _standalone(ctx, alg, x, y, 0.01)
    o = (orc.gnc_tls if alg == 0 else orc.quatro)(x, y, 100, 1e-6, 1.4, 0.01)
    assert d["iterations"] == o["iterations"] == 1
    assert d["cost"] == o["cost"] == math.inf
    assert d["inliers"].all()


@pytest.mark.parametrize("alg", [0, 1, 2])
def test_zero_iterations_is_identity(ctx, alg):
    x, y, _ = ref.tim_problem(100, 0.3, 6)
    d, _ = _standalone(ctx, alg, x, y, 0.01, max_iterations=0)
    assert np.array_equal(d["R"], np.eye(3)) and d["cost"] == math.inf and d["iterations"] == 0
    assert d["inliers"].all()


@pytest.mark.parametrize("alg", [0, 2])
def test_gnc_zero_cost_threshold_runs_to_the_limit(ctx, alg):
    x, y, _ = ref.tim_problem(300, 0.3, 8, planar=alg == 2)
    d, _ = _standalone(ctx, alg, x, y, 0.01, max_iterations=17, cost_threshold=0.0)
    assert d["iterations"] == 17


@pytest.mark.parametrize("alg", [0, 2])
def test_gnc_at_least_two_iterations(ctx, alg):
    """The first cost difference is |cost - inf| = inf: with mu > 0 no run stops after one iteration."""
    x, y, _ = ref.tim_problem(300, 0.5, 9, planar=alg == 2)
    d, _ = _standalone(ctx, alg, x, y, 0.01, cost_threshold=1e300)
    assert d["iterations"] == 2


@pytest.mark.parametrize("alg", [0, 2])
def test_gnc_tiny_noise_bound_substitution(ctx, alg):
    """noise_bound^2 < 1e-16 is replaced by 1e-2 (the reference's guard): 1e-9 and 0 give the same bits."""
    x, y, _ = ref.tim_problem(257, 0.3, 10, planar=alg == 2, noise=0.02)
    d, _ = _standalone(ctx, alg, x, y, 1e-9)
    d0, _ = _standalone(ctx, alg, x, y, 0.0)
    assert _bits_eq(d["R"], d0["R"]) and _bits_eq(d["cost"], d0["cost"]) and d["iterations"] == d0["iterations"]
    o = (orc.gnc_tls if alg == 0 else orc.quatro)(x, y, 100, 1e-6, 1.4, 0.0)
    assert np.abs(d["R"] - o["R"]).max() <= 1e-9 and abs(d["iterations"] - o["iterations"]) <= 1


def test_fgr_one_iteration_when_mu_below_one(ctx):
    x, y, _ = ref.tim_problem(129, 0.3, 11, spread=0.2)
    d, r = _standalone(ctx, 1, x, y, 2.0, cost_threshold=0.0)  # mu = (D / nb^2)^2 / nb^2 < 1
    assert d["iterations"] == 1


def test_fgr_weights_underflow_to_zero(ctx):
    """One iteration at a huge noise bound: the Geman-McClure weight q^2 of the farthest outliers underflows to 0
    (mask false) next to outliers whose weight is subnormal but positive (mask true)."""
    x, y, _ = ref.tim_problem(64, 0.0, 12)
    far = np.array([1e25, 1e27, 1e28, 3e29, 1e30])
    y[:far.size] = far[:, None] * np.array([0.6, 0.0, 0.8])
    d, r = _standalone(ctx, 1, x, y, 1e41, max_iterations=5)
    w = r["weights"]
    assert d["iterations"] == 1
    assert (w == 0.0).any() and ((w > 0.0) & (w < 1e-300)).any(), w[:far.size]
    assert np.array_equal(d["inliers"], w != 0.0)


def test_fgr_float_rounded_diameter(ctx):
    """The diameter is rounded to float before mu is formed; on these data the rounding changes it."""
    for k in range(4):
        x, y, _ = ref.tim_problem(100 + k, 0.2, 14 + k)
        t = ref.plain_tims(x, y)
        assert ref.diameter(t, t.x) != ref.diameter(t, t.x, rounded=False)
        _standalone(ctx, 1, x, y, 0.05, cost_threshold=0.005)


def test_quatro_ignores_z(ctx):
    x, y, _ = ref.tim_problem(300, 0.3, 15, planar=True)
    d0 = ctx.rotation_solve(2, x, y, 0.01)
    y2 = y.copy()
    y2[:, 2] = np.random.default_rng(16).normal(0, 100, y.shape[0])
    d1, _ = _standalone(ctx, 2, x, y2, 0.01)
    assert _bits_eq(d0["R"], d1["R"]) and _bits_eq(d0["cost"], d1["cost"])
    assert np.array_equal(d0["inliers"], d1["inliers"]) and d0["iterations"] == d1["iterations"]


# ------------------------------------------------------------------------------------------------ through the solve
def _cloud_problem(n_in, n_out, seed, scale=1.0, noise=5e-3):
    rng = np.random.default_rng(seed)
    n = n_in + n_out
    src = rng.uniform(-1, 1, (n, 3))
    R = ref.random_rotation(rng)
    t = rng.uniform(-1, 1, 3)
    dst = scale * src @ R.T + t + rng.uniform(-noise, noise, (n, 3))
    dst[n_in:] = rng.uniform(-5, 5, (n_out, 3))
    perm = rng.permutation(n)
    return src[perm].copy(), dst[perm].copy()


def _replay_solve(src, dst, p, clique, scale):
    build = ref.complete_tims if p.rotation_tim_graph == 1 else ref.chain_tims
    t = build(src, dst, clique, scale)
    nb = ref.rotation_noise_bound(p.noise_bound, scale)
    r = ref.solve(p.rotation_estimation_algorithm, t, nb, p.rotation_gnc_factor, p.rotation_max_iterations,
                  p.rotation_cost_threshold)
    return t, nb, r


def _check_record(rec, r):
    assert _bits_eq(capi.rotation_from_solution_record(rec), r["R"])
    assert _bits_eq(rec["gnc_cost"], r["cost"])
    assert int(rec["gnc_iterations"]) == r["iterations"]
    assert int(rec["n_rotation_inliers"]) == int(r["inliers"].sum())


@pytest.mark.parametrize("graph", [0, 1])
@pytest.mark.parametrize("alg", [0, 1, 2])
@pytest.mark.parametrize("est", [0, 1])
@pytest.mark.parametrize("n_in,n_out", [(2, 12), (3, 20), (127, 60), (128, 60), (129, 60), (300, 100)])
def test_solve_rotation_replay(ctx, n_in, n_out, est, alg, graph):
    src, dst = _cloud_problem(n_in, n_out, 100 * n_in + 10 * est + alg, scale=1.3 if est else 1.0)
    p = capi.default_params(noise_bound=0.01, estimate_scaling=est, rotation_estimation_algorithm=alg,
                            rotation_tim_graph=graph, rotation_cost_threshold=0.005 if alg == 1 else 1e-6)
    g = ctx.solve(src, dst, p)
    if not g["valid"]:
        assert g["clique"].size <= 1
        return
    t, nb, r = _replay_solve(src, dst, p, g["clique"], g["scale"])
    assert _bits_eq(g["R"], r["R"])
    assert _bits_eq(g["sol"].gnc_cost, r["cost"]) and g["gnc_iterations"] == r["iterations"]
    assert np.array_equal(g["rot_inliers"], r["inliers"])
    assert g["sol"].n_rotation_inliers == int(r["inliers"].sum())
    if graph == 0:  # the standalone entry point on the same chain TIMs gives the same bits
        d = ctx.rotation_solve(alg, t.x, t.y, nb, p.rotation_gnc_factor, p.rotation_max_iterations,
                               p.rotation_cost_threshold)
        assert _bits_eq(d["R"], r["R"]) and _bits_eq(d["cost"], r["cost"]) and d["iterations"] == r["iterations"]
        assert np.array_equal(d["inliers"], r["inliers"])


@pytest.mark.parametrize("graph", [0, 1])
@pytest.mark.parametrize("alg", [0, 1, 2])
def test_solve_batch_mixed_cliques(ctx, alg, graph):
    n = 200
    probs = [_cloud_problem(k, n - k, 7000 + k) for k in (2, 3, 40, 127, 128, 129, 190)]
    p = capi.default_params(noise_bound=0.01, estimate_scaling=0, rotation_estimation_algorithm=alg,
                            rotation_tim_graph=graph, rotation_cost_threshold=0.005 if alg == 1 else 1e-6)
    sols, cliques = ctx.solve_batch([a for a, _ in probs], [b for _, b in probs], p)
    for b, (src, dst) in enumerate(probs):
        assert sols[b]["valid"], b
        _, _, r = _replay_solve(src, dst, p, cliques[b], float(sols[b]["scale"]))
        _check_record(sols[b], r)


# ------------------------------------------------------------------------------------------------ COMPLETE workspace
def _centred_H(src, dst, clique):
    """sum over clique pairs i < j of (s_j - s_i)(d_j - d_i)^T = m * sum (s_k - mean)(d_k - mean)^T."""
    s, d = src[clique], dst[clique]
    s, d = s - s.mean(0), d - d.mean(0)
    return clique.size * (s.T @ d)


def test_complete_workspace_edge(ctx):
    """B = 256 sizes the workspace at floor(2^32 / (9 B)) = 1,864,135 TIMs per problem.  A 1932-point clique
    (1,865,346 TIMs) is too large and reported; the same batch with a 1931-point clique (1,863,415 TIMs) is solved."""
    B, n = 256, 1932
    assert (4 << 30) // (9 * B) == 1864135 and n * (n - 1) // 2 > 1864135 >= (n - 1) * (n - 2) // 2
    rng = np.random.default_rng(20)
    src = rng.uniform(-1, 1, (B, n, 3))
    dst = rng.uniform(-5, 5, (B, n, 3))
    Rt = ref.random_rotation(rng)
    for b in range(B):  # 40 noise-free inliers, the rest scattered
        dst[b, :40] = src[b, :40] @ Rt.T
    dst[0] = src[0] @ Rt.T  # problem 0: every point an inlier
    p = capi.default_params(noise_bound=0.01, estimate_scaling=0, rotation_tim_graph=1)
    with pytest.raises(capi.TzrError, match="COMPLETE"):
        ctx.solve_batch_array(src, dst, p)
    dst[0, n - 1] = [50.0, 50.0, 50.0]  # one outlier: the clique shrinks to 1931 points
    sols, cl = ctx.solve_batch_array(np.ascontiguousarray(src), np.ascontiguousarray(dst), p)
    assert sols[0]["clique_size"] == n - 1 and sols[0]["valid"]
    for b in (0, 1, B - 1):  # noise-free: one GNC pass, then mu <= 0
        m = int(sols[b]["clique_size"])
        assert sols[b]["valid"] and sols[b]["gnc_iterations"] == 1
        assert int(sols[b]["n_rotation_inliers"]) == m * (m - 1) // 2
        H = _centred_H(src[b], dst[b], cl[b, :m])
        count = m * (m - 1) // 2
        ok, detail = ref.within_exact(capi.rotation_from_solution_record(sols[b]), H, k=64.0 + count / 128)
        assert ok, (b, detail)


def test_complete_too_large_single(ctx):
    """B = 1: floor(2^32 / 9) = 477,218,588 TIMs; an all-inlier COMPLETE solve of 30895 points (477,235,065 TIMs) is
    reported before any GNC work."""
    n = 30895
    assert n * (n - 1) // 2 > (4 << 30) // 9 >= (n - 1) * (n - 2) // 2
    rng = np.random.default_rng(21)
    src = rng.uniform(-1, 1, (n, 3))
    dst = src @ ref.random_rotation(rng).T
    p = capi.default_params(noise_bound=0.01, estimate_scaling=0, rotation_tim_graph=1, use_max_clique=0)
    with pytest.raises(capi.TzrError, match="COMPLETE"):
        ctx.solve(src, dst, p)
