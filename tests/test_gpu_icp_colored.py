"""Coloured ICP and colour gradients on the device (run on an H100: `pytest -m gpu`).

The gradients against the restatement (tests/icp_colored_reference.py) bit for bit on both search routes, with ties at
the 30th place and a neighbourhood of more than 4096 points; one step against the exact step for every kernel at lambda
0, 0.968 and 1; full runs against the restatement; batches against each problem alone; lambda = 1 against the
point-to-plane entries bit for bit; normal signs; the row drop rules; lambda's range; the textured plane that
point-to-plane cannot align; the retained solve and the launch count.
"""
import importlib
import os
import subprocess
import sys

import numpy as np
import pytest

import icp_colored_reference as ref
from test_gpu_icp import _retained, perturbed, scan_pair  # noqa: F401
from test_gpu_icp_plane import as_bytes, with_flags

capi = importlib.import_module("teaser-plusplus_b200.capi")

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "teaser-plusplus_b200", "host")
CSRC = os.path.join(ROOT, "teaser-plusplus_b200", "csrc")

R_CORR = 0.05
RN = 0.15
U = 2.0 ** -53
FBRUTE, FGRID = capi.FLAG_FPFH_BRUTE_FORCE, capi.FLAG_FPFH_GRID
KERNELS = [None, ("l1", 0.0), ("huber", 0.01), ("cauchy", 0.01), ("gm", 1e-4), ("tukey", 0.03)]
KIDS = ["none", "l1", "huber", "cauchy", "gm", "tukey"]


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.set_flags(0)
    c.close()


def colours_of(pts, seed=0):
    """A smooth texture over the scans' (x, y) plus a little per-point noise."""
    p = np.asarray(pts, dtype=np.float64)
    rng = np.random.default_rng(seed)
    return (ref.texture(p[:, :2] * 2.0) + 0.01 * rng.standard_normal((len(p), 3))).astype(np.float32)


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def same(a, b):
    """Bit for bit where finite or infinite, NaN at the same places (the header leaves a NaN's payload open)."""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and np.array_equal(na, nb) and np.array_equal(_bits(np.where(na, 0.0, a)),
                                                                           _bits(np.where(nb, 0.0, b)))


@pytest.fixture(scope="module")
def case(ctx):
    """A scan pair with normals, colours of one texture (the source's seen through the true motion) and the target's
    gradients from the device at 2 r, checked once against the restatement."""
    src, dst, R, t = scan_pair(41, 1500, 1800)
    dn = ctx.estimate_normals(dst, RN)
    back = (dst.astype(np.float64) - t) @ R  # the target's points in the source frame: one texture for both
    sc, dc = colours_of(src, 1), colours_of(back, 2)
    grad = ctx.estimate_color_gradients(dst, dn, dc, 2 * R_CORR)
    return dict(src=src, dst=dst, R=R, t=t, dn=dn, sc=sc, dc=dc, grad=grad,
                init=perturbed(R, t, 41, deg=1.0, shift=0.3 * R_CORR))


# ---- gradients ----------------------------------------------------------------------------------------------------------
def test_gradients_bit_identical_on_both_routes(ctx, case):
    dst, dn, dc = case["dst"], case["dn"].copy(), case["dc"].copy()
    rng = np.random.default_rng(5)
    dn[rng.random(len(dn)) < 0.02, :3] = np.nan
    dc[rng.random(len(dc)) < 0.02, 1] = np.nan
    want = ref.color_gradients(dst, dn, dc, 2 * R_CORR)
    assert np.isnan(want).any() and (np.isfinite(want).all(1)).sum() > 0.5 * len(want)
    for flags in (0, FBRUTE, FGRID):
        got = with_flags(ctx, flags, lambda: ctx.estimate_color_gradients(dst, dn, dc, 2 * R_CORR))
        assert same(got, want), flags
    assert same(case["grad"], ref.color_gradients(dst, case["dn"], case["dc"], 2 * R_CORR))


def test_gradient_ties_at_the_thirtieth_place(ctx):
    g = np.arange(-4, 5) * 0.25
    X, Y, Z = np.meshgrid(g, g, g * 0.5, indexing="ij")
    P = np.stack([X.ravel(), Y.ravel(), Z.ravel()], axis=1).astype(np.float32)
    rng = np.random.default_rng(9)
    N = np.concatenate([rng.normal(size=(len(P), 3)), np.zeros((len(P), 1))], axis=1).astype(np.float32)
    C = rng.random((len(P), 3)).astype(np.float32)
    want = ref.color_gradients(P, N, C, 0.6)
    nb = ref.neighbours(P, 0.6, nn=31)
    assert sum(len(x) == 31 for x in nb) > 100
    for flags in (FBRUTE, FGRID):
        got = with_flags(ctx, flags, lambda: ctx.estimate_color_gradients(P, N, C, 0.6))
        assert same(got, want), flags


def test_ties_at_the_thirtieth_place_across_a_compaction(ctx):
    """A cubic lattice where interior points have more than 256 neighbours, so the selection compacts its buffer before
    the final sort, and the 30th place falls inside a shell of equal d^2 (1 + 6 + 12 + 8 = 27 nearer, 6 at two
    steps)."""
    g = np.arange(-7, 8) * 0.25
    X, Y, Z = np.meshgrid(g, g, g, indexing="ij")
    P = np.stack([X.ravel(), Y.ravel(), Z.ravel()], axis=1).astype(np.float32)
    rng = np.random.default_rng(10)
    N = np.concatenate([rng.normal(size=(len(P), 3)), np.zeros((len(P), 1))], axis=1).astype(np.float32)
    C = rng.random((len(P), 3)).astype(np.float32)
    counts = [len(x) for x in ref.neighbours(P, 1.05, nn=len(P))]
    assert sum(n > 256 for n in counts) > 200
    want = ref.color_gradients(P, N, C, 1.05)
    for flags in (FBRUTE, FGRID):
        got = with_flags(ctx, flags, lambda: ctx.estimate_color_gradients(P, N, C, 1.05))
        assert same(got, want), flags


def test_dense_neighbourhood_is_not_refused(ctx):
    """5000 points inside one radius: every point has 4999 neighbours, more than the normals' 4096."""
    rng = np.random.default_rng(4)
    P = (rng.uniform(-0.03, 0.03, (5000, 3)) * [1, 1, 0.2]).astype(np.float32)
    N = np.tile(np.array([0, 0, 1, 0], dtype=np.float32), (len(P), 1))
    C = ref.texture(P[:, :2].astype(np.float64) * 20)
    want = ref.color_gradients(P, N, C, 0.1)
    for flags in (0, FBRUTE, FGRID):
        got = with_flags(ctx, flags, lambda: ctx.estimate_color_gradients(P, N, C, 0.1))
        assert same(got, want), flags


def test_gradients_batch_equals_single(ctx, case):
    rng = np.random.default_rng(6)
    clouds = [case["dst"], case["dst"][:300], case["src"], rng.uniform(-1, 1, (5000, 3)).astype(np.float32)]
    normals = [ctx.estimate_normals(c, RN) for c in clouds]
    cols = [colours_of(c, k) for k, c in enumerate(clouds)]
    singles = [ctx.estimate_color_gradients(c, n, k, 2 * R_CORR) for c, n, k in zip(clouds, normals, cols)]
    for order in ([0, 1, 2, 3], [3, 2, 1, 0]):
        got = ctx.estimate_color_gradients_batch([clouds[j] for j in order], [normals[j] for j in order],
                                                 [cols[j] for j in order], 2 * R_CORR)
        for g, j in zip(got, order):
            assert same(g, singles[j]), j


# ---- one step -------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def small(ctx):
    """case()'s construction at 400 / 500 points, for the exact steps."""
    src, dst, R, t = scan_pair(43, 400, 500)
    dn = ctx.estimate_normals(dst, RN)
    sc, dc = colours_of(src, 3), colours_of((dst.astype(np.float64) - t) @ R, 4)
    return dict(src=src, dst=dst, dn=dn, sc=sc, dc=dc, grad=ctx.estimate_color_gradients(dst, dn, dc, 2 * R_CORR),
                init=perturbed(R, t, 43, deg=1.0, shift=0.3 * R_CORR))


def _corr_at_seed(case):
    init = case["init"]
    ev = ref.evaluate(case["src"], case["dst"], 1.0, np.asarray(init["rotation"]), init["translation"], R_CORR ** 2)
    m = ref.margins(ev["p"], case["dst"], R_CORR ** 2)
    assert m["tie"] > 1e-9 and m["bound"] > 1e-9, m
    src = np.nonzero(ev["idx"] >= 0)[0]
    return np.stack([src, ev["idx"][src]], axis=1)


@pytest.mark.parametrize("lam", [0.0, 0.968, 1.0])
@pytest.mark.parametrize("kk", range(len(KERNELS)), ids=KIDS)
def test_one_step_against_the_exact_step(ctx, small, lam, kk):
    case, kernel = small, KERNELS[kk]
    init = case["init"]
    got, _ = ctx.icp_colored(case["src"], case["dst"], case["dn"], case["sc"], case["dc"], R_CORR, init=init,
                             lambda_geometric=lam, max_iteration=1, kernel=kernel)
    corr = _corr_at_seed(case)
    loss, k = (None, 1.0) if kernel is None else kernel
    e = ref.step_exact(case["src"], case["dst"], case["dn"], case["sc"], case["dc"], case["grad"], corr, 1.0,
                       np.asarray(init["rotation"]), np.asarray(init["translation"]), lam, loss, k)
    assert got["iterations"] == 1 and e["rank"] > 0
    tol_R, tol_t = _step_tolerance(case, corr, e, lam, loss, k)
    err_R, err_t = np.abs(got["R"] - e["R"]).max(), np.abs(got["t"] - e["t"]).max()
    assert err_R <= tol_R and err_t <= tol_t, (err_R, tol_R, err_t, tol_t)


def _step_tolerance(case, corr, e, lam, loss, k):
    """(tol_R, tol_t) of a float64 step against the exact one.  Each of the 27 sums adds m terms (two rows per
    correspondence at most), so its rounding is at most 2 m u times the sum of the terms' magnitudes: SA = sum |w| |J|
    |J|^T for A and Sg = sum |w| |J| |r| for g.  The rows are formed from p rounded at its absolute size P (and q at
    Q): u and the residuals move by u (P + Q) times (1 + |g|) (the photometric row projects through the gradient), which
    moves g by that times sum |w| |J|.  Then |dx| <= (|dA| |x| + |dg|) / lambda_min over the pivoted block, R_u moves by
    |dx| plus a few u for sin / cos, and t = R_u (t0 - c) + c + x_t by |dR| |t0 - c| + |dx| + a few u |c|, |t0|."""
    init = case["init"]
    R0, t0 = np.asarray(init["rotation"]), np.asarray(init["translation"])
    ev = ref.evaluate(case["src"], case["dst"], 1.0, R0, t0, R_CORR ** 2)
    c = np.array([float(v) for v in e["c"]])
    SA, Sg, SJ = ref.system(ev, case["dst"], case["dn"], case["sc"], case["dc"], case["grad"], c,
                            ref.effective_lambda(lam), loss, k, absolute=True)
    xs = np.array([float(v) for v in e["x"]])
    m = len(corr)
    P = np.abs(ev["p"][ev["idx"] >= 0]).max() + np.abs(case["dst"].astype(np.float64)).max()
    G = 1.0 + np.abs(case["grad"][np.isfinite(case["grad"]).all(1)]).max()
    dA, dg = 2 * m * U * np.abs(SA).max(), 2 * m * U * np.abs(Sg).max() + 4 * U * P * G * np.abs(SJ).max()
    dx = 6 * (dA * np.abs(xs).max() + dg) / e["lam_min"]
    tol_R = dx + 16 * U
    tol_t = tol_R * np.linalg.norm(t0 - c) + dx + 16 * U * (np.linalg.norm(c) + np.linalg.norm(t0))
    return tol_R, tol_t


# ---- full runs ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kernel", [None, ("tukey", 0.03)], ids=["none", "tukey"])
def test_full_run_against_the_restatement(ctx, case, kernel):
    init = case["init"]
    loss, k = (None, 1.0) if kernel is None else kernel
    want = ref.icp(case["src"], case["dst"], case["dn"], case["sc"], case["dc"], R_CORR, lam=0.968, loss=loss, k=k,
                   grad=case["grad"], s=1.0, R=np.asarray(init["rotation"]), t=init["translation"], trace=True)
    for m in want["margins"]:
        assert m["tie"] > 1e-9 and m["bound"] > 1e-9, m
    got, corr = ctx.icp_colored(case["src"], case["dst"], case["dn"], case["sc"], case["dc"], R_CORR, init=init,
                                kernel=kernel)
    assert want["iterations"] > 1
    assert (got["iterations"], got["converged"], got["n_correspondences"]) == \
        (want["iterations"], want["converged"], want["n_correspondences"])
    assert np.array_equal(corr, want["corr"])
    np.testing.assert_allclose(got["R"], want["R"], rtol=0, atol=1e-8)
    np.testing.assert_allclose(got["t"], want["t"], rtol=0, atol=1e-8)


def _problems(ctx):
    probs = []
    for j, (ns, nd) in enumerate([(300, 1000), (1000, 1023), (1500, 1024), (5000, 4200), (20001, 20000)]):
        src, dst, R, t = scan_pair(80 + j, ns, nd)
        back = (dst.astype(np.float64) - t) @ R
        probs.append((src, dst, ctx.estimate_normals(dst, RN), colours_of(src, j), colours_of(back, j + 50),
                      perturbed(R, t, 80 + j, deg=1.0, shift=0.3 * R_CORR)))
    far_src, far_dst, _, _ = scan_pair(91, 300, 300)
    far_dst = far_dst + np.float32(50)
    probs.append((far_src, far_dst, ctx.estimate_normals(far_dst, RN), colours_of(far_src), colours_of(far_dst), None))
    return probs


@pytest.mark.parametrize("kernel", [None, ("huber", 0.01)], ids=["none", "huber"])
def test_batch_equals_single_forward_and_reverse(ctx, kernel):
    probs = _problems(ctx)

    def call(ps, single=False):
        return ctx.icp_colored_batch([p[0] for p in ps], [p[1] for p in ps], [p[2] for p in ps], [p[3] for p in ps],
                                     [p[4] for p in ps], R_CORR, [p[5] for p in ps], kernel=kernel, single=single)

    singles = [call([p], single=True) for p in probs]
    for j, p in enumerate(probs):
        b1 = call([p])
        assert as_bytes(b1[0]) == as_bytes(singles[j][0]) and np.array_equal(b1[1][0], singles[j][1][0])
    for order in (list(range(len(probs))), list(reversed(range(len(probs))))):
        res, corr = call([probs[j] for j in order])
        for i, j in enumerate(order):
            assert as_bytes(res[i:i + 1]) == as_bytes(singles[j][0]), j
            assert np.array_equal(corr[i], singles[j][1][0]), j
    assert singles[4][0][0]["n_correspondences"] > 10000 and singles[4][0][0]["iterations"] > 1
    far = singles[-1][0][0]
    assert (far["n_correspondences"], far["iterations"], far["converged"]) == (0, 1, 1)


# ---- lambda = 1 -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kk", range(len(KERNELS)), ids=KIDS)
def test_lambda_one_equals_point_to_plane(ctx, kk):
    kernel = KERNELS[kk]
    probs = _problems(ctx)[:4]
    args = ([p[0] for p in probs], [p[1] for p in probs], [p[2] for p in probs])
    inits = [p[5] for p in probs]
    col = ctx.icp_colored_batch(*args, [p[3] for p in probs], [p[4] for p in probs], R_CORR, inits,
                                lambda_geometric=1.0, kernel=kernel)
    plain = ctx.icp_point_to_plane_batch(*args, R_CORR, inits, kernel=kernel)
    assert as_bytes(col[0]) == as_bytes(plain[0])
    assert all(np.array_equal(a, b) for a, b in zip(col[1], plain[1]))
    if kernel is None:  # the L2 kernel runs the same system as no kernel
        l2 = ctx.icp_colored_batch(*args, [p[3] for p in probs], [p[4] for p in probs], R_CORR, inits,
                                   lambda_geometric=1.0, kernel="l2")
        assert as_bytes(l2[0]) == as_bytes(plain[0])


# ---- normals, drop rules and lambda ---------------------------------------------------------------------------------------
def test_flipped_normals_give_identical_bits(ctx, case):
    rng = np.random.default_rng(23)
    flip = case["dn"].copy()
    flip[rng.random(len(flip)) < 0.5, :3] *= -1
    flip[:, 3] = 7.0  # the fourth float is ignored
    a = ctx.icp_colored(case["src"], case["dst"], case["dn"], case["sc"], case["dc"], R_CORR, init=case["init"])
    b = ctx.icp_colored(case["src"], case["dst"], flip, case["sc"], case["dc"], R_CORR, init=case["init"])
    assert all(np.array_equal(a[0][f], b[0][f]) for f in a[0]) and np.array_equal(a[1], b[1])
    ga = ctx.estimate_color_gradients(case["dst"], flip, case["dc"], 2 * R_CORR)
    assert same(ga, case["grad"])


def test_non_finite_inputs_drop_the_rows_the_header_names(ctx, case):
    rng = np.random.default_rng(8)
    dn, sc, dc = case["dn"].copy(), case["sc"].copy(), case["dc"].copy()
    dn[rng.random(len(dn)) < 0.03, :3] = np.nan
    sc[rng.random(len(sc)) < 0.05, 0] = np.nan
    dc[rng.random(len(dc)) < 0.02, 2] = np.inf
    grad = ctx.estimate_color_gradients(case["dst"], dn, dc, 2 * R_CORR)
    assert (~np.isfinite(grad).all(1)).sum() > 10
    assert same(grad, ref.color_gradients(case["dst"], dn, dc, 2 * R_CORR))
    init = case["init"]
    want = ref.icp(case["src"], case["dst"], dn, sc, dc, R_CORR, grad=grad, R=np.asarray(init["rotation"]),
                   t=init["translation"])
    got, corr = ctx.icp_colored(case["src"], case["dst"], dn, sc, dc, R_CORR, init=init)
    assert np.isfinite(got["R"]).all() and np.isfinite(got["t"]).all()
    assert (got["iterations"], got["n_correspondences"]) == (want["iterations"], want["n_correspondences"])
    assert np.array_equal(corr, want["corr"])
    np.testing.assert_allclose(got["R"], want["R"], rtol=0, atol=1e-8)
    np.testing.assert_allclose(got["t"], want["t"], rtol=0, atol=1e-8)


def test_lambda_outside_the_unit_interval_is_the_default_and_nan_is_refused(ctx, case):
    run = lambda lam: ctx.icp_colored(case["src"], case["dst"], case["dn"], case["sc"], case["dc"], R_CORR,  # noqa
                                      init=case["init"], lambda_geometric=lam, max_iteration=5)
    base = run(0.968)
    for lam in (1.5, -0.2, 1e300):
        got = run(lam)
        assert all(np.array_equal(base[0][f], got[0][f]) for f in base[0]) and np.array_equal(base[1], got[1]), lam
    for lam in (float("nan"), float("inf")):
        with pytest.raises(capi.TzrError):
            run(lam)
    with pytest.raises(capi.TzrError):
        ctx.icp_colored(case["src"], case["dst"], case["dn"], case["sc"], case["dc"], R_CORR, kernel=("huber", -1.0))


# ---- the textured plane ---------------------------------------------------------------------------------------------------
def test_flat_textured_target_offset_removed(ctx):
    src, dst, nrm, sc, dc, off = ref.textured_plane(step=0.02, extent=1.0)
    col, _ = ctx.icp_colored(src, dst, nrm, sc, dc, R_CORR, max_iteration=30)
    pp, _ = ctx.icp_point_to_plane(src, dst, nrm, R_CORR, max_iteration=30)
    err_pp = np.linalg.norm(pp["t"][:2] - off[:2])
    err_col = np.linalg.norm(col["t"][:2] - off[:2])
    assert err_pp > 0.99 * np.linalg.norm(off[:2])
    assert err_col < 0.1 * err_pp, (err_col, err_pp)


# ---- workspace and launches -----------------------------------------------------------------------------------------------
def test_retained_solve_survives_the_new_calls(ctx, case):
    rng = np.random.default_rng(3)
    from scipy.spatial.transform import Rotation
    s = rng.uniform(-1, 1, (120, 3))
    R = Rotation.from_rotvec([0.1, 0.2, -0.1]).as_matrix()
    d = s @ R.T + [0.1, 0.0, 0.2]
    d[:30] = rng.uniform(-1, 1, (30, 3))
    ctx.solve(s, d, capi.default_params(noise_bound=0.01, estimate_scaling=0, rotation_cost_threshold=1e-12))
    before = _retained(ctx, 1)
    ctx.estimate_color_gradients(case["dst"], case["dn"], case["dc"], 2 * R_CORR)
    ctx.estimate_color_gradients_batch([case["dst"], case["src"]], [case["dn"], case["dn"][:len(case["src"])]],
                                       [case["dc"], case["sc"]], 2 * R_CORR)
    ctx.icp_colored(case["src"], case["dst"], case["dn"], case["sc"], case["dc"], R_CORR, init=case["init"])
    assert _retained(ctx, 1) == before


def test_launch_count_does_not_depend_on_B(ctx):
    src, dst, R, t = scan_pair(99, 5000, 5000)
    nrm = ctx.estimate_normals(dst, RN)
    sc, dc = colours_of(src), colours_of(dst)
    counts = []
    for B in (1, 5):
        l0 = ctx.kernel_launches()
        ctx.icp_colored_batch([src] * B, [dst] * B, [nrm] * B, [sc] * B, [dc] * B, R_CORR,
                              [perturbed(R, t, 99)] * B, max_iteration=7)
        counts.append(ctx.kernel_launches() - l0)
    assert counts == [(4 + 1) + 4 + 2 + 4 * 7] * 2  # gradient grid + pass, ICP grid, evaluation, iterations
    l0 = ctx.kernel_launches()
    ctx.icp_colored_batch([src[:500]] * 3, [dst[:500]] * 3, [nrm[:500]] * 3, [sc[:500]] * 3, [dc[:500]] * 3, R_CORR,
                          max_iteration=5)
    assert ctx.kernel_launches() - l0 == 1 + 2 + 4 * 5


# ---- voxel downsampling with colours -----------------------------------------------------------------------------------
def _sequential_means(cols, trace, m):
    """Each voxel's colour: float64 sum from 0.0 in ascending input index, divided by the count, rounded once."""
    acc, cnt = np.zeros((m, 3)), np.zeros(m)
    c64 = cols.astype(np.float64)
    for i in range(len(trace)):
        if trace[i] >= 0:
            acc[trace[i]] = acc[trace[i]] + c64[i]
            cnt[trace[i]] += 1
    return (acc / cnt[:, None]).astype(np.float32)


def test_voxel_colours_are_sequential_means_and_points_unchanged(ctx):
    rng = np.random.default_rng(12)
    clouds = [rng.uniform(-1, 1, (n, 3)).astype(np.float32) for n in (3000, 1, 700)]
    clouds[2][5] = np.nan  # a point in no voxel
    cols = [rng.random((len(c), 3)).astype(np.float32) * 255 for c in clouds]
    plain, traces = ctx.voxel_downsample_batch(clouds, 0.2, return_trace=True)
    got, gcols, gtraces = ctx.voxel_downsample_batch(clouds, 0.2, return_trace=True, colors=cols)
    for b in range(len(clouds)):
        assert got[b].tobytes() == plain[b].tobytes() and np.array_equal(gtraces[b], traces[b])
        want = _sequential_means(cols[b], traces[b], len(plain[b]))
        assert gcols[b].tobytes() == want.tobytes(), b
        p1, c1, t1 = ctx.voxel_downsample(clouds[b], 0.2, return_trace=True, colors=cols[b])
        assert p1.tobytes() == got[b].tobytes() and c1.tobytes() == gcols[b].tobytes() and np.array_equal(t1, traces[b])
    assert len(plain[0]) < len(clouds[0])
    l0 = ctx.kernel_launches()
    ctx.voxel_downsample_batch(clouds, 0.2, colors=cols)
    assert ctx.kernel_launches() - l0 == 10
    with pytest.raises(capi.TzrError):
        ctx.voxel_downsample(clouds[0], 0.2, colors=cols[0][:10])


# ---- façades -----------------------------------------------------------------------------------------------------------
def test_cpp_facade_equals_the_c_abi(tmp_path):
    """ColoredICP::refine / refineBatch, estimateColorGradients(Batch) and voxelDownSample(Batch) with colours against
    the C-ABI (tests/cpp/icp_colored_test.cc)."""
    subprocess.check_call(["make", "-s", "-C", HOST])
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    exe = str(tmp_path / "icp_colored_test")
    subprocess.check_call([cxx, "-std=c++17", "-O1", "-I", os.path.join(HOST, "include"), "-I",
                           os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "icp_colored_test.cc"),
                           "-L", HOST, "-lteaser_registration", "-L", CSRC, "-lteaser_b200",
                           f"-Wl,-rpath,{HOST}:{CSRC}", "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr


def test_pybind_equals_ctypes(ctx, case):
    subprocess.check_call(["make", "-s", "-C", HOST])
    sys.path.insert(0, os.path.join(HOST, "python"))
    import teaserpp_python as tpp
    src, dst, dn, sc, dc, init = case["src"], case["dst"], case["dn"], case["sc"], case["dc"], case["init"]
    g = tpp.estimate_color_gradients(dst, dn, dc, 2 * R_CORR)
    assert same(g, case["grad"])
    gb = tpp.estimate_color_gradients_batch([src, dst], [dn[:len(src)], dn], [sc, dc], 2 * R_CORR)
    assert same(gb[1], case["grad"])
    seed = tpp.RegistrationSolution()
    seed.scale = 1.0
    seed.rotation = np.asarray(init["rotation"], dtype=np.float64)
    seed.translation = np.asarray(init["translation"], dtype=np.float64)
    for kernel, tk in ((None, tpp.RobustKernel()), (("tukey", 0.03), tpp.RobustKernel("tukey", 0.03))):
        icp = tpp.ColoredICP(R_CORR, lambda_geometric=0.9, kernel=tk)
        got = icp.refine(src, dst, dn, sc, dc, seed)
        want, corr = ctx.icp_colored(src, dst, dn, sc, dc, R_CORR, init=init, lambda_geometric=0.9, kernel=kernel)
        assert np.array_equal(np.asarray(got["solution"].rotation), want["R"])
        assert np.array_equal(np.asarray(got["solution"].translation).ravel(), want["t"])
        assert (got["fitness"], got["inlier_rmse"], got["iterations"], got["converged"]) == \
            (want["fitness"], want["inlier_rmse"], want["iterations"], want["converged"])
        assert np.array_equal(np.array(got["correspondences"], dtype=np.int32).reshape(-1, 2), corr)
        batch = icp.refine_batch([src, src], [dst, dst], [dn, dn[:, :3]], [sc, sc], [dc, dc], [seed, seed])
        assert all(b["iterations"] == got["iterations"] and b["fitness"] == got["fitness"] for b in batch)
    vp, vc = tpp.voxel_down_sample(dst, 0.05, colors=dc)
    wp, wc = ctx.voxel_downsample(dst, 0.05, colors=dc)
    assert vp.tobytes() == wp.tobytes() and vc.tobytes() == wc.tobytes()
    assert tpp.voxel_down_sample(dst, 0.05).tobytes() == wp.tobytes()
    bp, bc = tpp.voxel_down_sample_batch([src, dst], 0.05, colors=[sc, dc])
    assert bp[1].tobytes() == wp.tobytes() and bc[1].tobytes() == wc.tobytes()
