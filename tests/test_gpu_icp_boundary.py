"""The ICP stage where it can be wrong (run on an H100: `pytest -m gpu`).

  a. One device step of every system (point-to-point, point-to-plane, generalized, and both Gauss-Newton systems under
     every robust kernel) against the exact step of tests/icp_exact_reference.py, on the wavy scans at the origin and
     at 1e4, at s in {1, 0.5, 3}, and generalized ICP with exactly parallel normals at small epsilon.
  b. The truncated 6 x 6 solve through real geometry of known rank (plane, octahedral "sphere", cylinder, wedge), the
     tolerance's edge one float32 step either side, and sums that overflow.
  c. Sums past 32 chunks: the lane wrap of the fixed-order chunk combine, for every system and both search routes.
  d. The loop's edges: the strict convergence test at a dyadic fitness step, and the automatic route switch at 1024
     targets inside one batch.

Tolerances.  A step is compared with the exact step through x (the Gauss-Newton unknowns) or the Kabsch rotation.  The
device forms every term of its sums from float64 roundings of its inputs, so each sum has an error of at most
c u S, u = 2^-53, where S is the same sum with every term replaced by a bound on its size computed from the absolute
coordinates (so that centring at 1e4 is accounted for) and, for generalized ICP, multiplied by kappa(M) (the
adjugate's relative error grows like u kappa(M)).  c = 64 bounds the roundings along one term's path: at most 6 in
the transform and the centring, 4 in a product of J entries and the residual, and one per level of the fixed-order
sum (8 inside a CTA, up to 15 over the chunks at 2^20 points, 5 in the butterfly), plus the solve's own backward error
of a few u relative to |A| (a diagonally pivoted LDL^T of order 6).  A perturbation dA, dg moves x by at most
(|dA| |x| + |dg|) / lambda_min, lambda_min the smallest eigenvalue of A on the pivoted block; for Kabsch a
perturbation dH moves R by at most |dH| / (sigma_2 + sigma_3).  The rotation update then differs by at most that
(the Euler map and the quaternion's rotation are 1-Lipschitz in the angle) plus sincos's few ulps, and t by the
rotation's error times the lever arm |t| + |c| plus the same sums' rounding at that size.  No tolerance is fitted to an
observed error.
"""
import importlib

import numpy as np
import pytest

import icp_exact_reference as ex
import icp_generalized_reference as gref
import icp_plane_reference as pref
import icp_reference as ref
import icp_robust_reference as rref
from test_gpu_icp import perturbed, scan_pair

capi = importlib.import_module("teaser-plusplus_b200.capi")

pytestmark = pytest.mark.gpu

BRUTE, GRID = capi.FLAG_ICP_BRUTE_FORCE, capi.FLAG_ICP_GRID
U = 2.0 ** -53
C_ROUND = 64
R_CORR = 0.05
RN = 0.15
KERNELS = ["l1", "huber", "cauchy", "gm", "tukey"]
K_PLANE, K_GICP = 0.02, 0.1


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.set_flags(0)
    c.close()


def as_bytes(res):
    return np.ascontiguousarray(res).tobytes()


# ---- running one step on the device ----------------------------------------------------------------------------------
def device(ctx, method, src, dst, init, sn=None, dn=None, epsilon=1e-3, kernel=None, r=R_CORR, **kw):
    if method == "point":
        return ctx.icp(src, dst, r, init=init, **kw)
    if method == "plane":
        return ctx.icp_point_to_plane(src, dst, dn, r, init=init, kernel=kernel, **kw)
    return ctx.icp_generalized(src, dst, sn, dn, r, init=init, epsilon=epsilon, kernel=kernel, **kw)


def one_step(ctx, method, src, dst, init, **kw):
    """The seed's correspondences (max_iteration = 0) and the device's first step from the same seed."""
    _, corr = device(ctx, method, src, dst, init, max_iteration=0, **kw)
    got, _ = device(ctx, method, src, dst, init, max_iteration=1, relative_fitness=-1.0, relative_rmse=-1.0, **kw)
    assert got["iterations"] == 1
    return corr, got


# ---- tolerances (module docstring) -------------------------------------------------------------------------------------
def _sizes(src, dst, corr, init, c):
    """Per correspondence: P the size p = s (R x) + t is rounded at (absolute coordinates), L = |p - c| the centred
    lever, rho = P + |q| the size the residual's operands are rounded at, d = |p - q|; and the float64 p, q."""
    x = src[corr[:, 0]].astype(np.float64)
    R, t, s = np.asarray(init["rotation"]), np.asarray(init["translation"]), float(init["scale"])
    p = s * (x @ R.T) + t
    q = dst[corr[:, 1]].astype(np.float64)
    P = np.linalg.norm(abs(s) * np.abs(x) @ np.abs(R).T + np.abs(t), axis=1) + np.linalg.norm(c)
    L = np.linalg.norm(p - c, axis=1)
    return P, L, P + np.linalg.norm(q, axis=1), np.linalg.norm(p - q, axis=1), p, q


def _weights(loss, k, r):
    """w(e) and |dw/de| at e = |r| (central difference of the restatement's weight; 0 where not finite: the device
    drops a correspondence of infinite weight)."""
    e = np.abs(r)
    if loss is None:
        return np.ones_like(e), np.zeros_like(e)
    f = lambda v: rref.weight(rref.LOSSES[loss], k, v)  # noqa: E731
    h = np.maximum(e * 1e-6, 1e-300)
    lo = np.maximum(e - h, 0.0)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        w, dw = f(e), np.abs(f(e + h) - f(lo)) / (e + h - lo)
    ok = np.isfinite(w) & np.isfinite(dw)
    return np.where(ok, w, 0.0), np.where(ok, dw, 0.0)


def tol_gn(e, src, dst, corr, init, size_i, wd_i=None, theta=0.0, energy=0.0):
    """(tol_R, tol_t) of a Gauss-Newton step.  size_i: a bound on |w_i A_i| (w |n|^2 for point-to-plane, w beta |A_i|
    for generalized ICP); wd_i: |dw/de| rho_i |A_i|, the weight's change per unit of relative rounding of the residual.
    Rounding p at its absolute size P moves the lever u = p - c and the residual by C u P, so one term of A moves by
    C u size ((L+1)^2 + 2 (L+1) P) and one of g by C u size ((L+1) rho + P d): the absolute size times the centred
    lever, never the absolute size squared.  |dx| <= (|dA| |x| + |dg|) / lambda_min, plus, for generalized ICP, the
    multiplicative change theta of each term (the determinant's relative error) in the A-norm:
    theta (|x|_A + energy) / sqrt(lambda_min), energy^2 = sum d^T A_i d.  Then t = R_u (t0 - c) + c + x_t."""
    c = np.array([float(v) for v in e["c"]])
    P, L, rho, d, _, _ = _sizes(src, dst, corr, init, c)
    wd = np.zeros_like(P) if wd_i is None else wd_i
    SA = float((size_i * ((L + 1) ** 2 + 2 * (L + 1) * P) + wd * (L + 1) ** 2).sum())
    Sg = float((size_i * ((L + 1) * rho + P * d) + wd * (L + 1) * d).sum())
    xs = np.array([float(v) for v in e["x"]])
    A = np.array([[float(v) for v in row] for row in e["A"]])
    dx = C_ROUND * U * (SA * np.linalg.norm(xs) + Sg) / e["lam_min"]
    if theta >= 1:  # the determinant may have lost every digit: no bound
        dx = np.inf
    elif theta:
        dx += theta * (np.sqrt(max(xs @ A @ xs, 0.0)) + energy) / np.sqrt(e["lam_min"]) / (1 - theta)
    tR = dx + 8 * U
    t0 = np.asarray(init["translation"], dtype=np.float64)
    tt = tR * np.linalg.norm(t0 - c) + dx + C_ROUND * U * (np.linalg.norm(c) + np.linalg.norm(t0))
    return tR, tt


def tol_kabsch(e, src, dst, corr, init):
    """(tol_R, tol_t) of a Kabsch step: centring rounds u = p - mu_p at |p| + |mu_p| and w = q - mu_q at
    |q| + |mu_q|, so dH <= C u sum ((P + |mu_p|) |w| + (|q| + |mu_q|) |u| + |u| |w|) + C u sigma_1 (the SVD);
    dR <= dH / (sigma_2 + sigma_3); t = R_u (t0 - mu_p) + mu_q."""
    mp_ = np.array([float(v) for v in e["mu_p"]])
    mq = np.array([float(v) for v in e["mu_q"]])
    P, L, _, _, _, q = _sizes(src, dst, corr, init, mp_)
    W = np.linalg.norm(q - mq, axis=1)
    SH = float((P * W + (np.linalg.norm(q, axis=1) + np.linalg.norm(mq)) * L + L * W).sum()) + e["sigma"][0]
    tR = C_ROUND * U * SH / e["gap"]
    t0 = np.asarray(init["translation"], dtype=np.float64)
    tt = tR * np.linalg.norm(t0 - mp_) + C_ROUND * U * (np.linalg.norm(mq) + np.linalg.norm(mp_) + np.linalg.norm(t0))
    return tR, tt


def plane_sizes(src, dst, dn, corr, init, c, loss=None, k=1.0):
    _, _, rho, _, p, q = _sizes(src, dst, corr, init, c)
    N = dn[corr[:, 1], :3].astype(np.float64)
    ok = np.isfinite(N).all(1)
    N = np.where(ok[:, None], N, 0.0)
    n2 = (N * N).sum(1)
    w, dw = _weights(loss, k, ((p - q) * N).sum(1))
    return w * n2, C_ROUND * U * dw * rho * np.sqrt(n2) * n2


def gicp_sizes(src_n, dst_n, src, dst, corr, init, epsilon, c, loss=None, k=1.0):
    """size_i = w beta |A_i| (beta = (s^2 + 1) / min(1, s^2) bounds |M|^2 / (det |A|): the adjugate's absolute error
    over det), wd_i, theta = C u max kappa(M_i) (det's relative error) and the energy of tol_gn, in float64 (sizes)."""
    R, s = np.asarray(init["rotation"]), float(init["scale"])
    m = src_n[corr[:, 0], :3].astype(np.float64) @ R.T
    n = dst_n[corr[:, 1], :3].astype(np.float64)
    ok = np.isfinite(m).all(1) & np.isfinite(n).all(1)
    m[~ok], n[~ok] = (0.0, 0.0, 1.0), (0.0, 0.0, 1.0)
    M = s * s * gref.covariance(m, epsilon) + gref.covariance(n, epsilon)
    ev, V = np.linalg.eigh(M)
    _, _, rho, _, p, q = _sizes(src, dst, corr, init, c)
    dv = p - q
    Wd = np.einsum("nak,nk,nbk,nb->na", V, 1 / np.sqrt(ev), V, dv)  # whitened residuals M^-1/2 d
    w, dw = _weights(loss, k, Wd)
    wmax, dwmax = w.max(1), dw.max(1)
    an = np.where(ok, 1.0 / ev[:, 0], 0.0)
    beta = (s * s + 1) / min(1.0, s * s)
    energy = np.sqrt(float((np.where(ok, wmax, 0) * np.einsum("na,nak,nk,nbk,nb->n", dv, V, 1 / ev, V, dv)).sum()))
    theta = C_ROUND * U * float((ev[ok, 2] / ev[ok, 0]).max())
    return wmax * beta * an, C_ROUND * U * dwmax * rho * np.sqrt(an) * an, theta, energy


def check_step(got, e, tR, tt):
    errR = float(np.abs(got["R"] - e["R"]).max())
    errt = float(np.abs(got["t"] - e["t"]).max())
    assert errR <= tR and errt <= tt, (errR, tR, errt, tt)
    return errR, errt


# ---- a. exact steps ----------------------------------------------------------------------------------------------------
def _problem(ctx, seed, ns, offset, s, with_src_normals=False):
    off = np.asarray(offset, dtype=np.float64)
    src, dst, R, t = scan_pair(seed, ns, ns, offset=tuple(off))
    if s != 1.0:  # the target is s (R x) + t of the source: shrink the source so that the seed's scale brings it back
        src = ((src.astype(np.float64) - off) / s + off / s).astype(np.float32)
    init = perturbed(R, t, seed, deg=1.0, shift=0.3 * R_CORR, center=tuple(off))
    init["scale"] = s
    dn = ctx.estimate_normals(dst, RN)
    sn = ctx.estimate_normals(src, RN / s) if with_src_normals else None
    return src, dst, init, sn, dn


OFFSETS = {"origin": (0.5, -0.2, 2.0), "far": (1e4, -1e4, 5e3)}


def exact_and_tol(method, src, dst, corr, init, sn=None, dn=None, epsilon=1e-3, loss=None, k=1.0):
    """The exact step and its (tol_R, tol_t)."""
    s, R0, t0 = float(init["scale"]), np.asarray(init["rotation"]), np.asarray(init["translation"])
    if method == "point":
        e = ex.step_point(src, dst, corr, s, R0, t0)
        return e, tol_kabsch(e, src, dst, corr, init)
    if method == "plane":
        e = ex.step_plane(src, dst, dn, corr, s, R0, t0, loss, k)
        c = np.array([float(v) for v in e["c"]])
        return e, tol_gn(e, src, dst, corr, init, *plane_sizes(src, dst, dn, corr, init, c, loss, k))
    e = ex.step_generalized(src, dst, sn, dn, corr, s, R0, t0, epsilon, loss, k)
    c = np.array([float(v) for v in e["c"]])
    size, wd, theta, energy = gicp_sizes(sn, dn, src, dst, corr, init, epsilon, c, loss, k)
    return e, tol_gn(e, src, dst, corr, init, size, wd, theta, energy)


def _float32_step(method, src, dst, corr, init, sn, dn):
    """The restatement's step with every transformed point rounded to float32: a loss of precision at the absolute
    size that a centred computation must not have."""
    R0, t0 = np.asarray(init["rotation"]), np.asarray(init["translation"])
    ev = _ev(src, dst, corr, init)
    ev["p"] = ev["p"].astype(np.float32).astype(np.float64)
    if method == "point":
        Ru, tu = ref.update(ev, dst)
    elif method == "plane":
        Ru, tu = pref.update(ev, dst, dn)
    else:
        Ru, tu = gref.Update(sn, init["scale"], R0, 1e-3)(ev, dst, dn)
    return Ru @ R0, Ru @ t0 + tu


@pytest.mark.parametrize("where", sorted(OFFSETS))
@pytest.mark.parametrize("s", [1.0, 0.5, 3.0])
@pytest.mark.parametrize("method", ["point", "plane", "generalized"])
def test_step_is_the_exact_step(ctx, method, s, where):
    gen = method == "generalized"
    src, dst, init, sn, dn = _problem(ctx, 31, 700 if gen else 1500, OFFSETS[where], s, with_src_normals=gen)
    corr, got = one_step(ctx, method, src, dst, init, sn=sn, dn=dn)
    assert len(corr) > 0.5 * len(src)
    e, (tR, tt) = exact_and_tol(method, src, dst, corr, init, sn, dn)
    if method != "point":
        assert e["rank"] == 6
    err = check_step(got, e, tR, tt)
    print(f"{method} s={s} {where}: |dR| {err[0]:.2e} (tol {tR:.2e}), |dt| {err[1]:.2e} (tol {tt:.2e})")
    # the step moved well beyond the tolerance: an identity or a transposed step would not match
    assert np.abs(e["R"] - np.asarray(init["rotation"])).max() > 10 * tR
    if where == "far":  # and a step computed from float32 points at 1e4 is rejected
        R32, t32 = _float32_step(method, src, dst, corr, init, sn, dn)
        assert np.abs(R32 - e["R"]).max() > tR or np.abs(t32 - e["t"]).max() > tt


@pytest.mark.parametrize("loss", KERNELS)
@pytest.mark.parametrize("method", ["plane", "generalized"])
def test_robust_step_is_the_exact_step(ctx, method, loss):
    d = rref.clutter_pair(5, n=1500 if method == "plane" else 400)
    init = dict(scale=1.0, rotation=d["R0"], translation=d["t0"])
    k = K_PLANE if method == "plane" else K_GICP
    kw = dict(sn=d["src_normals"], dn=d["dst_normals"])
    corr, got = one_step(ctx, method, d["src"], d["dst"], init, r=d["r"], kernel=(loss, k), **kw)
    e, (tR, tt) = exact_and_tol(method, d["src"], d["dst"], corr, init, loss=loss, k=k, **kw)
    assert e["rank"] == 6
    err = check_step(got, e, tR, tt)
    print(f"{method} {loss}: |dR| {err[0]:.2e} (tol {tR:.2e}), |dt| {err[1]:.2e} (tol {tt:.2e})")
    assert np.abs(e["R"] - d["R0"]).max() > 10 * tR


def _parallel_problem(ctx, s, n=400):
    """The wavy scan with the seed's rotation the identity and every source normal the very floats of its seed
    correspondence's target normal, so that m' = R m = n exactly and M has the eigenvalue (s^2 + 1) epsilon."""
    src, dst, _, _ = scan_pair(41, n, n)
    src = src + np.float32(0.01)
    init = dict(scale=s, rotation=np.eye(3), translation=np.array([0.004, -0.003, 0.002]))
    if s != 1.0:
        src = (src.astype(np.float64) / s).astype(np.float32)
    dn = ctx.estimate_normals(dst, RN)
    _, corr = ctx.icp(src, dst, R_CORR, init=init, max_iteration=0)
    sn = np.full((len(src), 4), np.nan, dtype=np.float32)
    sn[corr[:, 0]] = dn[corr[:, 1]]
    return src, dst, init, sn, dn


@pytest.mark.parametrize("epsilon", [1e-3, 1e-6, 1e-9])
def test_generalized_step_with_parallel_normals(ctx, epsilon):
    """The bound grows like u / epsilon once: the adjugate's absolute error is C u beta |A_i| (beta = 2 here), and
    the determinant's relative error theta = C u kappa(M) = C u / epsilon scales each term as a whole, which moves x by
    theta in the A-norm.  The step must exceed ten times it, so a dropped or identity system fails."""
    src, dst, init, sn, dn = _parallel_problem(ctx, 1.0)
    corr, got = one_step(ctx, "generalized", src, dst, init, sn=sn, dn=dn, epsilon=epsilon)
    e, (tR, tt) = exact_and_tol("generalized", src, dst, corr, init, sn, dn, epsilon)
    ok = np.isfinite(dn[corr[:, 1], :3]).all(1)
    assert e["used"] == ok.sum() > 100 and abs(e["kappa"] * epsilon - 1) < 1e-6
    err = check_step(got, e, tR, tt)
    print(f"parallel normals, epsilon {epsilon:.0e}: |dR| {err[0]:.2e} (tol {tR:.2e}), |dt| {err[1]:.2e} (tol {tt:.2e})")
    assert np.abs(e["R"] - np.eye(3)).max() > 10 * tR and np.abs(e["t"] - init["translation"]).max() > 10 * tt


def test_epsilon_floor_on_the_device(ctx):
    """The generalized step with m' = n at decreasing epsilon against the exact step: the adjugate's relative error
    grows like u / epsilon, so the step's error does too.  Prints the table DESIGN.md §3.14 records.  Each accepted
    epsilon's error must stay within its own bound (test_generalized_step_with_parallel_normals's); below 1e-12 the
    bound exceeds the step, and the row is printed only."""
    src, dst, init, sn, dn = _parallel_problem(ctx, 1.0, n=300)
    for epsilon in (1e-3, 1e-6, 1e-9, 1e-10, 1e-11, 1e-12, 1e-15, 1e-20):
        corr, got = one_step(ctx, "generalized", src, dst, init, sn=sn, dn=dn, epsilon=epsilon)
        e, (tR, tt) = exact_and_tol("generalized", src, dst, corr, init, sn, dn, epsilon)
        errR = float(np.abs(got["R"] - e["R"]).max())
        errt = float(np.abs(got["t"] - e["t"]).max())
        step = float(np.abs(e["R"] - np.eye(3)).max())
        print("epsilon %.0e: |dR| %.2e |dt| %.2e (tol %.2e %.2e, step %.2e)" % (epsilon, errR, errt, tR, tt, step))
        if tR < step:
            assert errR <= tR and errt <= tt, epsilon


# ---- b. the truncated solve through geometry of known rank -------------------------------------------------------------
def _shape(kind):
    """Dyadic targets with axis-aligned normals (0.25 grid), a count that is a power of two, and per-point
    displacements a_i along the normal (multiples of 2^-8): the source is q_i + a_i n_i.  Every sum of the system is
    then exact in float64."""
    g = np.arange(-3.5, 4.0, 1.0) * 0.25  # 8 values, symmetric
    pts, nrm = [], []
    rng = np.random.default_rng(len(kind))
    if kind == "plane":  # z = 0: rank 3 (rotations about x and y, t_z)
        for x in g:
            for y in g:
                pts.append((x, y, 0.0))
                nrm.append((0.0, 0.0, 1.0))
    elif kind == "sphere":  # radial normals about the centroid: every lever is parallel to its normal, rank 3
        for k, sgn, off in [(0, 1, 0), (0, -1, 0), (1, 1, 0), (1, -1, 0), (2, 1, 0), (2, -1, 0), (2, 1, 1), (2, -1, 1)]:
            v = np.zeros(3)
            v[k] = sgn
            for j in range(8):
                pts.append(tuple(v * (1.0 + j / 8 + off / 16)))
                nrm.append(tuple(v))
    elif kind == "cylinder":  # axis z: rank 4 (no rotation about z, no t_z)
        for z in np.arange(-7.5, 8.0, 1.0) * 0.125:
            for v in [(1.0, 0.0), (-1.0, 0.0), (0.0, 1.0), (0.0, -1.0)]:
                pts.append((v[0], v[1], z))
                nrm.append((v[0], v[1], 0.0))
    elif kind == "wedge":  # planes z = -1 and x = -1 meeting along a line parallel to y: rank 5 (no t_y)
        for a in g:
            for b in g:
                pts.append((a, b, -1.0))
                nrm.append((0.0, 0.0, 1.0))
                pts.append((-1.0, b, a))
                nrm.append((1.0, 0.0, 0.0))
    q = np.array(pts, dtype=np.float64)
    n = np.array(nrm, dtype=np.float64)
    a = rng.integers(-4, 5, size=len(q)) * 2.0 ** -8
    if kind == "sphere":  # opposite poles move alike, so the centroid stays at the centre
        a = np.repeat(rng.integers(-4, 5, size=(4, 1, 8)) * 2.0 ** -8, 2, axis=1).reshape(-1)
    src = q + a[:, None] * n
    if kind == "sphere":  # and a common shift, so that the step has a translation to find
        src = src + np.array([2.0 ** -7, -(2.0 ** -8), 2.0 ** -7])
    return src.astype(np.float32), q.astype(np.float32), np.concatenate([n, np.zeros((len(n), 1))], 1).astype(np.float32)


@pytest.mark.parametrize("kind,rank", [("plane", 3), ("sphere", 3), ("cylinder", 4), ("wedge", 5)])
def test_known_rank_geometry(ctx, kind, rank):
    src, dst, dn = _shape(kind)
    assert len(src) & (len(src) - 1) == 0
    init = dict(scale=1.0, rotation=np.eye(3), translation=np.zeros(3))
    r = 0.03  # above every displacement (<= 2^-6), below half of every target spacing
    corr, got = one_step(ctx, "plane", src, dst, init, dn=dn, r=r)
    assert len(corr) == len(src)
    e = ex.step_plane(src, dst, dn, corr, 1.0, np.eye(3), np.zeros(3))
    assert e["rank"] == rank
    # the sums are exact, so the device's A and g are the exact ones; what remains is the solve's rounding on the
    # pivoted block (C u cond |x|) and sincos
    xs = np.array([float(v) for v in e["x"]])
    tol = C_ROUND * U * (e["lam_max"] / e["lam_min"]) * np.abs(xs).max() + 8 * U
    np.testing.assert_allclose(got["R"], e["R"], rtol=0, atol=tol)
    # t = R_u (t0 - c) + c + x_t with t0 = 0: the rotation's error times the lever |c|, plus x_t's own and the
    # rounding of c + x_t (every centroid here is within 4 of the origin)
    c = np.array([float(v) for v in e["c"]])
    np.testing.assert_allclose(got["t"], e["t"], rtol=0, atol=tol * (1 + np.linalg.norm(c)) + tol + 8 * U * 4)
    assert np.abs(xs).max() > 1e-3


def _tol_problem(f):
    """Targets on the x axis at +-1..+-7 (normal e_x) and two at (0, +-1, 0) whose normal is (0, f, 0): A is
    diag(0, 0, 0, 14, 2 f^2, 0) exactly (every lever is parallel to its normal), g = (0, 0, 0, 14 dx, 2 f^2 dy, 0)."""
    q = [(float(x), 0.0, 0.0) for x in range(-7, 8) if x] + [(0.0, 1.0, 0.0), (0.0, -1.0, 0.0)]
    n = [(1.0, 0.0, 0.0)] * 14 + [(0.0, float(f), 0.0)] * 2
    q = np.array(q, dtype=np.float32)
    delta = np.array([2.0 ** -6, 2.0 ** -7, 0.0])
    return (q + delta).astype(np.float32), q, np.concatenate([np.array(n), np.zeros((16, 1))], 1).astype(np.float32), \
        delta


def test_truncation_at_the_tolerance_edge(ctx):
    tol = np.float64(1e-10) * 14.0
    f = np.float32(np.sqrt(tol / 2))
    while 2.0 * np.float64(f) ** 2 <= tol:
        f = np.nextafter(f, np.float32(1))
    while 2.0 * np.float64(np.nextafter(f, np.float32(0))) ** 2 > tol:
        f = np.nextafter(f, np.float32(0))
    lo = np.nextafter(f, np.float32(0))
    assert 2.0 * np.float64(f) ** 2 > tol >= 2.0 * np.float64(lo) ** 2
    init = dict(scale=1.0, rotation=np.eye(3), translation=np.zeros(3))
    for ff, taken in ((f, True), (lo, False)):
        src, dst, dn, delta = _tol_problem(ff)
        corr, got = one_step(ctx, "plane", src, dst, init, dn=dn, r=0.0625)
        assert len(corr) == 16
        e = ex.step_plane(src, dst, dn, corr, 1.0, np.eye(3), np.zeros(3))
        assert e["rank"] == (2 if taken else 1) and e["piv"][0] == 3
        assert np.array_equal(got["R"], np.eye(3))
        want = -delta if taken else np.array([-delta[0], 0.0, 0.0])
        assert np.array_equal(got["t"], want), (ff, got["t"])
        assert np.array_equal(e["t"], want)


def _four_squares(K):
    """Four integers whose squares sum to K (Lagrange), by search from the largest."""
    from math import isqrt
    for a in range(isqrt(K), -1, -1):
        r1 = K - a * a
        for b in range(min(a, isqrt(r1)), -1, -1):
            r2 = r1 - b * b
            for c in range(min(b, isqrt(r2)), -1, -1):
                dd = r2 - c * c
                if isqrt(dd) ** 2 == dd:
                    return a, b, c, isqrt(dd)
    raise AssertionError(K)


def test_diagonal_exactly_at_the_tolerance_is_truncated(ctx):
    """A(4,4) == fl(1e-10 max A_kk) exactly: the pivot test is strict, so the pivot is not taken.  Targets at x = +-1..+-5
    (normal e_x, A(3,3) = 10) and at y = +-1, +-2, +-3 with normals (0, f_j, 0): A(4,4) = sum f_j^2.  f_1 (twice) is
    the largest float32 with 2 f_1^2 <= tol; the rest, tol - 2 f_1^2 = K 2^(2e), is four squares m_j^2 2^(2e) with
    f_j = m_j 2^e, so every f_j^2 and every partial sum is exact in float64."""
    from fractions import Fraction as F
    tol = np.float64(1e-10) * 10.0
    f1 = np.float32(np.sqrt(tol / 2))
    while 2.0 * np.float64(f1) ** 2 > tol:
        f1 = np.nextafter(f1, np.float32(0))
    res = F(float(tol)) - 2 * F(float(f1)) ** 2
    e = next(e for e in range(-30, -60, -1) if (res / F(2) ** (2 * e)).denominator == 1)
    K = res / F(2) ** (2 * e)
    assert K.denominator == 1 and 0 < K < 2 ** 48
    ms = _four_squares(int(K))
    fs = [float(f1), float(f1)] + [float(np.float32(m * 2.0 ** e)) for m in ms]
    assert all(F(f) == F(m) * F(2) ** e for f, m in zip(fs[2:], ms))
    assert sum(F(f) ** 2 for f in fs) == F(float(tol))
    ys = [1.0, -1.0, 2.0, -2.0, 3.0, -3.0]
    q = [(float(x), 0.0, 0.0) for x in range(-5, 6) if x] + [(0.0, y, 0.0) for y in ys]
    n = [(1.0, 0.0, 0.0)] * 10 + [(0.0, f, 0.0) for f in fs]
    q = np.array(q, dtype=np.float32)
    delta = np.array([2.0 ** -6, 2.0 ** -7, 0.0])
    src = (q + delta).astype(np.float32)
    dn = np.concatenate([np.array(n), np.zeros((16, 1))], 1).astype(np.float32)
    init = dict(scale=1.0, rotation=np.eye(3), translation=np.zeros(3))
    corr, got = one_step(ctx, "plane", src, q, init, dn=dn, r=0.0625)
    assert len(corr) == 16
    ex_step = ex.step_plane(src, q, dn, corr, 1.0, np.eye(3), np.zeros(3))
    assert ex_step["A"][4][4] == F(float(tol)) and ex_step["rank"] == 1
    assert np.array_equal(got["t"], [-delta[0], 0.0, 0.0]) and np.array_equal(got["R"], np.eye(3))


def test_overflowing_sums_give_the_identity(ctx):
    """s = 1e130 puts the points near 1e130, r = 1e200 (r^2 = inf) still matches them, and normals of size 1e38 give
    levers whose squares overflow: the rotation diagonals are inf, so tol = 1e-10 inf = inf, no pivot is taken, and
    the update is the identity."""
    rng = np.random.default_rng(5)
    src = rng.uniform(-1, 1, (64, 3)).astype(np.float32)
    dst = rng.uniform(-1, 1, (64, 3)).astype(np.float32)
    dn = np.tile(np.array([1e38, -1e38, 1e38, 0], dtype=np.float32), (64, 1))
    init = dict(scale=1e130, rotation=np.eye(3), translation=np.zeros(3))
    for method in ("plane", "generalized"):
        got, corr = device(ctx, method, src, dst, init, sn=dn, dn=dn, r=1e200, max_iteration=1, relative_fitness=-1,
                           relative_rmse=-1)
        assert got["n_correspondences"] == 64 and got["iterations"] == 1
        assert np.array_equal(got["R"], np.eye(3)) and np.array_equal(got["t"], np.zeros(3)), method


# ---- c. sums past 32 chunks --------------------------------------------------------------------------------------------
def _wide(ctx, ns, seed=61):
    src, dst, R, t = scan_pair(seed, ns, max(ns, 2000))
    init = perturbed(R, t, seed, deg=1.0, shift=0.3 * R_CORR)
    return src, dst, init, ctx.estimate_normals(src, RN), ctx.estimate_normals(dst, RN)


def _ev(src, dst, corr, init):
    p = ref.transform(src, init["scale"], np.asarray(init["rotation"]), init["translation"])
    idx = np.full(len(src), -1)
    idx[corr[:, 0]] = corr[:, 1]
    return dict(p=p, idx=idx)


def _restated(method, src, dst, corr, init, sn, dn, kernel=None):
    ev = _ev(src, dst, corr, init)
    R0, t0 = np.asarray(init["rotation"]), np.asarray(init["translation"])
    if method == "point":
        Ru, tu = ref.update(ev, dst)
    elif method == "plane" and kernel:
        Ru, tu = rref.PlaneUpdate(rref.LOSSES[kernel[0]], kernel[1])(ev, dst, dn)
    elif method == "plane":
        Ru, tu = pref.update(ev, dst, dn)
    elif kernel:
        Ru, tu = rref.GicpUpdate(sn, init["scale"], R0, 1e-3, rref.LOSSES[kernel[0]], kernel[1])(ev, dst, dn)
    else:
        Ru, tu = gref.Update(sn, init["scale"], R0, 1e-3)(ev, dst, dn)
    return Ru @ R0, Ru @ t0 + tu


@pytest.mark.parametrize("ns", [255, 256, 257, 8192, 8193, 20001])
@pytest.mark.parametrize("method", ["point", "plane", "generalized", "plane-huber", "generalized-cauchy"])
def test_sums_past_32_chunks(ctx, method, ns):
    method, _, loss = method.partition("-")
    kernel = (loss, K_PLANE if method == "plane" else K_GICP) if loss else None
    src, dst, init, sn, dn = _wide(ctx, ns)
    res = []
    for flag in (BRUTE, GRID):
        ctx.set_flags(flag)
        try:
            res.append((device(ctx, method, src, dst, init, sn=sn, dn=dn, kernel=kernel, max_iteration=0),
                        one_step(ctx, method, src, dst, init, sn=sn, dn=dn, kernel=kernel)))
        finally:
            ctx.set_flags(0)
    (z0, c0), (z1, c1) = res[0][0], res[1][0]
    assert as_bytes(np.array([z0["fitness"], z0["inlier_rmse"]])) == as_bytes(np.array([z1["fitness"], z1["inlier_rmse"]]))
    assert np.array_equal(c0, c1) and np.array_equal(res[0][1][1]["R"], res[1][1][1]["R"])
    corr, got = res[0][1]
    # the evaluation's sums: the count and sum d^2 over every chunk
    assert z0["n_correspondences"] == len(corr) > 0.5 * ns and z0["fitness"] == len(corr) / ns
    p = ref.transform(src[corr[:, 0]], init["scale"], np.asarray(init["rotation"]), init["translation"])
    d2 = ((p - dst[corr[:, 1]].astype(np.float64)) ** 2).sum(1)
    assert abs(z0["inlier_rmse"] - np.sqrt(d2.mean())) <= 1e-12 * z0["inlier_rmse"]
    R1, t1 = _restated(method, src, dst, corr, init, sn, dn, kernel)
    np.testing.assert_allclose(got["R"], R1, rtol=0, atol=1e-10)
    np.testing.assert_allclose(got["t"], t1, rtol=0, atol=1e-10)


@pytest.mark.parametrize("method", ["point", "plane", "generalized"])
def test_only_chunk_35_matches(ctx, method):
    """ns = 40 * 256, and only the points of chunk 35 lie within r of a target: the count, H and the 27 sums all come
    from lane 3's second chunk of the combine."""
    src, dst, init, sn, dn = _wide(ctx, 2000, seed=62)
    far = np.float32(100.0)
    big = np.full((40 * 256, 3), far, dtype=np.float32) + np.arange(40 * 256, dtype=np.float32)[:, None] * 0.5
    big[35 * 256:35 * 256 + 256] = src[:256]
    bsn = np.tile(sn[:1], (40 * 256, 1))
    bsn[35 * 256:36 * 256] = sn[:256]
    _, corr0 = device(ctx, method, src[:256], dst, init, sn=sn[:256], dn=dn, max_iteration=0)
    corr, got = one_step(ctx, method, big, dst, init, sn=bsn, dn=dn)
    assert len(corr) == len(corr0) > 100 and (corr[:, 0] // 256 == 35).all()
    alone, _ = device(ctx, method, src[:256], dst, init, sn=sn[:256], dn=dn, max_iteration=1, relative_fitness=-1.0,
                      relative_rmse=-1.0)
    R1, t1 = _restated(method, big, dst, corr, init, bsn, dn)
    np.testing.assert_allclose(got["R"], R1, rtol=0, atol=1e-10)
    np.testing.assert_allclose(got["t"], t1, rtol=0, atol=1e-10)
    assert np.abs(got["R"] - np.asarray(init["rotation"])).max() > 1e-6
    np.testing.assert_allclose(got["R"], alone["R"], rtol=0, atol=1e-12)


def test_ragged_batch_of_chunk_boundaries(ctx):
    probs = [_wide(ctx, ns, seed=70 + k) for k, ns in enumerate([255, 256, 257, 8192, 8193, 20001])]
    calls = {
        "point": lambda P: ctx.icp_batch([p[0] for p in P], [p[1] for p in P], R_CORR, [p[2] for p in P],
                                         max_iteration=5),
        "plane": lambda P: ctx.icp_point_to_plane_batch([p[0] for p in P], [p[1] for p in P], [p[4] for p in P],
                                                        R_CORR, [p[2] for p in P], max_iteration=5),
        "generalized": lambda P: ctx.icp_generalized_batch([p[0] for p in P], [p[1] for p in P], [p[3] for p in P],
                                                           [p[4] for p in P], R_CORR, [p[2] for p in P],
                                                           max_iteration=5)}
    for method, call in calls.items():
        singles = [call([p]) for p in probs]
        for order in (list(range(len(probs))), list(reversed(range(len(probs))))):
            res, corr = call([probs[k] for k in order])
            for j, k in enumerate(order):
                assert as_bytes(res[j:j + 1]) == as_bytes(singles[k][0]), (method, k)
                assert np.array_equal(corr[j], singles[k][1][0])


# ---- d. the loop's edges -----------------------------------------------------------------------------------------------
def test_convergence_test_is_strict_at_a_dyadic_fitness_step(ctx):
    """ns = 2^10: a 32 x 32 grid shifted by delta, and one corner point lifted by h so that it lies beyond r at the seed
    and within r once the first step has removed delta.  The fitness then moves by exactly 2^-10 at iteration 1 and by
    0 at iteration 2, and relative_rmse is huge: relative_fitness = 2^-10 must not converge at iteration 1 (the test is
    strict) and nextafter(2^-10, inf) must."""
    g = np.arange(32) * 0.25
    X, Y = np.meshgrid(g, g)
    dst = np.stack([X.ravel(), Y.ravel(), np.zeros(1024)], axis=1).astype(np.float32)
    src = (dst.astype(np.float64) + [0.03, 0.0, 0.0]).astype(np.float32)
    src[-1, 2] = np.float32(0.045)  # |(0.03, 0, 0.045)| > 0.05 > 0.045
    r = 0.05
    z, _ = ctx.icp(src, dst, r, max_iteration=0)
    one, _ = ctx.icp(src, dst, r, max_iteration=1, relative_fitness=-1, relative_rmse=-1)
    assert (z["n_correspondences"], one["n_correspondences"]) == (1023, 1024)
    assert one["fitness"] - z["fitness"] == 2.0 ** -10
    for rf, iters in ((2.0 ** -10, 2), (np.nextafter(2.0 ** -10, np.inf), 1)):
        got, _ = ctx.icp(src, dst, r, max_iteration=5, relative_fitness=rf, relative_rmse=1e30)
        want = ref.icp(src, dst, r, max_iteration=5, relative_fitness=rf, relative_rmse=1e30)
        assert (got["iterations"], got["converged"]) == (want["iterations"], want["converged"]) == (iters, True), rf


def test_batch_converging_at_different_iterations(ctx):
    """One batch whose problems stop at iteration 1 (no correspondence), at several iterations, and at max_iteration:
    each as it does alone.  That the third problem, seeded 4 degrees off, still moves by more than 1e-6 in fitness or
    rmse at iteration 4 is a property of its seed, checked by the last assertion."""
    src, dst, R, t = scan_pair(95, 1500, 1500)
    far = (dst + np.float32(10.0)).astype(np.float32)
    probs = [(src, far, None), (src, dst, perturbed(R, t, 95)), (src, dst, perturbed(R, t, 96, deg=4.0))]
    res, _ = ctx.icp_batch([p[0] for p in probs], [p[1] for p in probs], R_CORR, [p[2] for p in probs],
                           max_iteration=4)
    its = [int(r["iterations"]) for r in res]
    for k, p in enumerate(probs):
        alone, _ = ctx.icp_batch([p[0]], [p[1]], R_CORR, [p[2]], max_iteration=4)
        assert as_bytes(alone) == as_bytes(res[k:k + 1]), k
    assert its[0] == 1 and res[0]["converged"] and 1 < its[1] and its[2] == 4 and not res[2]["converged"], its


def test_automatic_route_switch_inside_one_batch(ctx):
    probs = []
    for k, nd in enumerate([1023, 1024, 5000]):
        src, dst, R, t = scan_pair(90 + k, 1500, nd)
        probs.append((src, dst, ctx.estimate_normals(dst, RN), perturbed(R, t, 90 + k)))
    run = lambda: ctx.icp_point_to_plane_batch([p[0] for p in probs], [p[1] for p in probs],  # noqa: E731
                                               [p[2] for p in probs], R_CORR, [p[3] for p in probs])
    auto = run()
    for flag in (BRUTE, GRID):
        ctx.set_flags(flag)
        try:
            forced = run()
        finally:
            ctx.set_flags(0)
        assert as_bytes(forced[0]) == as_bytes(auto[0]), flag
        assert all(np.array_equal(a, b) for a, b in zip(forced[1], auto[1]))
    assert all(r["iterations"] > 1 for r in auto[0])
