"""Numpy float64 restatement of the coloured ICP of include/teaser_b200.h (tzr_estimate_color_gradients and
tzr_icp_colored, DESIGN.md §3.17).

The colour gradients follow the header operation for operation: the float32 radius test, the (d^2, index) order cut to
30 entries, the rows in list order with the constraint row last, and the truncated, pivoted 3 x 3 LDL^T written as
plain float64 scalar code.  So the gradients are the device's bit for bit.  The coloured step reuses point-to-plane's
transform, search, evaluation, loop, 6 x 6 solve and Euler update (tests/icp_plane_reference.py); its sums run in
numpy's order, so R and t agree with the device to rounding.  step_exact() is the one-step form of
tests/icp_exact_reference.py: every sum and the 6 x 6 solve in exact arithmetic from the float inputs, the gradients and
the float64 factors sqrt(lambda) and sqrt(1 - lambda).
"""
from __future__ import annotations

import math
from fractions import Fraction as F

import numpy as np

import icp_exact_reference as ex
import icp_plane_reference as plane
import icp_robust_reference as robust
from icp_plane_reference import evaluate, margins, transform  # noqa: F401  (re-exported for the tests)

NN = 30
LAMBDA_DEFAULT = 0.968
LOSSES = robust.LOSSES


def intensity(colors):
    """((r + g) + b) / 3 per row, in float64 from the float32 colours."""
    c = np.asarray(colors, dtype=np.float32).astype(np.float64)
    return ((c[:, 0] + c[:, 1]) + c[:, 2]) / 3.0


def effective_lambda(lam):
    """Open3D's constructor rule: a value outside [0, 1] becomes 0.968."""
    return LAMBDA_DEFAULT if (lam < 0.0 or lam > 1.0) else float(lam)


# ---- the neighbour lists -------------------------------------------------------------------------------------------

def neighbours(pts, radius, nn=NN):
    """For every point: the local indices of its first min(count, nn) neighbours in (d^2, index) order, d^2 the float32
    ((dx dx + dy dy) + dz dz) of the radius normals and r^2 = float32(radius * radius); a list of int arrays."""
    P = np.asarray(pts, dtype=np.float32)
    r2 = np.float32(float(radius) * float(radius))
    out = []
    idx = np.arange(len(P))
    with np.errstate(invalid="ignore", over="ignore"):
        for k in range(len(P)):
            d = P[k] - P
            d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
            ok = d2 < r2
            cand, dd = idx[ok], d2[ok]
            order = np.lexsort((cand, dd))
            out.append(cand[order][:nn])
    return out


# ---- the 3 x 3 solve -----------------------------------------------------------------------------------------------

def solve3(M, h):
    """x with M x = h by the header's truncated LDL^T with diagonal pivoting (plane.solve6's steps at size 3), plain
    float64 scalar code.  M: 3 x 3 symmetric."""
    N = 3
    S = [[float(M[i][j]) for j in range(N)] for i in range(N)]
    amax = max((S[i][i] for i in range(N) if not math.isnan(S[i][i])), default=float("nan"))
    tol = 1e-10 * amax
    used, piv, d = [False] * N, [], []
    L = [[0.0] * N for _ in range(N)]
    for s in range(N):
        best = -1
        for i in range(N):
            if used[i]:
                continue
            if best < 0 or S[i][i] > S[best][best] or (math.isnan(S[best][best]) and not math.isnan(S[i][i])):
                best = i
        if not S[best][best] > tol:
            break
        used[best] = True
        piv.append(best)
        d.append(S[best][best])
        for i in range(N):
            if not used[i]:
                L[i][s] = S[i][best] / d[s]
        for i in range(N):
            if not used[i]:
                for c in range(N):
                    if not used[c]:
                        S[i][c] = S[i][c] - L[i][s] * S[best][c]
    rank = len(piv)
    y = [0.0] * rank
    for s in range(rank):
        z = float(h[piv[s]])
        for q in range(s):
            z = z - L[piv[s]][q] * y[q]
        y[s] = z
    for s in range(rank):
        y[s] = y[s] / d[s]
    for s in range(rank - 1, -1, -1):
        z = y[s]
        for q in range(s + 1, rank):
            z = z - L[piv[q]][s] * y[q]
        y[s] = z
    x = [0.0] * N
    for s in range(rank):
        x[piv[s]] = y[s]
    return np.array(x)


# ---- colour gradients ----------------------------------------------------------------------------------------------

def gradient_system(pts, normals, colors, k, nb):
    """(M, h) of point k from its neighbour list nb (entry 0 skipped), in the header's order; None when nn < 4."""
    nn = len(nb)
    if nn < 4:
        return None
    P = np.asarray(pts, dtype=np.float32).astype(np.float64)
    n = np.asarray(normals, dtype=np.float32)[k, :3].astype(np.float64)
    I = intensity(colors)
    vk, ik = P[k], I[k]
    M = np.zeros((3, 3))
    h = np.zeros(3)
    with np.errstate(invalid="ignore", over="ignore"):
        for e in range(1, nn):
            v = P[nb[e]]
            s = ((v[0] - vk[0]) * n[0] + (v[1] - vk[1]) * n[1]) + (v[2] - vk[2]) * n[2]
            a = np.array([(v[c] - s * n[c]) - vk[c] for c in range(3)])
            b = I[nb[e]] - ik
            for r in range(3):
                for c in range(3):
                    M[r, c] = M[r, c] + a[r] * a[c]
                h[r] = h[r] + a[r] * b
        w = float(nn - 1)
        cr = np.array([w * n[0], w * n[1], w * n[2]])
        for r in range(3):
            for c in range(3):
                M[r, c] = M[r, c] + cr[r] * cr[c]
    return M, h


def color_gradients(pts, normals, colors, radius, nb=None):
    """The header's gradients of one cloud: (n, 3) float64, bit for bit the device's.  nb: neighbours(), if known."""
    nb = neighbours(pts, radius) if nb is None else nb
    out = np.zeros((len(nb), 3))
    for k, lst in enumerate(nb):
        sys_ = gradient_system(pts, normals, colors, k, lst)
        if sys_ is None:
            continue
        M, h = sys_
        if not (np.isfinite(M).all() and np.isfinite(h).all()):
            out[k] = np.nan
            continue
        out[k] = solve3(M, h)
    return out


# ---- the coloured system -------------------------------------------------------------------------------------------

def _rows(ev, y, normals, src_colors, dst_colors, grad):
    """The correspondences whose normal is finite: transformed source points, target points, normals, gradients,
    source colours and target colours (float64 rows)."""
    m = ev["idx"] >= 0
    j = ev["idx"][m]
    P = ev["p"][m]
    src_i = np.nonzero(m)[0]
    Q = np.asarray(y, dtype=np.float32).astype(np.float64)[j]
    N = np.asarray(normals, dtype=np.float32)[:, :3].astype(np.float64)[j]
    G = np.asarray(grad, dtype=np.float64)[j]
    CS = np.asarray(src_colors, dtype=np.float32).astype(np.float64)[src_i]
    CT = np.asarray(dst_colors, dtype=np.float32).astype(np.float64)[j]
    ok = np.isfinite(N).all(axis=1)
    P, Q, N, G, CS, CT = P[ok], Q[ok], N[ok], G[ok], CS[ok], CT[ok]
    return P, Q, N, G, CS, CT


def system(ev, y, normals, src_colors, dst_colors, grad, centre, lam, loss=None, k=1.0, absolute=False):
    """(A, g): the header's sums of both rows of every correspondence (numpy's order), with the row drop rules.
    absolute: (sum |w| |J| |J|^T, sum |w| |J| |r|, sum |w| |J|) over the same rows instead, the sizes a rounding-error
    bound needs."""
    P, Q, N, G, CS, CT = _rows(ev, y, normals, src_colors, dst_colors, grad)
    sg, si = math.sqrt(lam), math.sqrt(1.0 - lam)
    u = P - np.asarray(centre, dtype=np.float64)
    cross = lambda a, b: np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],  # noqa
                                   a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], axis=1)
    r = ((P[:, 0] - Q[:, 0]) * N[:, 0] + (P[:, 1] - Q[:, 1]) * N[:, 1]) + (P[:, 2] - Q[:, 2]) * N[:, 2]
    A, g = np.zeros((6, 6)), np.zeros(6)
    sj = np.zeros(6) if absolute else None
    lw = LOSSES["l2"] if loss is None else LOSSES.get(loss, loss)
    with np.errstate(invalid="ignore", over="ignore"):
        if sg != 0.0:
            J = sg * np.concatenate([cross(u, N), N], axis=1)
            rg = sg * r
            A, g = _add(A, g, J, rg, lw, k, sj)
        fin = np.isfinite(G).all(1) & np.isfinite(CS).all(1) & np.isfinite(CT).all(1)
        if si != 0.0 and fin.any():
            P2, Q2, N2, G2, u2, r2 = P[fin], Q[fin], N[fin], G[fin], u[fin], r[fin]
            i_s = ((CS[fin, 0] + CS[fin, 1]) + CS[fin, 2]) / 3.0
            i_t = ((CT[fin, 0] + CT[fin, 1]) + CT[fin, 2]) / 3.0
            d = (P2 - r2[:, None] * N2) - Q2
            ihat = ((G2[:, 0] * d[:, 0] + G2[:, 1] * d[:, 1]) + G2[:, 2] * d[:, 2]) + i_t
            mvec = -np.einsum("na,nab->nb", G2, np.eye(3)[None] - N2[:, :, None] * N2[:, None, :])
            J = si * np.concatenate([cross(u2, mvec), mvec], axis=1)
            ri = si * (i_s - ihat)
            A, g = _add(A, g, J, ri, lw, k, sj)
    return (A, g, sj) if absolute else (A, g)


def _add(A, g, J, r, loss, k, sj=None):
    """A + sum w J J^T, g + sum w J r over the rows of finite weight, in the forms of plane.system (L2) and
    robust.plane_system (the kernels), so that lambda = 1 gives their bits.  sj (given: the absolute form): the same
    with |w|, |J| and |r|, and sj += sum |w| |J|."""
    if sj is not None:
        w = np.ones(len(r)) if loss == LOSSES["l2"] else robust.weight(loss, k, r)
        keep = np.isfinite(w)
        aJ, ar, aw = np.abs(J[keep]), np.abs(r[keep]), np.abs(w[keep])
        sj += (aw[:, None] * aJ).sum(axis=0)
        return A + (aw[:, None] * aJ).T @ aJ, g + (aw[:, None] * aJ).T @ ar
    if loss == LOSSES["l2"]:
        return A + J.T @ J, g + J.T @ r
    w = robust.weight(loss, k, r)
    keep = np.isfinite(w)
    J, r, w = J[keep], r[keep], w[keep]
    wJ = w[:, None] * J
    return A + wJ.T @ J, g + wJ.T @ r


class ColoredUpdate:
    """The update of tzr_icp_colored as an icp_plane_reference.icp update_fn (the normals argument is the target's)."""

    def __init__(self, src_colors, dst_colors, grad, lam, loss=None, k=1.0):
        self.sc, self.dc, self.grad = src_colors, dst_colors, grad
        self.lam, self.loss, self.k = effective_lambda(lam), loss, float(k)

    def __call__(self, ev, y, normals):
        m = ev["idx"] >= 0
        if not m.any():
            return np.eye(3), np.zeros(3)
        c = ev["p"][m].mean(axis=0)
        A, g = system(ev, y, normals, self.sc, self.dc, self.grad, c, self.lam, self.loss, self.k)
        x = plane.solve6(A, g)
        if not np.isfinite(x).all():
            return np.eye(3), np.zeros(3)
        Ru = plane.euler(*x[:3])
        return Ru, (c + x[3:]) - Ru @ c


def icp(x, y, normals, src_colors, dst_colors, r, lam=LAMBDA_DEFAULT, loss=None, k=1.0, grad=None, s=1.0, R=None,
        t=None, **kw):
    """The loop of tzr_icp_colored on one problem; grad: the target's gradients (None: color_gradients at 2 r).
    Returns what icp_reference.icp returns, plus the gradients used."""
    if grad is None:
        grad = color_gradients(y, normals, dst_colors, 2.0 * float(r))
    out = plane.icp(x, y, normals, r, s=s, R=R, t=t, update_fn=ColoredUpdate(src_colors, dst_colors, grad, lam, loss,
                                                                              k), **kw)
    out["grad"] = grad
    return out


# ---- one exact step ------------------------------------------------------------------------------------------------

def step_exact(x, y, normals, src_colors, dst_colors, grad, corr, s, R, t, lam, loss=None, k=1.0):
    """One coloured step in exact arithmetic (icp_exact_reference's machinery) from the correspondences corr at the
    seed (s, R, t): both rows of every correspondence with a finite normal, each weighted and dropped by the header's
    rules, the exact sums about c = mu_p, the truncated 6 x 6 solve, Rz Ry Rx."""
    lam = effective_lambda(lam)
    loss = LOSSES.get(loss, loss) if loss is not None else None
    corr = np.asarray(corr, dtype=np.int64).reshape(-1, 2)
    if len(corr) == 0:
        return ex._identity(R, t, 0)
    sg, si = F(math.sqrt(lam)), F(math.sqrt(1.0 - lam))
    P = ex.transform(ex.exact_points(np.asarray(x)[corr[:, 0]]), s, R, t)
    c = ex._mean(P)
    Nf = np.asarray(normals, dtype=np.float32)[:, :3][corr[:, 1]]
    Qf = np.asarray(y)[corr[:, 1]]
    Gf = np.asarray(grad, dtype=np.float64)[corr[:, 1]]
    CSf = np.asarray(src_colors, dtype=np.float32)[corr[:, 0]]
    CTf = np.asarray(dst_colors, dtype=np.float32)[corr[:, 1]]
    A = [[F(0)] * 6 for _ in range(6)]
    g = [F(0)] * 6

    def add(J, r):
        w = F(1) if loss in (None, LOSSES["l2"]) else ex.weight(loss, k, r)
        if w is not None:
            ex._accumulate(A, g, [J], None, r, w)

    for p, qf, nf, gf, csf, ctf in zip(P, Qf, Nf, Gf, CSf, CTf):
        if not ex._finite(nf):
            continue
        n, q = ex.exact_points([nf])[0], ex.exact_points([qf])[0]
        u = [p[i] - c[i] for i in range(3)]
        r = sum(((p[i] - q[i]) * n[i] for i in range(3)), F(0))
        if sg != 0:
            add([sg * v for v in ex._cross(u, n) + n], sg * r)
        if si != 0 and ex._finite(gf) and ex._finite(csf) and ex._finite(ctf):
            gv, cs, ct = ex.exact_points([gf])[0], ex.exact_points([csf])[0], ex.exact_points([ctf])[0]
            i_s, i_t = sum(cs, F(0)) / 3, sum(ct, F(0)) / 3
            d = [(p[i] - r * n[i]) - q[i] for i in range(3)]
            ihat = sum((gv[i] * d[i] for i in range(3)), F(0)) + i_t
            m = [-sum((gv[a] * ((1 if a == b else 0) - n[a] * n[b]) for a in range(3)), F(0)) for b in range(3)]
            add([si * v for v in ex._cross(u, m) + m], si * (i_s - ihat))
    return ex._gn_finish(ex._mirror(A), g, c, R, t, len(corr), {})


# ---- fixtures ------------------------------------------------------------------------------------------------------

def texture(xy):
    """A smooth colour field on the plane: r, g, b in [0, 1] from two sine waves."""
    a = 0.5 + 0.4 * np.sin(9.0 * xy[:, 0]) * np.cos(7.0 * xy[:, 1])
    b = 0.5 + 0.4 * np.cos(5.0 * xy[:, 0] + 3.0 * xy[:, 1])
    return np.stack([a, b, 0.5 * (a + b)], axis=1).astype(np.float32)


def textured_plane(step=0.02, extent=1.0, offset=(0.01, 0.008, 0.0)):
    """A flat target z = 0 on a grid with a smooth texture and normals (0, 0, 1), and a source: the same surface
    sampled on the same grid shifted in-plane by `offset` (so its colour at each point is the texture there).  Returns
    (src, dst, normals, src_colors, dst_colors, offset)."""
    gv = np.arange(-extent, extent, step)
    X, Y = np.meshgrid(gv, gv)
    dst = np.stack([X.ravel(), Y.ravel(), np.zeros(X.size)], axis=1).astype(np.float32)
    nrm = np.tile(np.array([0, 0, 1, 0], dtype=np.float32), (len(dst), 1))
    off = np.asarray(offset, dtype=np.float64)
    src_true = dst.astype(np.float64) + off  # a point of the surface sampled at (x + ox, y + oy)
    src_colors = texture(src_true[:, :2])
    src = dst.copy()  # placed at the target's grid: the in-plane offset is what ICP must find
    return src, dst, nrm, src_colors, texture(dst[:, :2].astype(np.float64)), off
