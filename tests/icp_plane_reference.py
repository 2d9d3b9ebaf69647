"""Numpy float64 restatement of the point-to-plane ICP of include/teaser_b200.h (tzr_icp_point_to_plane, DESIGN.md
§3.13).

The transform, the nearest-neighbour search and the evaluation are point-to-point ICP's (tests/icp_reference.py), so
the correspondences are the device's wherever icp_reference.margins() keeps the decisions clear of ties.  The system's
sums run in numpy's order and sin / cos are the host libm's, so R and t agree with the device to rounding, not bit for
bit.  The 6 x 6 solve is written as plain float64 scalar code, step for step the header's truncated, pivoted LDL^T.
"""
from __future__ import annotations

import math

import numpy as np

from icp_reference import evaluate, margins, nearest, transform  # noqa: F401  (re-exported for the tests)


def system(ev, y, normals, centre):
    """(A, g) = (sum J J^T, sum J r) over the correspondences of an evaluation whose normal is finite, with
    J = ((p - centre) x n, n) and r = ((p0 - q0) n0 + (p1 - q1) n1) + (p2 - q2) n2."""
    m = ev["idx"] >= 0
    P = ev["p"][m]
    Q = np.asarray(y, dtype=np.float32).astype(np.float64)[ev["idx"][m]]
    N = np.asarray(normals, dtype=np.float32)[:, :3].astype(np.float64)[ev["idx"][m]]
    ok = np.isfinite(N).all(axis=1)
    P, Q, N = P[ok], Q[ok], N[ok]
    u = P - np.asarray(centre, dtype=np.float64)
    a = np.stack([u[:, 1] * N[:, 2] - u[:, 2] * N[:, 1], u[:, 2] * N[:, 0] - u[:, 0] * N[:, 2],
                  u[:, 0] * N[:, 1] - u[:, 1] * N[:, 0]], axis=1)
    J = np.concatenate([a, N], axis=1)
    r = ((P[:, 0] - Q[:, 0]) * N[:, 0] + (P[:, 1] - Q[:, 1]) * N[:, 1]) + (P[:, 2] - Q[:, 2]) * N[:, 2]
    return J.T @ J, J.T @ r


def solve6(A, g):
    """x with A x = -g: the truncated LDL^T with diagonal pivoting of the header, in plain float64 scalar code."""
    S = [[float(A[i][j]) for j in range(6)] for i in range(6)]
    amax = max((S[i][i] for i in range(6) if not math.isnan(S[i][i])), default=float("nan"))
    tol = 1e-10 * amax
    used = [False] * 6
    piv, d = [], []
    L = [[0.0] * 6 for _ in range(6)]
    for s in range(6):
        best = -1
        for i in range(6):
            if used[i]:
                continue
            if best < 0 or S[i][i] > S[best][best] or (math.isnan(S[best][best]) and not math.isnan(S[i][i])):
                best = i
        if not S[best][best] > tol:
            break
        used[best] = True
        piv.append(best)
        d.append(S[best][best])
        for i in range(6):
            if not used[i]:
                L[i][s] = S[i][best] / d[s]
        for i in range(6):
            if not used[i]:
                for c in range(6):
                    if not used[c]:
                        S[i][c] = S[i][c] - L[i][s] * S[best][c]
    rank = len(piv)
    y = [0.0] * rank
    for s in range(rank):
        z = -float(g[piv[s]])
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
    x = [0.0] * 6
    for s in range(rank):
        x[piv[s]] = y[s]
    return np.array(x)


def euler(x0, x1, x2):
    """R = Rz(x2) Ry(x1) Rx(x0), written out as in the header."""
    sa, ca, sb, cb, sg, cg = math.sin(x0), math.cos(x0), math.sin(x1), math.cos(x1), math.sin(x2), math.cos(x2)
    return np.array([[cg * cb, (cg * sb) * sa - sg * ca, (cg * sb) * ca + sg * sa],
                     [sg * cb, (sg * sb) * sa + cg * ca, (sg * sb) * ca - cg * sa],
                     [-sb, cb * sa, cb * ca]])


def update(ev, y, normals):
    """(R_u, t_u) of the header: the centred system about c = mu_p, its solve, the Euler rotation, t_u = (c + tau) -
    R_u c; the identity for no correspondence or a non-finite solution."""
    m = ev["idx"] >= 0
    if not m.any():
        return np.eye(3), np.zeros(3)
    c = ev["p"][m].mean(axis=0)
    A, g = system(ev, y, normals, c)
    x = solve6(A, g)
    if not np.isfinite(x).all():
        return np.eye(3), np.zeros(3)
    Ru = euler(*x[:3])
    return Ru, (c + x[3:]) - Ru @ c


def icp(x, y, normals, r, s=1.0, R=None, t=None, max_iteration=30, relative_fitness=1e-6, relative_rmse=1e-6,
        trace=False, update_fn=update):
    """The loop of tzr_icp_point_to_plane (update_fn: the update, for comparisons with other forms).  Returns what
    icp_reference.icp returns."""
    r2 = float(r) * float(r)
    R = np.eye(3) if R is None else np.asarray(R, dtype=np.float64).copy()
    t = np.zeros(3) if t is None else np.asarray(t, dtype=np.float64).copy()
    ev = evaluate(x, y, s, R, t, r2)
    marg = [margins(ev["p"], y, r2)] if trace else []
    iterations, converged = 0, False
    for i in range(max_iteration):
        Ru, tu = update_fn(ev, y, normals)
        R, t = Ru @ R, Ru @ t + tu
        prev = ev
        ev = evaluate(x, y, s, R, t, r2)
        if trace:
            marg.append(margins(ev["p"], y, r2))
        iterations = i + 1
        if abs(prev["fitness"] - ev["fitness"]) < relative_fitness and abs(prev["rmse"] - ev["rmse"]) < relative_rmse:
            converged = True
            break
    src = np.nonzero(ev["idx"] >= 0)[0]
    out = dict(scale=float(s), R=R, t=t, fitness=ev["fitness"], inlier_rmse=ev["rmse"], iterations=iterations,
               n_correspondences=ev["count"], converged=converged,
               corr=np.stack([src, ev["idx"][src]], axis=1).astype(np.int32).reshape(-1, 2))
    if trace:
        out["margins"] = marg
    return out
