"""Numpy float64 restatement of the point-to-point ICP of include/teaser_b200.h (tzr_icp, DESIGN.md §3.11).

The transform is computed in the device's operation order, so p_i is bit-identical to the kernel's; the nearest-neighbour
decisions (strict d^2 < r^2, lowest index among equal d^2, no match for non-finite points) are therefore the device's
wherever no decision lies within rounding of a tie, which margins() measures.  The sums run in numpy's order, not the
device's, so R and t agree to rounding, not bit for bit.
"""
from __future__ import annotations

import numpy as np


def transform(x, s, R, t):
    """p = s (R x) + t per point, row r as s * ((R[r,0] x + R[r,1] y) + R[r,2] z) + t[r] (no fused multiply-add)."""
    x = np.asarray(x, dtype=np.float32).astype(np.float64)
    R = np.asarray(R, dtype=np.float64)
    t = np.asarray(t, dtype=np.float64)
    p = np.empty_like(x)
    with np.errstate(invalid="ignore", over="ignore"):  # non-finite points stay non-finite, as on the device
        for r in range(3):
            rx = (R[r, 0] * x[:, 0] + R[r, 1] * x[:, 1]) + R[r, 2] * x[:, 2]
            p[:, r] = s * rx + t[r]
    return p


def sq_dist(p, y):
    """(n, m) matrix of d^2 = (dx dx + dy dy) + dz dz between float64 points p and float targets y."""
    y = np.asarray(y, dtype=np.float32).astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        dx = p[:, None, 0] - y[None, :, 0]
        dy = p[:, None, 1] - y[None, :, 1]
        dz = p[:, None, 2] - y[None, :, 2]
        return (dx * dx + dy * dy) + dz * dz


def nearest(p, y, r2, block=2048):
    """Index of the nearest target with d^2 < r2 (lowest index among equal d^2), -1 where none; and that d^2."""
    n = p.shape[0]
    idx = np.full(n, -1, dtype=np.int64)
    dist = np.zeros(n)
    fin = np.isfinite(p).all(axis=1)
    for a in range(0, n, block):
        d2 = sq_dist(p[a:a + block], y)
        ok = d2 < r2  # NaN and inf compare false
        d2 = np.where(ok, d2, np.inf)
        j = np.argmin(d2, axis=1)  # first minimum: the lowest index
        hit = ok.any(axis=1) & fin[a:a + block]
        idx[a:a + block] = np.where(hit, j, -1)
        dist[a:a + block] = np.where(hit, d2[np.arange(d2.shape[0]), j], 0.0)
    return idx, dist


def margins(p, y, r2, block=2048):
    """How close the nearest-neighbour decisions for the points p came to flipping: tie = the smallest relative gap
    (second - best) / r2 between the two smallest d^2 below r2 of any query, bound = the smallest |d^2 - r2| / r2 of
    any pair.  Both are +inf when there is no such pair."""
    tie, bound = np.inf, np.inf
    fin = np.isfinite(p).all(axis=1)
    for a in range(0, p.shape[0], block):
        d2 = sq_dist(p[a:a + block][fin[a:a + block]], y)
        if d2.size == 0:
            continue
        with np.errstate(invalid="ignore"):
            g = np.abs(d2 - r2) / r2
        g = g[np.isfinite(g)]
        if g.size:
            bound = min(bound, float(g.min()))
        below = np.where(d2 < r2, d2, np.inf)
        if below.shape[1] >= 2:
            two = np.partition(below, 1, axis=1)[:, :2]
            both = np.isfinite(two).all(axis=1)
            if both.any():
                tie = min(tie, float(((two[both, 1] - two[both, 0]) / r2).min()))
    return dict(tie=tie, bound=bound)


def rotation_from_H(H):
    """R = V U^T of H = U S V^T with the reflection fix (utils::svdRot)."""
    U, _, Vt = np.linalg.svd(H)
    V = Vt.T
    if np.linalg.det(U) * np.linalg.det(V) < 0:
        V[:, 2] = -V[:, 2]
    return V @ U.T


def evaluate(x, y, s, R, t, r2):
    p = transform(x, s, R, t)
    idx, d2 = nearest(p, y, r2)
    m = idx >= 0
    count = int(m.sum())
    fitness = count / x.shape[0] if count else 0.0
    rmse = float(np.sqrt(d2[m].sum() / count)) if count else 0.0
    return dict(p=p, idx=idx, count=count, fitness=fitness, rmse=rmse)


def update(ev, y):
    """(R_u, t_u) from the correspondences of an evaluation: centred Kabsch for 3 or more, a translation for 1 or 2,
    the identity for none."""
    m = ev["idx"] >= 0
    count = int(m.sum())
    if count == 0:
        return np.eye(3), np.zeros(3)
    P = ev["p"][m]
    Q = np.asarray(y, dtype=np.float32).astype(np.float64)[ev["idx"][m]]
    mp, mq = P.mean(axis=0), Q.mean(axis=0)
    if count < 3:
        return np.eye(3), mq - mp
    H = (P - mp).T @ (Q - mq)
    Ru = rotation_from_H(H)
    return Ru, mq - Ru @ mp


def icp(x, y, r, s=1.0, R=None, t=None, max_iteration=30, relative_fitness=1e-6, relative_rmse=1e-6, trace=False):
    """The loop of tzr_icp.  Returns a dict with scale, R, t, fitness, inlier_rmse, iterations, n_correspondences,
    converged and corr ((m,2) rows (source, target) ascending by source); with trace=True also margins, the margins()
    of every evaluation."""
    r2 = float(r) * float(r)
    R = np.eye(3) if R is None else np.asarray(R, dtype=np.float64).copy()
    t = np.zeros(3) if t is None else np.asarray(t, dtype=np.float64).copy()
    ev = evaluate(x, y, s, R, t, r2)
    marg = [margins(ev["p"], y, r2)] if trace else []
    iterations, converged = 0, False
    for i in range(max_iteration):
        Ru, tu = update(ev, y)
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
