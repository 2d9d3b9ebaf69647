"""Numpy float64 restatement of tzr_pose_graph_optimize_line_process (include/teaser_b200.h, DESIGN.md §3.22): Open3D's
global_optimization with the Levenberg-Marquardt line process, two passes, pruning and reference compensation.

optimize() makes the device's decisions with the device's reductions (block_sum: the one-block fixed order) and the
device's per-block assembly order, but forms products with numpy and factors with numpy, so it agrees with the device to
rounding, not bit for bit.  Poses are (4,4) float64 rigid matrices; edges are (s, d) with p_d ~ X p_s.
"""
from __future__ import annotations

import numpy as np
import scipy.linalg

import pose_graph_reference as pg

SMALL, LARGE = 256, 1024  # threads of the device's edge-sum and 6K-sum blocks
STOP = {"right_term": 1, "relative_increment": 2, "relative_residual": 3, "lm_trials": 4, "min_residual": 5,
        "max_iteration": 6}
DEFAULTS = dict(edge_prune_threshold=0.25, preference_loop_closure=1.0, reference_node=0, max_iteration=100,
                min_relative_increment=1e-6, min_relative_residual_increment=1e-6, min_right_term=1e-6,
                min_residual=1e-6, max_iteration_lm=20, upper_scale_factor=2.0 / 3.0, lower_scale_factor=1.0 / 3.0)


def block_sum(x, threads):
    """The device's one-block sum: thread t adds x[t], x[t + threads], ... in turn, then the shared-memory tree."""
    x = np.asarray(x, dtype=np.float64).ravel()
    a = np.zeros(threads)
    for lo in range(0, x.size, threads):
        part = x[lo:lo + threads]
        a[:part.size] = a[:part.size] + part
    s = threads >> 1
    while s:
        a[:s] = a[:s] + a[s:2 * s]
        s >>= 1
    return float(a[0])


# ---- the linearisation -------------------------------------------------------------------------------------------------
def lin(N):
    """lin of a 4 x 4 (or 3 x 4) matrix: ((N21 - N12) / 2, (N02 - N20) / 2, (N10 - N01) / 2, N03, N13, N23)."""
    return np.array([0.5 * (N[2, 1] - N[1, 2]), 0.5 * (N[0, 2] - N[2, 0]), 0.5 * (N[1, 0] - N[0, 1]),
                     N[0, 3], N[1, 3], N[2, 3]])


def generators():
    """G_0, G_1, G_2: the skew generators about x, y, z; G_3, G_4, G_5: the unit translations (4 x 4)."""
    G = []
    for i in range(3):
        g = np.zeros((4, 4))
        g[:3, :3] = pg.skew(np.eye(3)[i])
        G.append(g)
    for i in range(3):
        g = np.zeros((4, 4))
        g[i, 3] = 1.0
        G.append(g)
    return G


GEN = generators()


def misalignment(Ts, Td, X):
    return pg.inv(X) @ pg.inv(Td) @ Ts


def zeta(Ts, Td, X):
    return lin(misalignment(Ts, Td, X))


def jacobians(Ts, Td, X):
    """(J_s, J_d): J_s[:, i] = lin(X^-1 T_d^-1 G_i T_s), J_d[:, i] = lin(X^-1 T_d^-1 (-G_i) T_s)."""
    P = pg.inv(X) @ pg.inv(Td)
    Js = np.stack([lin(P @ G @ Ts) for G in GEN], axis=1)
    Jd = np.stack([lin(P @ (-G) @ Ts) for G in GEN], axis=1)
    return Js, Jd


def V(d):
    """Open3D's TransformVector6dToMatrix4d: [R_z(d2) R_y(d1) R_x(d0) | (d3, d4, d5)]."""
    cx, sx, cy, sy, cz, sz = np.cos(d[0]), np.sin(d[0]), np.cos(d[1]), np.sin(d[1]), np.cos(d[2]), np.sin(d[2])
    Rz = np.array([[cz, -sz, 0.0], [sz, cz, 0.0], [0.0, 0.0, 1.0]])
    Ry = np.array([[cy, 0.0, sy], [0.0, 1.0, 0.0], [-sy, 0.0, cy]])
    Rx = np.array([[1.0, 0.0, 0.0], [0.0, cx, -sx], [0.0, sx, cx]])
    T = np.eye(4)
    T[:3, :3] = (Rz @ Ry) @ Rx
    T[:3, 3] = d[3:6]
    return T


def euler(T):
    """Open3D's TransformMatrix4dToVector6d: ZYX Euler angles from atan2 (its sy < 1e-6 branch), then t."""
    R = T[:3, :3]
    sy = np.sqrt(R[0, 0] * R[0, 0] + R[1, 0] * R[1, 0])
    if not sy < 1e-6:
        a = (np.arctan2(R[2, 1], R[2, 2]), np.arctan2(-R[2, 0], sy), np.arctan2(R[1, 0], R[0, 0]))
    else:
        a = (np.arctan2(-R[1, 2], R[1, 1]), np.arctan2(-R[2, 0], sy), 0.0)
    return np.array([a[0], a[1], a[2], T[0, 3], T[1, 3], T[2, 3]])


def confidence(mu, c):
    """The line-process confidence minimising l c + mu (sqrt(l) - 1)^2: (mu / (mu + c))^2."""
    q = mu / (mu + c)
    return q * q


# ---- one pass ------------------------------------------------------------------------------------------------------------
def _terms(P, edges, T, L):
    out = []
    for e, (s, d) in enumerate(edges):
        z = zeta(P[s], P[d], T[e])
        Js, _ = jacobians(P[s], P[d], T[e])
        LJ = L[e] @ Js
        out.append((Js.T @ LJ, Js.T @ (L[e] @ z), float(z @ (L[e] @ z))))
    return out


def _residual(l, terms, mu):
    return block_sum([l[e] * t[2] + mu * ((np.sqrt(l[e]) - 1.0) * (np.sqrt(l[e]) - 1.0)) for e, t in enumerate(terms)],
                     SMALL)


def linear_system(K, edges, live, l, terms):
    """(H, b) over all 6 K unknowns, assembled per block in ascending edge index as the device does."""
    n = 6 * K
    H, b = np.zeros((n, n)), np.zeros(n)
    for e, (s, d) in enumerate(edges):
        if not live[e]:
            continue
        M, v = l[e] * terms[e][0], l[e] * terms[e][1]
        i, j = 6 * s, 6 * d
        H[i:i + 6, i:i + 6] = H[i:i + 6, i:i + 6] + M
        H[j:j + 6, j:j + 6] = H[j:j + 6, j:j + 6] + M
        b[i:i + 6] = b[i:i + 6] + v
        b[j:j + 6] = b[j:j + 6] + (-v)
        lo, hi = (i, j) if i > j else (j, i)
        H[lo:lo + 6, hi:hi + 6] = H[lo:lo + 6, hi:hi + 6] + (-M)
    H = np.tril(H) + np.tril(H, -1).T
    return H, -b


def _pass(K, edges, T, L, unc, live, poses, l, mu, o, trace=None):
    """One pass from poses with confidences l.  Returns (poses, l, F, iterations, trials, reason, terms)."""
    l = np.array(l, dtype=np.float64)
    P = [p.copy() for p in poses]
    cur = _terms(P, edges, T, L)
    F = _residual(l, cur, mu)
    for e in range(len(edges)):
        if unc[e]:
            l[e] = confidence(mu, cur[e][2])
    H, b = linear_system(K, edges, live, l, cur)
    lam, nu = 1e-5 * float(np.max(np.diag(H))), 2.0
    xnorm = np.sqrt(block_sum([np.sum(euler(p) ** 2) for p in P], LARGE))
    it = trials = reason = 0
    if np.max(b) < o["min_right_term"]:
        return P, l, F, 0, 0, STOP["right_term"], cur
    n = 6 * K
    while True:
        it += 1
        lm = 0
        while True:
            lm += 1
            trials += 1
            A = H + lam * np.eye(n)
            try:
                delta = scipy.linalg.cho_solve((np.linalg.cholesky(A), True), b)
                ok = bool(np.isfinite(delta).all())
            except np.linalg.LinAlgError:
                ok = False
            accepted = False
            rec = dict(it=it, lam=lam, F=F) if trace is not None else None
            if ok:
                dnorm = np.sqrt(block_sum(delta * delta, LARGE))
                pred = block_sum(delta * (lam * delta + b), LARGE)
                if rec is not None:
                    rec.update(dnorm=dnorm, dtol=o["min_relative_increment"] * (xnorm + o["min_relative_increment"]))
            if ok and dnorm < o["min_relative_increment"] * (xnorm + o["min_relative_increment"]):
                reason = STOP["relative_increment"]
            else:
                rho = -1.0
                if ok:
                    cand = [V(delta[6 * k:6 * k + 6]) @ P[k] for k in range(K)]
                    cterms = _terms(cand, edges, T, L)
                    Fc = _residual(l, cterms, mu)
                    rho = (F - Fc) / (pred + 1e-3)
                    if rec is not None:
                        rec.update(Fc=Fc, rho=rho)
                if rho > 0 and F - Fc < o["min_relative_residual_increment"] * F:
                    reason = STOP["relative_residual"]
                elif rho > 0:
                    q = 2.0 * rho - 1.0
                    lam = lam * max(o["lower_scale_factor"], min(o["upper_scale_factor"], 1.0 - (q * q) * q))
                    nu = 2.0
                    F, P, cur = Fc, cand, cterms
                    for e in range(len(edges)):
                        if unc[e]:
                            l[e] = confidence(mu, cur[e][2])
                    accepted = True
                else:
                    lam, nu = lam * nu, 2.0 * nu
            if trace is not None:
                rec["outcome"] = "accept" if accepted else "stop" if reason else "reject"
                trace.append(rec)
            if not reason and lm >= o["max_iteration_lm"]:
                reason = STOP["lm_trials"]
            if accepted or reason:
                break
        if reason:
            return P, l, F, it, trials, reason, cur
        # the end of an outer iteration ended by an accepted trial
        H, b = linear_system(K, edges, live, l, cur)
        xnorm = np.sqrt(block_sum([np.sum(euler(p) ** 2) for p in P], LARGE))
        if np.max(b) < o["min_right_term"]:
            return P, l, F, it, trials, STOP["right_term"], cur
        if F < o["min_residual"]:
            return P, l, F, it, trials, STOP["min_residual"], cur
        if it >= o["max_iteration"]:
            return P, l, F, it, trials, STOP["max_iteration"], cur


def _mu(L, idx, c, pref):
    if not len(idx):
        return 0.0
    a = 0.0
    for e in idx:
        a = a + L[e][5, 5]
    return pref * (c * c) * (a / len(idx))


def optimize(K, edges, T, L, c, uncertain=None, init=None, trace=None, **kw):
    """tzr_pose_graph_optimize_line_process.  edges (E,2), T (E,4,4), L (E,6,6).  Returns None for a disconnected graph,
    else a dict: poses (K,4,4), confidence, kept, residuals (zeta^T Lambda zeta at the returned poses), iterations,
    trials, stop_reason, mu (per pass), pruned, residual (the final F).  trace (a list or None) receives one dict per
    trial of both passes."""
    o = dict(DEFAULTS)
    o.update(kw)
    edges = np.asarray(edges).reshape(-1, 2)
    E = edges.shape[0]
    T = [np.asarray(x, dtype=np.float64) for x in T]
    L = [np.asarray(x, dtype=np.float64).copy() for x in L]
    unc = np.zeros(E, dtype=bool) if uncertain is None else np.asarray(uncertain).astype(bool)
    live = [edges[e, 0] != edges[e, 1] and L[e][5, 5] > 0 for e in range(E)]
    Lm = [x if x[5, 5] > 0 else np.zeros((6, 6)) for x in L]  # an edge without information carries none
    ref = o["reference_node"]
    start = pg.bfs(K, edges, T, live, unc, max(ref, 0))
    if start is None:
        return None
    if init is not None:
        start = [np.asarray(x, dtype=np.float64).copy() for x in init]
    pref = o["preference_loop_closure"]
    mu1 = _mu(L, range(E), c, pref)
    P, l1, F, it1, tr1, r1, _ = _pass(K, edges, T, Lm, unc, live, start, np.ones(E), mu1, o, trace)
    keep = [e for e in range(E) if not unc[e] or l1[e] > o["edge_prune_threshold"]]
    mu2 = _mu(L, keep, c, pref)
    P, l2, F, it2, tr2, r2, _ = _pass(K, edges[keep], [T[e] for e in keep], [Lm[e] for e in keep], unc[keep],
                                      [live[e] for e in keep], P, l1[keep], mu2, o, trace)
    if ref >= 0:
        C = start[ref] @ pg.inv(P[ref])
        P = [C @ p for p in P]
    conf = l1.copy()
    conf[keep] = l2
    kept = np.zeros(E, dtype=bool)
    kept[keep] = True
    res = np.array([float(z @ (Lm[e] @ z)) for e in range(E)
                    for z in [zeta(P[edges[e, 0]], P[edges[e, 1]], T[e])]])
    return dict(poses=np.stack(P), confidence=conf, kept=kept, residuals=res, iterations=[it1, it2],
                trials=[tr1, tr2], stop_reason=[r1, r2], mu=[mu1, mu2], pruned=E - len(keep), residual=F)
