"""Numpy float64 restatement of the multiway step of include/teaser_b200.h (DESIGN.md §3.16): the information matrices of
tzr_information_matrix(_batch) and the GNC-TLS pose graph of tzr_pose_graph_optimize.

information() runs tzr_icp's search (icp_reference.nearest) and sums G^T G in the device's chunk order (butterflies
included), so Lambda and the count are the device's bit for bit wherever no nearest-neighbour decision lies within
rounding of a tie.  optimize() makes the device's decisions (the same log and exponential branches, the same cost sums in
the same order, the same accept / reject / stop rules) but factors with numpy, so its poses agree to rounding, not bit
for bit.  Poses are (4,4) float64 rigid matrices.
"""
from __future__ import annotations

import numpy as np
import scipy.linalg

import icp_reference as icp

CHUNK = 256


# ---- information matrices ---------------------------------------------------------------------------------------------
def _butterfly(v):
    """The warp butterfly (xor 16, 8, 4, 2, 1) over axis 0 of a (32, ...) array; every lane ends with the same bits."""
    v = v.copy()
    for o in (16, 8, 4, 2, 1):
        v = v + v[np.arange(32) ^ o]
    return v[0]


def g_terms(q):
    """The 21 upper entries of G^T G (row by row) per target point q (m,3), as the kernel evaluates them."""
    x, y, z = q[:, 0], q[:, 1], q[:, 2]
    zero, one = np.zeros_like(x), np.ones_like(x)
    G = [[zero, z, -y, one, zero, zero], [-z, zero, x, zero, one, zero], [y, -x, zero, zero, zero, one]]
    out = []
    for a in range(6):
        for b in range(a, 6):
            out.append((G[0][a] * G[0][b] + G[1][a] * G[1][b]) + G[2][a] * G[2][b])
    return np.stack(out, axis=1)


def chunk_sum(v):
    """tzr_icp's fixed-order sum of per-source rows v (ns, K): per chunk of 256 the warp butterflies and the warps in
    order, then the chunks by lane k mod 32 and a butterfly."""
    ns, K = v.shape
    nc = (ns + CHUNK - 1) // CHUNK
    pad = np.zeros((nc * CHUNK, K))
    pad[:ns] = v
    parts = []
    for c in range(nc):
        blk = pad[c * CHUNK:(c + 1) * CHUNK].reshape(CHUNK // 32, 32, K)
        s = np.zeros(K)
        for w in range(CHUNK // 32):
            s = s + _butterfly(blk[w])
        parts.append(s)
    lanes = np.zeros((32, K))
    for c, p in enumerate(parts):
        lanes[c % 32] = lanes[c % 32] + p
    return _butterfly(lanes)


def information(x, y, s, R, t, r):
    """(Lambda (6,6), count) of tzr_information_matrix: the source x at (s, R, t) against the target y, distance r."""
    p = icp.transform(x, s, R, t)
    idx, _ = icp.nearest(p, y, float(r) * float(r))
    yf = np.asarray(y, dtype=np.float32).astype(np.float64)
    v = np.zeros((p.shape[0], 21))
    m = idx >= 0
    v[m] = g_terms(yf[idx[m]])
    up = chunk_sum(v)
    L = np.zeros((6, 6))
    k = 0
    for a in range(6):
        for b in range(a, 6):
            L[a, b] = L[b, a] = up[k]
            k += 1
    return L, int(up[20])


def information_direct(x, y, s, R, t, r):
    """Lambda as a plain sum of G^T G over the correspondences (numpy's order): the definition, not the device's order."""
    p = icp.transform(x, s, R, t)
    idx, _ = icp.nearest(p, y, float(r) * float(r))
    yf = np.asarray(y, dtype=np.float32).astype(np.float64)
    L = np.zeros((6, 6))
    for j in idx[idx >= 0]:
        q = yf[j]
        G = np.hstack([-skew(q), np.eye(3)])
        L += G.T @ G
    return L, int((idx >= 0).sum())


# ---- SO(3) / SE(3) ---------------------------------------------------------------------------------------------------
def skew(w):
    return np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])


def so3_log(R):
    """The log of include/teaser_b200.h with its small-angle (theta < 1e-5) and near-pi (c < -0.9) branches."""
    v = 0.5 * np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    s = np.sqrt((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2])
    c = 0.5 * (((R[0, 0] + R[1, 1]) + R[2, 2]) - 1.0)
    th = np.arctan2(s, c)
    if th < 1e-5:
        return (1.0 + th * th / 6.0) * v
    if c < -0.9:
        B = 0.5 * (R + R.T) - c * np.eye(3)
        k = 0
        if B[1, 1] > B[0, 0]:
            k = 1
        if B[2, 2] > B[k, k]:
            k = 2
        a = B[:, k] / np.sqrt(B[k, k] * (1.0 - c))
        if a @ v < 0:
            a = -a
        return th * a
    return (th / s) * v


def se3_exp(x):
    """Exp(omega, tau) in SE(3) as a (4,4) matrix (Rodrigues and V, series below theta = 1e-5)."""
    w, tau = np.asarray(x[:3], dtype=np.float64), np.asarray(x[3:], dtype=np.float64)
    th2 = (w[0] * w[0] + w[1] * w[1]) + w[2] * w[2]
    th = np.sqrt(th2)
    if th < 1e-5:
        A, Bq, Vc = 1.0 - th2 / 6.0, 0.5 - th2 / 24.0, 1.0 / 6.0 - th2 / 120.0
    else:
        A, Bq, Vc = np.sin(th) / th, (1.0 - np.cos(th)) / th2, (th - np.sin(th)) / (th2 * th)
    W = skew(w)
    W2 = W @ W
    T = np.eye(4)
    T[:3, :3] = (np.eye(3) + A * W) + Bq * W2
    T[:3, 3] = ((np.eye(3) + Bq * W) + Vc * W2) @ tau
    return T


def inv(T):
    out = np.eye(4)
    out[:3, :3] = T[:3, :3].T
    out[:3, 3] = -T[:3, :3].T @ T[:3, 3]
    return out


def adjoint(T):
    """Ad(T) = [[R, 0], [[t]x R, R]] for the ordering (omega, tau)."""
    R, t = T[:3, :3], T[:3, 3]
    A = np.zeros((6, 6))
    A[:3, :3] = R
    A[3:, 3:] = R
    A[3:, :3] = skew(t) @ R
    return A


def residual(Ts, Td, Tsd):
    """e = (log R_E, t_E) of E = T_d^-1 T_s T_sd^-1."""
    E = inv(Td) @ Ts @ inv(Tsd)
    return np.concatenate([so3_log(E[:3, :3]), E[:3, 3]])


def jacobians(Td):
    """(J_s, J_d) = (Ad(T_d^-1), -Ad(T_d^-1))."""
    A = adjoint(inv(Td))
    return A, -A


# ---- the pose graph --------------------------------------------------------------------------------------------------
LAMBDA0, LAMBDA_MAX, REL_TOL = 1e-4, 1e8, 1e-10


def _warp_sum(x):
    """The device's one-warp sum: lane l adds x[l], x[l + 32], ... in turn, then the butterfly."""
    lanes = np.zeros(32)
    for e, v in enumerate(x):
        lanes[e % 32] = lanes[e % 32] + v
    return _butterfly(lanes)


def _m33(a, b):
    """a b with entry (r, k) = (a[r,0] b[0,k] + a[r,1] b[1,k]) + a[r,2] b[2,k] (the host's order)."""
    out = np.zeros((3, 3))
    for r in range(3):
        for k in range(3):
            out[r, k] = (a[r, 0] * b[0, k] + a[r, 1] * b[1, k]) + a[r, 2] * b[2, k]
    return out


def _compose(Tu, Tsd, u_is_target):
    """The breadth-first step in the host's operation order: T_s = T_d T_sd, or T_d = T_s T_sd^-1."""
    Ru, tu, R, t = Tu[:3, :3], Tu[:3, 3], Tsd[:3, :3], Tsd[:3, 3]
    out = np.eye(4)
    if u_is_target:
        out[:3, :3] = _m33(Ru, R)
        x = _m33(Ru, np.tile(t[:, None], (1, 3)))[:, 0]
        out[:3, 3] = x + tu
    else:
        Rv = _m33(Ru, R.T.copy())
        out[:3, :3] = Rv
        x = _m33(Rv, np.tile(t[:, None], (1, 3)))[:, 0]
        out[:3, 3] = tu - x
    return out


def bfs(K, edges, T, live, uncertain, ref):
    """Breadth-first initial poses from the reference node (identity): certain edges first, then all; None when some
    node is not reached."""
    adj = [[] for _ in range(K)]
    for e, (s, d) in enumerate(edges):
        if live[e]:
            adj[s].append(e)
            adj[d].append(e)
    poses = [None] * K
    poses[ref] = np.eye(4)
    order = [ref]
    for phase in (0, 1):
        queue = list(order)
        head = 0
        while head < len(queue):
            u = queue[head]
            head += 1
            for e in adj[u]:
                if phase == 0 and uncertain[e]:
                    continue
                s, d = edges[e]
                v = d if u == s else s
                if poses[v] is not None:
                    continue
                poses[v] = _compose(poses[u], T[e], u == d)
                queue.append(v)
                order.append(v)
    return None if len(order) < K else poses


def optimize(K, edges, T, L, c, uncertain=None, init=None, ref=0, gnc_factor=1.4, cost_threshold=1e-6,
             max_iterations=100, max_inner_iterations=10, trace=None):
    """tzr_pose_graph_optimize.  edges (E,2), T (E,4,4), L (E,6,6).  Returns None for a disconnected graph, else a dict:
    poses (K,4,4), weights, mask, residuals (r-bar), iterations, inner_iterations, cost.

    trace (a list, or None): every decision is appended to it, so a test can check that none of them lies within
    rounding of flipping.  Per inner iteration: dict(kind="inner", it, lam, F, Fc (nan when the step was not formed),
    tol (1e-10 F + the floor), eig (the smallest and largest |eigenvalue| of the damped H), factored, outcome: "stop",
    "accept", "reject" or "reject-stop" (lambda past 1e8)).  Per GNC weight update: dict(kind="gnc", it, mu, cost,
    diff)."""
    edges = np.asarray(edges).reshape(-1, 2)
    E = edges.shape[0]
    T = [np.asarray(x, dtype=np.float64) for x in T]
    L = [np.asarray(x, dtype=np.float64).copy() for x in L]
    unc = np.zeros(E, dtype=bool) if uncertain is None else np.asarray(uncertain).astype(bool)
    live = [edges[e, 0] != edges[e, 1] and L[e][5, 5] > 0 for e in range(E)]
    inv_norm = np.zeros(E)
    info_sum = 0.0
    for e in range(E):
        l55 = L[e][5, 5]
        info_sum += l55
        if l55 > 0:
            inv_norm[e] = 1.0 / ((c * c) * l55)
        else:
            L[e][:] = 0.0
    poses = bfs(K, edges, T, live, unc, ref)
    if poses is None:
        return None
    if init is not None:
        poses = [np.asarray(x, dtype=np.float64).copy() for x in init]
    floor = 1e-24 * (c * c) * info_sum
    free = [k for k in range(K) if k != ref]
    fidx = {k: i for i, k in enumerate(free)}
    n = 6 * (K - 1)

    def terms(P):
        out = []
        for e in range(E):
            s, d = edges[e]
            err = residual(P[s], P[d], T[e])
            ce = err @ L[e] @ err
            A = adjoint(inv(P[d]))
            out.append((A.T @ L[e] @ A, A.T @ L[e] @ err, ce, ce * inv_norm[e]))
        return out

    w = np.ones(E)
    cur = terms(poses)
    mu, prev, outer, inner_total, cost = 0.0, np.inf, 0, 0, 0.0
    for it in range(max_iterations):
        cost = _warp_sum([w[e] * cur[e][2] for e in range(E)])
        lam, inner = LAMBDA0, 0
        for _ in range(max_inner_iterations):
            H, g = np.zeros((n, n)), np.zeros(n)
            for e in range(E):
                if not live[e]:
                    continue
                s, d = edges[e]
                M, v = w[e] * cur[e][0], w[e] * cur[e][1]
                for k, sg in ((s, 1.0), (d, -1.0)):
                    if k == ref:
                        continue
                    i = 6 * fidx[k]
                    H[i:i + 6, i:i + 6] += M
                    g[i:i + 6] += sg * v
                if s != ref and d != ref:
                    i, j = 6 * fidx[s], 6 * fidx[d]
                    lo, hi = (i, j) if i > j else (j, i)
                    H[lo:lo + 6, hi:hi + 6] -= M
            H = np.tril(H) + np.tril(H, -1).T
            H[np.diag_indices(n)] += lam * (np.diag(H) + 1.0)
            inner += 1
            rec = None
            if trace is not None:
                ev = np.linalg.eigvalsh(H) if np.isfinite(H).all() else np.array([np.nan])
                rec = dict(kind="inner", it=it, lam=lam, F=cost, tol=REL_TOL * cost + floor,
                           eig=(float(ev[0]), float(np.abs(ev).max())))
                trace.append(rec)
            try:
                C = np.linalg.cholesky(H)
                factored = True
                delta = scipy.linalg.solve_triangular(C.T, scipy.linalg.solve_triangular(C, -g, lower=True),
                                                      lower=False)
                ok = bool(np.isfinite(delta).all())
            except np.linalg.LinAlgError:
                factored = ok = False
            cand_cost = np.nan
            if ok:
                cand = [poses[k] if k == ref else se3_exp(delta[6 * fidx[k]:6 * fidx[k] + 6]) @ poses[k]
                        for k in range(K)]
                cand_terms = terms(cand)
                cand_cost = _warp_sum([w[e] * cand_terms[e][2] for e in range(E)])
                ok = bool(np.isfinite(cand_cost))
            if rec is not None:
                rec.update(Fc=cand_cost, factored=factored)
            if ok and abs(cost - cand_cost) <= REL_TOL * cost + floor:
                if rec is not None:
                    rec["outcome"] = "stop"
                if cand_cost < cost:
                    poses, cur, cost = cand, cand_terms, cand_cost
                break
            if ok and cand_cost < cost:
                poses, cur, cost = cand, cand_terms, cand_cost
                lam = lam * 0.1
                if rec is not None:
                    rec["outcome"] = "accept"
            else:
                lam = lam * 10.0
                if rec is not None:
                    rec["outcome"] = "reject-stop" if lam > LAMBDA_MAX else "reject"
                if lam > LAMBDA_MAX:
                    break
        outer, inner_total = it + 1, inner_total + inner
        if not unc.any():
            break
        rbar = np.array([cur[e][3] for e in range(E)])
        if it == 0:
            # fmax from 0 as the device does (a NaN r-bar is skipped); stop unless mu is finite and positive, which
            # includes max r-bar = 1/2 exactly (mu = +inf would make every weight NaN)
            rmax = np.float64(0.0)
            for r in rbar[unc]:
                rmax = np.fmax(rmax, r)
            with np.errstate(divide="ignore"):
                mu = np.float64(1.0) / (2.0 * rmax - 1.0)
            if not (mu > 0.0 and np.isfinite(mu)):
                break
        th1, th2 = (mu + 1.0) / mu, mu / (mu + 1.0)
        lanes = np.zeros(32)
        for e in range(E):
            if not unc[e]:
                continue
            r = rbar[e]
            lanes[e % 32] = lanes[e % 32] + w[e] * r
            w[e] = 0.0 if r >= th1 else 1.0 if r <= th2 else np.sqrt(mu * (mu + 1.0) / r) - mu
        gc = _butterfly(lanes)
        diff = abs(gc - prev)
        if trace is not None:
            trace.append(dict(kind="gnc", it=it, mu=mu, cost=gc, diff=diff))
        mu, prev = mu * gnc_factor, gc
        if diff < cost_threshold:
            break
    return dict(poses=np.stack(poses), weights=w, mask=w >= 0.5, residuals=np.array([x[3] for x in cur]),
                iterations=outer, inner_iterations=inner_total, cost=cost)
