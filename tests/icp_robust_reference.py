"""Numpy float64 restatement of the robust kernels of include/teaser_b200.h (tzr_icp_point_to_plane_robust_batch and
tzr_icp_generalized_robust_batch, DESIGN.md §3.15).

Everything but the weighting is point-to-plane ICP's (tests/icp_plane_reference.py) or generalized ICP's
(tests/icp_generalized_reference.py): the transform, the search, the evaluation, the loop, the 6 x 6 solve and the
Euler update are reused from there.  The generalized system is written as Open3D writes it: W = M^-1/2 from
numpy.linalg.eigh, three whitened rows per correspondence, each with its own weight.  The sums run in numpy's order, so R
and t agree with the device to rounding, not bit for bit.
"""
from __future__ import annotations

import numpy as np

import icp_generalized_reference as gicp
import icp_plane_reference as plane
import rotation_reference
from icp_plane_reference import evaluate, margins, transform  # noqa: F401  (re-exported for the tests)

LOSSES = {"l2": 0, "l1": 1, "huber": 2, "cauchy": 3, "gm": 4, "tukey": 5}


def weight(loss, k, r):
    """The header's weight of kernel `loss` (a LOSSES value) with parameter k, per residual, from e = |r|."""
    e = np.abs(np.asarray(r, dtype=np.float64))
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        if loss == LOSSES["l2"]:
            return np.ones_like(e)
        if loss == LOSSES["l1"]:
            return 1.0 / e
        if loss == LOSSES["huber"]:
            return k / np.maximum(e, k)
        if loss == LOSSES["cauchy"]:
            q = e / k
            return 1.0 / (1.0 + q * q)
        if loss == LOSSES["gm"]:
            t = k + e * e
            return k / (t * t)
        if loss == LOSSES["tukey"]:
            q = e / k
            t = 1.0 - q * q
            return np.where(e > k, 0.0, t * t)
    raise ValueError(f"unknown loss {loss}")


def rho(loss, k, r):
    """Open3D's published loss rho(r) of each kernel, whose rho'(r) / r the weights are."""
    r = np.asarray(r, dtype=np.float64)
    e = np.abs(r)
    if loss == LOSSES["l2"]:
        return 0.5 * r * r
    if loss == LOSSES["l1"]:
        return e
    if loss == LOSSES["huber"]:
        return np.where(e <= k, 0.5 * r * r, k * (e - 0.5 * k))
    if loss == LOSSES["cauchy"]:
        return 0.5 * k * k * np.log1p((r / k) ** 2)
    if loss == LOSSES["gm"]:
        return 0.5 * r * r / (k + r * r)
    if loss == LOSSES["tukey"]:
        return np.where(e <= k, k * k / 6.0 * (1.0 - (1.0 - (r / k) ** 2) ** 3), k * k / 6.0)
    raise ValueError(f"unknown loss {loss}")


# ---- point-to-plane ------------------------------------------------------------------------------------------------

def plane_system(ev, y, normals, centre, loss, k):
    """(A, g) = (sum w J J^T, sum w J r) over the correspondences of an evaluation whose normal is finite and whose
    weight w = weight(r) is finite, J and r as icp_plane_reference.system."""
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
    w = weight(loss, k, r)
    keep = np.isfinite(w)
    J, r, w = J[keep], r[keep], w[keep]
    wJ = w[:, None] * J
    return wJ.T @ J, wJ.T @ r


class PlaneUpdate:
    """The update of tzr_icp_point_to_plane_robust_batch as an icp_plane_reference.icp update_fn."""

    def __init__(self, loss, k):
        self.loss, self.k = int(loss), float(k)

    def __call__(self, ev, y, normals):
        m = ev["idx"] >= 0
        if not m.any():
            return np.eye(3), np.zeros(3)
        c = ev["p"][m].mean(axis=0)
        A, g = plane_system(ev, y, normals, c, self.loss, self.k)
        return _step(A, g, c)


def _step(A, g, c):
    x = plane.solve6(A, g)
    if not np.isfinite(x).all():
        return np.eye(3), np.zeros(3)
    Ru = plane.euler(*x[:3])
    return Ru, (c + x[3:]) - Ru @ c


def icp_plane(x, y, normals, r, loss, k=1.0, s=1.0, R=None, t=None, **kw):
    """The loop of tzr_icp_point_to_plane_robust_batch on one problem.  Returns what icp_reference.icp returns."""
    return plane.icp(x, y, normals, r, s=s, R=R, t=t, update_fn=PlaneUpdate(loss, k), **kw)


# ---- generalized ---------------------------------------------------------------------------------------------------

def whitening_eigh(M):
    """W = M^-1/2 per (3, 3) matrix from numpy.linalg.eigh, and the eigenvalues: (W (n, 3, 3), sigma (n, 3))."""
    sig, V = np.linalg.eigh(M)
    with np.errstate(divide="ignore", invalid="ignore"):
        q = 1.0 / np.sqrt(sig)
    return np.einsum("nak,nk,nbk->nab", V, q, V), sig


def whitening_svd3(M):
    """W = V diag(1 / sqrt(sigma)) V^T from rotation_reference.svd3 (the device's two-sided Jacobi, step for step) in
    the header's order: W_ab = ((V_a0 q_0) V_b0 + (V_a1 q_1) V_b1) + (V_a2 q_2) V_b2."""
    Ws, sigs = [], []
    for Mi in M:
        _, S, V, _ = rotation_reference.svd3(Mi)
        with np.errstate(divide="ignore", invalid="ignore"):
            q = [1.0 / np.sqrt(s) for s in S]
        W = [[((V[a][0] * q[0]) * V[b][0] + (V[a][1] * q[1]) * V[b][1]) + (V[a][2] * q[2]) * V[b][2]
              for b in range(3)] for a in range(3)]
        Ws.append(W)
        sigs.append(S)
    return np.array(Ws, dtype=np.float64).reshape(-1, 3, 3), np.array(sigs, dtype=np.float64).reshape(-1, 3)


def _gicp_terms(ev, y, src_normals, dst_normals, R, s, epsilon, centre, whiten):
    """Per valid correspondence: J (n, 3, 6), d (n, 3), W (n, 3, 3) and sigma (n, 3), normals and M as
    icp_generalized_reference.system."""
    m = ev["idx"] >= 0
    P = ev["p"][m]
    Q = np.asarray(y, dtype=np.float32).astype(np.float64)[ev["idx"][m]]
    Ms = np.asarray(src_normals, dtype=np.float32)[:, :3].astype(np.float64)[np.nonzero(m)[0]]
    Nt = np.asarray(dst_normals, dtype=np.float32)[:, :3].astype(np.float64)[ev["idx"][m]]
    with np.errstate(invalid="ignore", over="ignore"):
        ok = (np.isfinite(Ms).all(axis=1) & np.isfinite(Nt).all(axis=1) & (gicp._len2(Ms) > 0) &
              (gicp._len2(Nt) > 0))
    P, Q, Ms, Nt = P[ok], Q[ok], Ms[ok], Nt[ok]
    R = np.asarray(R, dtype=np.float64)
    Mr = np.stack([(R[r, 0] * Ms[:, 0] + R[r, 1] * Ms[:, 1]) + R[r, 2] * Ms[:, 2] for r in range(3)], axis=1)
    s2 = float(s) * float(s)
    M = s2 * gicp.covariance(Mr, epsilon) + gicp.covariance(Nt, epsilon)
    W, sig = whiten(M) if len(M) else (np.zeros((0, 3, 3)), np.zeros((0, 3)))
    J = gicp.jacobian(P - np.asarray(centre, dtype=np.float64))
    return J, P - Q, W, sig


def gicp_system(ev, y, src_normals, dst_normals, R, s, epsilon, centre, loss, k, whiten=whitening_eigh):
    """(A, g) as Open3D writes them: per correspondence the three rows W_k J with residuals r_k = W_k d and weights
    w_k = weight(r_k), A = sum_k w_k (W_k J)^T (W_k J), g = sum_k w_k (W_k J)^T r_k.  A correspondence adds nothing
    when a normal is invalid, some sigma is not > 0 or not finite, or some w_k is not finite."""
    J, d, W, sig = _gicp_terms(ev, y, src_normals, dst_normals, R, s, epsilon, centre, whiten)
    rows = np.einsum("nkl,nlj->nkj", W, J)
    r = np.einsum("nkl,nl->nk", W, d)
    w = weight(loss, k, r)
    with np.errstate(invalid="ignore"):
        keep = ((sig > 0) & np.isfinite(sig)).all(axis=1) & np.isfinite(w).all(axis=1)
    rows, r, w = rows[keep], r[keep], w[keep]
    return np.einsum("nk,nki,nkj->ij", w, rows, rows), np.einsum("nk,nki,nk->i", w, rows, r)


def gicp_system_atilde(ev, y, src_normals, dst_normals, R, s, epsilon, centre, loss, k, whiten=whitening_eigh):
    """The same system in the device's form: A~ = W diag(w) W once per correspondence, then J^T A~ J and J^T A~ d."""
    J, d, W, sig = _gicp_terms(ev, y, src_normals, dst_normals, R, s, epsilon, centre, whiten)
    r = np.einsum("nkl,nl->nk", W, d)
    w = weight(loss, k, r)
    with np.errstate(invalid="ignore"):
        keep = ((sig > 0) & np.isfinite(sig)).all(axis=1) & np.isfinite(w).all(axis=1)
    J, d, W, w = J[keep], d[keep], W[keep], w[keep]
    At = np.einsum("nka,nk,nkb->nab", W, w, W)
    return np.einsum("nki,nkl,nlj->ij", J, At, J), np.einsum("nki,nkl,nl->i", J, At, d)


class GicpUpdate:
    """The update of tzr_icp_generalized_robust_batch as an icp_plane_reference.icp update_fn; follows the current
    rotation as icp_generalized_reference.Update does."""

    def __init__(self, src_normals, s, R, epsilon, loss, k, whiten=whitening_eigh):
        self.src_normals, self.s, self.epsilon = src_normals, float(s), float(epsilon)
        self.loss, self.k, self.whiten = int(loss), float(k), whiten
        self.R = np.eye(3) if R is None else np.asarray(R, dtype=np.float64).copy()

    def __call__(self, ev, y, dst_normals):
        m = ev["idx"] >= 0
        if not m.any():
            Ru, tu = np.eye(3), np.zeros(3)
        else:
            c = ev["p"][m].mean(axis=0)
            A, g = gicp_system(ev, y, self.src_normals, dst_normals, self.R, self.s, self.epsilon, c, self.loss,
                               self.k, self.whiten)
            Ru, tu = _step(A, g, c)
        self.R = Ru @ self.R
        return Ru, tu


def icp_gicp(x, y, src_normals, dst_normals, r, loss, k=1.0, s=1.0, R=None, t=None, epsilon=1e-3, **kw):
    """The loop of tzr_icp_generalized_robust_batch on one problem.  Returns what icp_reference.icp returns."""
    return plane.icp(x, y, dst_normals, r, s=s, R=R, t=t,
                     update_fn=GicpUpdate(src_normals, s, R, epsilon, loss, k), **kw)


# ---- the clutter fixture -------------------------------------------------------------------------------------------

def _surface(uv):
    z = 0.3 * np.sin(3 * uv[:, 0]) * np.cos(2 * uv[:, 1])
    fx = 0.9 * np.cos(3 * uv[:, 0]) * np.cos(2 * uv[:, 1])
    fy = -0.6 * np.sin(3 * uv[:, 0]) * np.sin(2 * uv[:, 1])
    N = np.stack([-fx, -fy, np.ones(len(uv))], axis=1)
    return np.stack([uv[:, 0], uv[:, 1], z], axis=1), N / np.linalg.norm(N, axis=1, keepdims=True)


def clutter_pair(seed=0, n=3000, offset=0.04, clutter_from=0.3):
    """A partially overlapping scan with clutter: the source is a smooth surface, the target the same sampling moved
    by (R, t), except that its part with u > clutter_from (about a third of the overlap) is replaced by a parallel sheet
    `offset` along the surface normal, well inside the fixture's max_correspondence_distance (0.08).  The seed (R0, t0)
    is (R, t) composed with a small error, so that every true correspondence starts with a residual below the fixture's
    Tukey k.  Returns a dict: src, dst, src_normals, dst_normals ((n, 4) float32), R, t (the truth), R0, t0, r and the
    Tukey k of each method."""
    rng = np.random.default_rng(seed)
    uv = rng.uniform(-1, 1, (n, 2))
    P, N = _surface(uv)
    rot = lambda v: rotation_reference.axis_rotation(v / np.linalg.norm(v), np.linalg.norm(v))  # noqa: E731
    R = rot(np.array([0.02, -0.015, 0.03]))
    t = np.array([0.01, -0.02, 0.015])
    clutter = uv[:, 0] > clutter_from
    Pt = P + offset * clutter[:, None] * N
    src = P.astype(np.float32)
    dst = (Pt @ R.T + t).astype(np.float32)
    pad = np.zeros((n, 1))
    src_n = np.concatenate([N, pad], axis=1).astype(np.float32)
    dst_n = np.concatenate([N @ R.T, pad], axis=1).astype(np.float32)
    dR = rot(np.array([0.002, 0.003, -0.002]))
    R0 = dR @ R
    t0 = dR @ t + np.array([0.003, -0.002, 0.002])
    return dict(src=src, dst=dst, src_normals=src_n, dst_normals=dst_n, R=R, t=t, R0=R0, t0=t0, r=0.08,
                k_plane=0.02, k_gicp=0.1, clutter=clutter)


def pose_error(R, t, R_true, t_true):
    """||R - R_true||_F + ||t - t_true||."""
    return float(np.linalg.norm(np.asarray(R) - R_true) + np.linalg.norm(np.asarray(t) - t_true))
